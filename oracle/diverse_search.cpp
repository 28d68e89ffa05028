// diverse_search.cpp — CPU restatement of the reference's diversity-aware search (test infrastructure only).
//
// Diverse::search (diskann/src/graph/search/diverse_search.rs:189-234): search_internal (diskann/src/graph/index.rs:
// 1933-2000) with scratch.best a DiverseNeighborQueue (diskann/src/neighbor/diverse_priority_queue.rs:90-220), then
// best.post_process() and the strategy's default post-processing of best.iter().take(L): start points and deleted ids
// dropped, the first k kept.  The queue needs three NeighborPriorityQueue operations liboracle's queue does not have —
// remove, retain and truncate (neighbor/queue.rs:197-224, 427-474) — so this file carries its own copy of the queue.
//
// Built on its own into liboracle_diverse_search.so (oracle/diverse_search.mk), linked against liboracle.so for the
// distances.  C ABI (declared here, bound by tests/test_diverse_search.py):
//   NeighborPriorityQueue (fixed capacity):
//     orc_npq* orc_npq_new(uint32_t capacity);  void orc_npq_free(orc_npq*);
//     void orc_npq_insert(orc_npq*, uint32_t id, float dist);  int orc_npq_remove(orc_npq*, uint32_t id, float dist);
//     void orc_npq_retain(orc_npq*, const uint8_t* keep);  (keep[i]: the predicate's value for entry i, in order)
//     void orc_npq_truncate(orc_npq*, uint32_t len);
//     uint32_t orc_npq_size(const orc_npq*);  uint32_t orc_npq_cursor(const orc_npq*);
//     int orc_npq_has_notvisited(const orc_npq*);  int orc_npq_closest_notvisited(orc_npq*, uint32_t* id, float* dist);
//     void orc_npq_get(const orc_npq*, uint32_t i, uint32_t* id, float* dist, int* visited);
//   DiverseNeighborQueue over an attribute table of n_ids ids (ids >= n_ids, or with present[id] == 0, have none):
//     orc_dq* orc_diverse_queue_new(uint32_t l_value, uint32_t k_value, uint32_t diverse_k, const uint32_t* values,
//                                   const uint8_t* present, uint64_t n_ids);
//     void orc_diverse_queue_free(orc_dq*);  void orc_diverse_queue_insert(orc_dq*, uint32_t id, float dist);
//     void orc_diverse_queue_post_process(orc_dq*);  void orc_diverse_queue_clear(orc_dq*);
//     uint32_t orc_diverse_queue_size / _capacity / _search_l / _diverse_l (const orc_dq*);
//     void orc_diverse_queue_get(const orc_dq*, uint32_t i, uint32_t* id, float* dist, int* visited);
//     int orc_diverse_queue_has_notvisited(const orc_dq*);  int orc_diverse_queue_closest_notvisited(orc_dq*, uint32_t*, float*);
//     uint32_t orc_diverse_queue_n_local(const orc_dq*);
//     int orc_diverse_queue_local_size(const orc_dq*, uint32_t attribute);  (-1: no local queue for it)
//     void orc_diverse_queue_local_get(const orc_dq*, uint32_t attribute, uint32_t i, uint32_t* id, float* dist);
//     uint64_t orc_diverse_queue_failed_removals(const orc_dq*);
//   void orc_search_batch_diverse(const orc_index* idx, const void* queries, uint64_t query_stride, uint32_t nq, uint32_t k,
//                                 uint32_t l_search, uint32_t beam_width, uint32_t diverse_k, const uint32_t* attr_values,
//                                 const uint8_t* attr_present, const uint32_t* deleted, int flavour, uint32_t* out_ids,
//                                 float* out_dists, uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops,
//                                 uint64_t* failed_removals);
//     attr_values / attr_present: one entry per id of the index (n_points + n_start); deleted: NULL or a bitmap of
//     (n_total + 31) / 32 words, bit i of word i / 32 for id i.  failed_removals (may be NULL) takes, per query, how many
//     NeighborPriorityQueue::remove calls of the diverse queue found another entry at the lower bound.
#include "oracle.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <unordered_map>
#include <unordered_set>
#include <vector>

namespace {

// NeighborPriorityQueue, fixed capacity (queue.rs:96-106: search_param_l == capacity), with an optional u32 payload per
// entry (the global queue's VectorIdWithAttribute carries the attribute)
struct Npq {
    size_t size = 0, capacity = 0, cursor = 0;
    std::vector<uint32_t> ids, attrs;
    std::vector<uint8_t> visited;
    std::vector<float> dists;

    explicit Npq(size_t cap = 0) : capacity(cap) {}

    // queue.rs:229-280: the first entry whose distance is >= d
    size_t lower_bound(float d) const {
        for (size_t i = 0; i < size; ++i)
            if (dists[i] >= d) return i;
        return size;
    }
    bool is_full() const { return size == capacity; }

    // queue.rs:130-171
    void insert(uint32_t id, float d, uint32_t attr = 0) {
        if (std::isnan(d)) return;
        if (size == capacity && dists[size - 1] < d) return;
        const size_t at = size > 0 ? lower_bound(d) : 0;
        if (size == capacity) {
            ids.pop_back(), attrs.pop_back(), visited.pop_back(), dists.pop_back();
            --size;
        }
        ids.insert(ids.begin() + at, id);
        attrs.insert(attrs.begin() + at, attr);
        visited.insert(visited.begin() + at, 0);
        dists.insert(dists.begin() + at, d);
        ++size;
        if (at < cursor) cursor = at;
    }

    // queue.rs:197-224: only the entry at the lower bound of `d` is looked at
    bool remove(uint32_t id, float d) {
        if (size == 0) return false;
        const size_t at = lower_bound(d);
        if (at < size && ids[at] == id) {
            ids.erase(ids.begin() + at), attrs.erase(attrs.begin() + at), visited.erase(visited.begin() + at), dists.erase(dists.begin() + at);
            --size;
            if (at < cursor && cursor > 0) --cursor;
            return true;
        }
        return false;
    }

    // queue.rs:458-474
    void truncate(size_t len) {
        if (len < size) {
            ids.resize(len), attrs.resize(len), visited.resize(len), dists.resize(len);
            size = len;
            cursor = 0;
        }
    }

    // queue.rs:427-456: keep[i] is the predicate for entry i; order kept, visited flags cleared
    template <class Keep>
    void retain(Keep keep) {
        if (size == 0) return;
        size_t w = 0;
        for (size_t r = 0; r < size; ++r) {
            if (!keep(r)) continue;
            ids[w] = ids[r], attrs[w] = attrs[r], dists[w] = dists[r];
            visited[w] = 0;
            ++w;
        }
        truncate(w);
    }

    // queue.rs:316-318 (search_param_l == capacity)
    bool has_notvisited() const { return cursor < std::min(capacity, size); }

    // queue.rs:297-313: the entry at the cursor, then the cursor moves past visited entries
    bool closest_notvisited(uint32_t* id, float* d) {
        if (!has_notvisited()) return false;
        const size_t cur = cursor;
        visited[cur] = 1;
        ++cursor;
        while (cursor < size && visited[cursor]) ++cursor;
        *id = ids[cur];
        *d = dists[cur];
        return true;
    }
};

// AttributeValueProvider over a table: None for ids past the table or not present
struct Attributes {
    const uint32_t* values;
    const uint8_t* present;
    uint64_t n;
    bool get(uint32_t id, uint32_t* v) const {
        if (id >= n || !present[id]) return false;
        *v = values[id];
        return true;
    }
};

// DiverseNeighborQueue (diverse_priority_queue.rs:66-263)
struct Diverse {
    Npq global;
    std::unordered_map<uint32_t, Npq> local;
    Attributes attrs;
    size_t diverse_l, diverse_k;
    uint64_t failed_removals = 0;

    Diverse(size_t l_value, size_t k_value, size_t dk, Attributes a)
        : global(l_value), attrs(a), diverse_l(dk * l_value / k_value), diverse_k(dk) {}

    // :151-220
    void insert(uint32_t id, float d) {
        uint32_t a;
        if (!attrs.get(id, &a)) return;
        Npq& lq = local.try_emplace(a, diverse_l).first->second;
        const bool local_full = lq.is_full(), global_full = global.is_full();
        if (!local_full && !global_full) {
            lq.insert(id, d);
            global.insert(id, d, a);
        } else if (local_full) {
            if (d < lq.dists[diverse_l - 1]) {
                const uint32_t wid = lq.ids[diverse_l - 1];
                const float wd = lq.dists[diverse_l - 1];
                if (!global.remove(wid, wd)) ++failed_removals;
                lq.insert(id, d);
                global.insert(id, d, a);
            }
        } else if (d < global.dists[global.capacity - 1]) {
            const uint32_t gid = global.ids[global.capacity - 1], ga = global.attrs[global.capacity - 1];
            const float gd = global.dists[global.capacity - 1];
            lq.insert(id, d);
            global.insert(id, d, a);
            auto it = local.find(ga);
            if (it != local.end() && !it->second.remove(gid, gd)) ++failed_removals;
        }
    }

    // :112-138
    void post_process() {
        std::unordered_set<uint32_t> removed;
        for (auto& kv : local) {
            Npq& lq = kv.second;
            if (lq.size > diverse_k) {
                for (size_t i = diverse_k; i < lq.size; ++i) removed.insert(lq.ids[i]);
                lq.truncate(diverse_k);
            }
        }
        if (!removed.empty()) global.retain([&](size_t i) { return removed.count(global.ids[i]) == 0; });
    }

    void clear() {
        global.truncate(0);
        global.cursor = 0;
        local.clear();
    }
};

// the full-precision query distance of graph.cpp's QueryDist (f16 queries widened once, layers/full.rs:421-423)
struct QueryDist {
    const orc_index* idx;
    int flavour, dq;
    const void* q;
    std::vector<float> widened;
    QueryDist(const orc_index* i, const void* query, int fl) : idx(i), flavour(fl), dq(i->dtype), q(query) {
        if (idx->dtype == ORC_F16) {
            widened.resize(idx->dim);
            const uint16_t* h = (const uint16_t*)query;
            for (uint32_t k = 0; k < idx->dim; ++k) widened[k] = orc_f16_to_f32(h[k]);
            dq = ORC_F32;
            q = widened.data();
        }
    }
    float operator()(uint32_t id) const {
        return orc_distance(flavour, dq, idx->dtype, idx->metric, q, (const char*)idx->vectors + (size_t)id * idx->row_stride, idx->dim, nullptr);
    }
};

uint32_t search_one(const orc_index* idx, const void* query, uint32_t k, uint32_t l_search, uint32_t beam_width, uint32_t diverse_k,
                    const Attributes& attrs, const uint32_t* deleted, int flavour, uint32_t* out_ids, float* out_dists, uint32_t* out_cmps,
                    uint32_t* out_hops, uint64_t* failed) {
    const QueryDist dist(idx, query, flavour);
    // Diverse::create_scratch (diverse_search.rs:149-177): the global queue holds L entries, not L + #start
    Diverse best(l_search, k, diverse_k, attrs);
    std::unordered_set<uint32_t> visited;
    uint32_t cmps = 0, hops = 0;
    const uint64_t total = idx->n_points + idx->n_start;
    // start_point_distances (diskann-inmem/src/provider.rs:406-433)
    for (uint32_t s = 0; s < idx->n_start; ++s) {
        const uint32_t id = (uint32_t)(idx->n_points + s);
        visited.insert(id);
        best.insert(id, dist(id));
        ++cmps;
    }
    if (beam_width == 0) beam_width = 1;
    std::vector<uint32_t> beam, list;
    std::vector<float> ds;
    while (best.global.has_notvisited()) {
        beam.clear();
        uint32_t id;
        float d;
        while (beam.size() < beam_width && best.global.closest_notvisited(&id, &d)) beam.push_back(id);
        // expand_beam (provider.rs:436-479): unvisited, in-bounds neighbours of the beam in adjacency order
        list.clear();
        for (uint32_t node : beam) {
            const uint32_t* row = idx->adj + (size_t)node * idx->adj_stride;
            for (uint32_t j = 0; j < row[0]; ++j) {
                const uint32_t n = row[1 + j];
                if (!visited.insert(n).second) continue;
                if (n >= total) continue;
                list.push_back(n);
            }
        }
        ds.clear();
        for (uint32_t n : list) ds.push_back(dist(n));
        for (size_t i = 0; i < list.size(); ++i) best.insert(list[i], ds[i]);
        cmps += (uint32_t)list.size();
        hops += (uint32_t)beam.size();
    }
    best.post_process();
    // best.iter().take(L) through the default post-processor: start points and deleted ids dropped, the first k kept
    const size_t n = std::min<size_t>(best.global.size, l_search);
    uint32_t count = 0;
    for (size_t i = 0; i < n && count < k; ++i) {
        const uint32_t id = best.global.ids[i];
        if (id >= idx->n_points) continue;
        if (deleted && (deleted[id >> 5] >> (id & 31) & 1u)) continue;
        out_ids[count] = id;
        out_dists[count] = best.global.dists[i];
        ++count;
    }
    for (uint32_t i = count; i < k; ++i) {
        out_ids[i] = 0xFFFFFFFFu;
        out_dists[i] = std::numeric_limits<float>::infinity();
    }
    *out_cmps = cmps;
    *out_hops = hops;
    *failed = best.failed_removals;
    return count;
}

}  // namespace

struct orc_npq {
    Npq q;
};
struct orc_dq {
    std::vector<uint32_t> values;
    std::vector<uint8_t> present;
    Diverse q;
    orc_dq(uint32_t l, uint32_t k, uint32_t dk, const uint32_t* v, const uint8_t* p, uint64_t n)
        : values(v, v + n), present(p, p + n), q(l, k, dk, Attributes{nullptr, nullptr, 0}) {
        q.attrs = Attributes{values.data(), present.data(), n};
    }
};

extern "C" {

orc_npq* orc_npq_new(uint32_t capacity) {
    orc_npq* q = new orc_npq();
    q->q.capacity = capacity;
    return q;
}
void orc_npq_free(orc_npq* q) { delete q; }
void orc_npq_insert(orc_npq* q, uint32_t id, float dist) { q->q.insert(id, dist); }
int orc_npq_remove(orc_npq* q, uint32_t id, float dist) { return q->q.remove(id, dist) ? 1 : 0; }
void orc_npq_retain(orc_npq* q, const uint8_t* keep) { q->q.retain([&](size_t i) { return keep[i] != 0; }); }
void orc_npq_truncate(orc_npq* q, uint32_t len) { q->q.truncate(len); }
uint32_t orc_npq_size(const orc_npq* q) { return (uint32_t)q->q.size; }
uint32_t orc_npq_cursor(const orc_npq* q) { return (uint32_t)q->q.cursor; }
int orc_npq_has_notvisited(const orc_npq* q) { return q->q.has_notvisited() ? 1 : 0; }
int orc_npq_closest_notvisited(orc_npq* q, uint32_t* id, float* dist) { return q->q.closest_notvisited(id, dist) ? 1 : 0; }
void orc_npq_get(const orc_npq* q, uint32_t i, uint32_t* id, float* dist, int* visited) {
    *id = q->q.ids[i];
    *dist = q->q.dists[i];
    *visited = q->q.visited[i];
}

orc_dq* orc_diverse_queue_new(uint32_t l_value, uint32_t k_value, uint32_t diverse_k, const uint32_t* values, const uint8_t* present,
                              uint64_t n_ids) {
    return new orc_dq(l_value, k_value, diverse_k, values, present, n_ids);
}
void orc_diverse_queue_free(orc_dq* q) { delete q; }
void orc_diverse_queue_insert(orc_dq* q, uint32_t id, float dist) { q->q.insert(id, dist); }
void orc_diverse_queue_post_process(orc_dq* q) { q->q.post_process(); }
void orc_diverse_queue_clear(orc_dq* q) { q->q.clear(); }
uint32_t orc_diverse_queue_size(const orc_dq* q) { return (uint32_t)q->q.global.size; }
uint32_t orc_diverse_queue_capacity(const orc_dq* q) { return (uint32_t)q->q.global.capacity; }
uint32_t orc_diverse_queue_search_l(const orc_dq* q) { return (uint32_t)q->q.global.capacity; }
uint32_t orc_diverse_queue_diverse_l(const orc_dq* q) { return (uint32_t)q->q.diverse_l; }
void orc_diverse_queue_get(const orc_dq* q, uint32_t i, uint32_t* id, float* dist, int* visited) {
    *id = q->q.global.ids[i];
    *dist = q->q.global.dists[i];
    *visited = q->q.global.visited[i];
}
int orc_diverse_queue_has_notvisited(const orc_dq* q) { return q->q.global.has_notvisited() ? 1 : 0; }
int orc_diverse_queue_closest_notvisited(orc_dq* q, uint32_t* id, float* dist) { return q->q.global.closest_notvisited(id, dist) ? 1 : 0; }
uint32_t orc_diverse_queue_n_local(const orc_dq* q) { return (uint32_t)q->q.local.size(); }
int orc_diverse_queue_local_size(const orc_dq* q, uint32_t attribute) {
    auto it = q->q.local.find(attribute);
    return it == q->q.local.end() ? -1 : (int)it->second.size;
}
void orc_diverse_queue_local_get(const orc_dq* q, uint32_t attribute, uint32_t i, uint32_t* id, float* dist) {
    const Npq& lq = q->q.local.at(attribute);
    *id = lq.ids[i];
    *dist = lq.dists[i];
}
uint64_t orc_diverse_queue_failed_removals(const orc_dq* q) { return q->q.failed_removals; }

void orc_search_batch_diverse(const orc_index* idx, const void* queries, uint64_t query_stride, uint32_t nq, uint32_t k, uint32_t l_search,
                              uint32_t beam_width, uint32_t diverse_k, const uint32_t* attr_values, const uint8_t* attr_present,
                              const uint32_t* deleted, int flavour, uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                              uint32_t* out_cmps, uint32_t* out_hops, uint64_t* failed_removals) {
    const Attributes attrs{attr_values, attr_present, idx->n_points + idx->n_start};
    for (uint32_t q = 0; q < nq; ++q) {
        uint32_t c = 0, h = 0;
        uint64_t f = 0;
        out_counts[q] = search_one(idx, (const char*)queries + (size_t)q * query_stride, k, l_search, beam_width, diverse_k, attrs, deleted,
                                   flavour, out_ids + (size_t)q * k, out_dists + (size_t)q * k, &c, &h, &f);
        out_cmps[q] = c;
        out_hops[q] = h;
        if (failed_removals) failed_removals[q] = f;
    }
}

}  // extern "C"
