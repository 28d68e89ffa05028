// oracle/graph.cpp — CPU restatement of the reference's greedy search, priority queue,
// robust prune and single-insert build.  TEST INFRASTRUCTURE ONLY (see oracle.h).

#include "oracle.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <thread>
#include <vector>

#if defined(__x86_64__)
#include <immintrin.h>
#endif

namespace {

// ------------------------------------------------------------------ NeighborPriorityQueue
// diskann/src/neighbor/queue.rs:66-318 (fixed-capacity flavour; search_param_l == capacity,
// queue.rs:96-106).
struct Queue {
    size_t size = 0, capacity = 0, cursor = 0;
    std::vector<uint32_t> ids;
    std::vector<uint8_t> visited;
    std::vector<float> dists;

    explicit Queue(size_t cap) : capacity(cap) {
        ids.reserve(cap);
        visited.reserve(cap);
        dists.reserve(cap);
    }

    // queue.rs:229-280: index of the first entry with distance >= target (linear scan)
    size_t lower_bound(float d) const {
        for (size_t i = 0; i < size; ++i)
            if (dists[i] >= d) return i;
        return size;
    }

    // queue.rs:130-171
    void insert(uint32_t id, float d) {
        if (std::isnan(d)) return;
        if (size == capacity && dists[size - 1] < d) return;
        size_t idx = size > 0 ? lower_bound(d) : 0;
        if (size == capacity) {
            ids.pop_back();
            visited.pop_back();
            dists.pop_back();
            --size;
        }
        ids.insert(ids.begin() + idx, id);
        visited.insert(visited.begin() + idx, 0);
        dists.insert(dists.begin() + idx, d);
        ++size;
        if (idx < cursor) cursor = idx;
    }

    // queue.rs:316-318
    bool has_notvisited() const { return cursor < std::min(capacity, size); }

    // queue.rs:297-313
    bool closest_notvisited(uint32_t* id, float* d) {
        if (!has_notvisited()) return false;
        size_t cur = cursor;
        visited[cur] = 1;
        ++cursor;
        while (cursor < size && visited[cursor]) ++cursor;
        *id = ids[cur];
        *d = dists[cur];
        return true;
    }
};

// ------------------------------------------------------------------ query distance
struct QueryDist {
    const orc_index* idx;
    int flavour;
    int dq;               // dtype of the prepared query
    const void* q;        // prepared query
    std::vector<float> widened;  // f16 query -> f32 (layers/full.rs:421-423)
    std::vector<float> lut;      // PQ table (TableL2 / TableIP)
    std::vector<float> qf32;     // PQ / SQ: f32 view of the query
    std::vector<uint8_t> sq_query;          // SQ: the compressed query, one code per byte
    mutable std::vector<uint8_t> sq_row;    // SQ: unpacked codes of the row being compared
    float sq_query_comp = 0.0f;

    QueryDist(const orc_index* i, const void* query, int fl) : idx(i), flavour(fl) {
        dq = idx->dtype;
        q = query;
        if (idx->dtype == ORC_F16) {
            widened.resize(idx->dim);
            const uint16_t* h = (const uint16_t*)query;
            for (uint32_t k = 0; k < idx->dim; ++k) widened[k] = orc_f16_to_f32(h[k]);
            dq = ORC_F32;
            q = widened.data();
        }
        if (idx->pq_codes || idx->sq_rows) {
            // providers QuantAccessor: query converted to f32 (T: Into<f32>), then
            // QueryComputer::new (pq/distance/dynamic.rs:63-87)
            qf32.resize(idx->dim);
            for (uint32_t k = 0; k < idx->dim; ++k) {
                switch (idx->dtype) {
                    case ORC_F32: qf32[k] = ((const float*)query)[k]; break;
                    case ORC_F16: qf32[k] = widened[k]; break;
                    case ORC_I8: qf32[k] = (float)((const int8_t*)query)[k]; break;
                    default: qf32[k] = (float)((const uint8_t*)query)[k]; break;
                }
            }
            if (idx->pq_codes && idx->metric != ORC_COSINE) {
                lut.resize((size_t)idx->pq_chunks * idx->pq_centers);
                orc_pq_populate_lut(idx->pq_pivots, idx->pq_centers, idx->dim, idx->pq_offsets,
                                    idx->pq_chunks,
                                    idx->metric == ORC_INNER_PRODUCT ? ORC_INNER_PRODUCT : ORC_L2,
                                    qf32.data(), lut.data());
            }
        }
        if (idx->sq_rows) {
            // SQStore::query_computer(query, is_search = true) (providers inmem/scalar.rs:227-253):
            // for metrics other than L2 / CosineNormalized the query is rescaled to the mean norm
            // of the training data (scalar/quantizer.rs:165-173, 300-310), then compressed with the
            // store's own quantizer into a CompensatedVector<NBITS>.
            if (idx->metric != ORC_L2 && idx->metric != ORC_COSINE_NORMALIZED && idx->sq_mean_norm != 0.0f) {
                const float norm_square = -orc_distance(flavour, ORC_F32, ORC_F32, ORC_INNER_PRODUCT, qf32.data(),
                                                        qf32.data(), idx->dim, nullptr);
                const float norm = std::sqrt(norm_square);
                if (norm != 0.0f) {
                    const float s = idx->sq_mean_norm / norm;
                    for (float& v : qf32) v *= s;
                }
            }
            sq_query.resize(idx->dim);
            sq_row.resize(idx->dim);
            sq_query_comp = orc_sq_compress(idx->sq_shift, idx->sq_scale, idx->dim, idx->sq_nbits, qf32.data(),
                                            sq_query.data(), nullptr);
        }
    }

    float operator()(uint32_t id) const {
        if (idx->sq_rows) {
            // QueryComputer::evaluate_similarity (scalar.rs:310-321) -> DistanceComputer (:267-297)
            const size_t nb = (size_t)idx->sq_nbits, stride = 4 + ((size_t)idx->dim * nb + 7) / 8;
            const uint8_t* row = idx->sq_rows + (size_t)id * stride;
            float comp;
            memcpy(&comp, row, 4);
            for (uint32_t i = 0; i < idx->dim; ++i) {
                const size_t bit = (size_t)i * nb;
                sq_row[i] = (uint8_t)((row[4 + bit / 8] >> (bit % 8)) & ((1u << nb) - 1u));
            }
            return orc_sq_distance(idx->metric, idx->sq_nbits, idx->sq_scale * idx->sq_scale, idx->sq_shift_square_norm,
                                   sq_query.data(), sq_query_comp, sq_row.data(), comp, idx->dim);
        }
        if (idx->pq_codes) {
            const uint8_t* code = idx->pq_codes + (size_t)id * idx->pq_chunks;
            if (idx->metric == ORC_COSINE)
                return orc_pq_direct_distance(idx->pq_pivots, idx->dim, idx->pq_offsets,
                                              idx->pq_chunks, ORC_COSINE, qf32.data(), code);
            return orc_pq_lookup(code, idx->pq_chunks, lut.data(), idx->pq_centers);
        }
        const char* row = (const char*)idx->vectors + (size_t)id * idx->row_stride;
        return orc_distance(flavour, dq, idx->dtype, idx->metric, q, row, idx->dim, nullptr);
    }
};

struct Visit {
    uint32_t id;
    float dist;
};

// The reference's visited set is a hashbrown HashSet<u32> created with the capacity estimate of
// scratch.rs:186-192 and kept in the pooled search scratch (cleared, not reallocated, between
// queries).  Same behaviour here: flat open addressing, 7/8 load factor, doubling growth.
struct VisitedSet {
    static constexpr uint32_t kEmpty = 0xFFFFFFFFu;
    std::vector<uint32_t> slots;
    size_t count = 0;
    bool has_empty_key = false;  // the one id that collides with the empty marker
    uint32_t shift = 28;

    void reset(size_t expected) {
        size_t cap = 16;
        while (cap * 7 / 8 < expected) cap <<= 1;
        if (slots.size() != cap) slots.assign(cap, kEmpty);
        else std::fill(slots.begin(), slots.end(), kEmpty);
        set_shift();
        count = 0;
        has_empty_key = false;
    }
    void set_shift() {
        uint32_t lg = 0;
        while (((size_t)1 << lg) < slots.size()) ++lg;
        shift = 32 - lg;
    }
    void grow() {
        std::vector<uint32_t> old;
        old.swap(slots);
        slots.assign(old.size() * 2, kEmpty);
        set_shift();
        for (uint32_t v : old)
            if (v != kEmpty) place(v);
    }
    void place(uint32_t id) {
        const size_t mask = slots.size() - 1;
        size_t h = (size_t)((id * 0x9E3779B1u) >> shift);
        while (slots[h] != kEmpty) h = (h + 1) & mask;
        slots[h] = id;
    }
    // HashSet::insert: true when the id was not present
    bool insert(uint32_t id) {
        if (id == kEmpty) {
            const bool fresh = !has_empty_key;
            has_empty_key = true;
            return fresh;
        }
        const size_t mask = slots.size() - 1;
        size_t h = (size_t)((id * 0x9E3779B1u) >> shift);
        while (slots[h] != kEmpty) {
            if (slots[h] == id) return false;
            h = (h + 1) & mask;
        }
        if ((count + 1) * 8 > slots.size() * 7) {
            grow();
            place(id);
        } else {
            slots[h] = id;
        }
        ++count;
        return true;
    }
};

// pooled per-thread search scratch (graph/search/scratch.rs)
struct SearchScratch {
    VisitedSet visited;
    std::vector<uint32_t> beam, list;
    std::vector<Visit> neighbors;
};

inline void prefetch_bytes(const void* p, size_t bytes) {
#if defined(__x86_64__)
    for (size_t off = 0; off < bytes; off += 64) _mm_prefetch((const char*)p + off, _MM_HINT_T0);
#else
    (void)p;
    (void)bytes;
#endif
}

// diskann/src/graph/index.rs:1933-2000.  `record` (optional) receives the nodes picked for
// expansion in order (VisitedSearchRecord, used by insert).
void search_internal(const orc_index* idx, const QueryDist& qd, uint32_t l_search,
                     uint32_t beam_width, Queue& best, uint32_t* cmps_out, uint32_t* hops_out,
                     std::vector<Visit>* record) {
    static thread_local SearchScratch scratch;
    VisitedSet& visited = scratch.visited;
    // estimate_node_visited_set_size (scratch.rs:186-192): 1.1 * max_degree * 1.3 * L
    visited.reset((size_t)(1.1 * (double)(idx->adj_stride ? idx->adj_stride - 1 : 64) * 1.3 * (double)l_search) + 1);
    uint32_t cmps = 0, hops = 0;
    const uint64_t total = idx->n_points + idx->n_start;
    // start_point_distances (diskann-inmem/src/provider.rs:406-433)
    for (uint32_t s = 0; s < idx->n_start; ++s) {
        uint32_t id = (uint32_t)(idx->n_points + s);
        visited.insert(id);
        best.insert(id, qd(id));
        ++cmps;
    }
    std::vector<uint32_t>& beam = scratch.beam;
    std::vector<uint32_t>& list = scratch.list;
    std::vector<Visit>& neighbors = scratch.neighbors;
    // what one distance evaluation reads (the row, or the PQ code of the point)
    const size_t sq_stride = idx->sq_rows ? 4 + ((size_t)idx->dim * (size_t)idx->sq_nbits + 7) / 8 : 0;
    const char* fetch_base = idx->sq_rows ? (const char*)idx->sq_rows : idx->pq_codes ? (const char*)idx->pq_codes : (const char*)idx->vectors;
    const size_t fetch_stride = idx->sq_rows ? sq_stride : idx->pq_codes ? (size_t)idx->pq_chunks : (size_t)idx->row_stride;
    size_t fetch_bytes = fetch_stride;
    if (!idx->pq_codes && !idx->sq_rows) {
        const size_t es = idx->dtype == ORC_F32 ? 4 : idx->dtype == ORC_F16 ? 2 : 1;
        fetch_bytes = (size_t)idx->dim * es;
    }
    if (beam_width == 0) beam_width = 1;
    while (best.has_notvisited()) {
        beam.clear();
        uint32_t id;
        float d;
        while (beam.size() < beam_width && best.closest_notvisited(&id, &d)) {
            if (record) record->push_back(Visit{id, d});
            beam.push_back(id);
        }
        neighbors.clear();
        // expand_beam (diskann-inmem/src/provider.rs:436-479): filter the adjacency lists ...
        list.clear();
        for (uint32_t node : beam) {
            const uint32_t* row = idx->adj + (size_t)node * idx->adj_stride;
            uint32_t deg = row[0];
            for (uint32_t j = 0; j < deg; ++j) {
                uint32_t n = row[1 + j];
                if (!visited.insert(n)) continue;  // pred.eval_mut
                if (n >= total) continue;          // is_in_bounds
                list.push_back(n);
            }
        }
        // ... then expand_beam_inner (provider.rs:620-690): distances in list order with the
        // rows prefetched `lookahead` = 8 entries ahead (Config::DEFAULT_PREFETCH_LOOKAHEAD, :169)
        {
            const size_t len = list.size(), lookahead = std::min<size_t>(8, len);
            for (size_t j = 0; j < lookahead; ++j) prefetch_bytes(fetch_base + (size_t)list[j] * fetch_stride, fetch_bytes);
            size_t j = lookahead == 0 ? len : lookahead;
            for (uint32_t n : list) {
                if (j != len) {
                    prefetch_bytes(fetch_base + (size_t)list[j] * fetch_stride, fetch_bytes);
                    ++j;
                }
                neighbors.push_back(Visit{n, qd(n)});
            }
        }
        for (const Visit& v : neighbors) best.insert(v.id, v.dist);
        cmps += (uint32_t)neighbors.size();
        hops += (uint32_t)beam.size();
    }
    *cmps_out = cmps;
    *hops_out = hops;
}

uint32_t search_one(const orc_index* idx, const void* query, uint32_t k, uint32_t l_search,
                    uint32_t beam_width, int flavour, uint32_t* out_ids, float* out_dists,
                    uint32_t* out_cmps, uint32_t* out_hops, bool rerank = false) {
    QueryDist qd(idx, query, flavour);
    // scratch.rs:195-208: queue capacity = L + number of start points
    Queue best((size_t)l_search + idx->n_start);
    uint32_t cmps = 0, hops = 0;
    search_internal(idx, qd, l_search, beam_width, best, &cmps, &hops, nullptr);
    if (rerank) {
        // Pipeline<FilterStartPoints, Rerank> (providers .../inmem/product.rs:391-400,
        // full_precision.rs:356-399): every entry of best.iter() that is not a start point gets its
        // full-precision Distance<T, T> to the query, the list is sorted by that distance
        // (`sort_unstable_by`: the order of exactly tied entries is unspecified in the reference;
        // here ties keep their traversal order) and the output buffer takes the first k.
        std::vector<Visit> cand;
        size_t n = std::min(best.capacity, best.size);
        for (size_t i = 0; i < n; ++i) {
            if (best.ids[i] >= idx->n_points) continue;
            const char* row = (const char*)idx->vectors + (size_t)best.ids[i] * idx->row_stride;
            cand.push_back(Visit{best.ids[i], orc_distance(flavour, idx->dtype, idx->dtype, idx->metric, query, row, idx->dim, nullptr)});
        }
        std::stable_sort(cand.begin(), cand.end(), [](const Visit& a, const Visit& b) { return a.dist < b.dist; });
        uint32_t count = (uint32_t)std::min<size_t>(k, cand.size());
        for (uint32_t i = 0; i < count; ++i) {
            out_ids[i] = cand[i].id;
            out_dists[i] = cand[i].dist;
        }
        for (uint32_t i = count; i < k; ++i) {
            out_ids[i] = 0xFFFFFFFFu;
            out_dists[i] = std::numeric_limits<float>::infinity();
        }
        if (out_cmps) *out_cmps = cmps;
        if (out_hops) *out_hops = hops;
        return count;
    }
    // post-process (diskann-inmem/src/provider.rs:907-950): skip ids with no external
    // mapping (start points), stop when the output buffer is full.
    uint32_t count = 0;
    size_t n = std::min(best.capacity, best.size);
    for (size_t i = 0; i < n && count < k; ++i) {
        if (best.ids[i] >= idx->n_points) continue;
        out_ids[count] = best.ids[i];
        out_dists[count] = best.dists[i];
        ++count;
    }
    for (uint32_t i = count; i < k; ++i) {
        out_ids[i] = 0xFFFFFFFFu;
        out_dists[i] = std::numeric_limits<float>::infinity();
    }
    if (out_cmps) *out_cmps = cmps;
    if (out_hops) *out_hops = hops;
    return count;
}

// ------------------------------------------------------------------ prune
struct State {
    float occlude_factor = 0.0f;
    uint16_t last_checked = 0;
    uint16_t neighbor = 0;
};

float pair_distance(const orc_index* idx, int flavour, uint32_t a, uint32_t b) {
    const char* base = (const char*)idx->vectors;
    return orc_distance(flavour, idx->dtype, idx->dtype, idx->metric, base + (size_t)a * idx->row_stride,
                        base + (size_t)b * idx->row_stride, idx->dim, nullptr);
}

// diskann/src/graph/internal/prune.rs:106-259
uint32_t robust_prune(const orc_index* idx, const uint32_t* pool_ids, const float* pool_dists,
                      const uint8_t* excluded, uint32_t pool_len, uint32_t degree, float alpha,
                      int flavour, uint32_t* out_pos, uint64_t* ncmp) {
    std::vector<State> states(pool_len);
    const int kind = idx->metric == ORC_INNER_PRODUCT ? 1 : 0;  // config/mod.rs:69-76
    float current_alpha = 1.0f;
    const float increment_factor = std::fmin(alpha, 1.2f);
    uint32_t found = 0;
    uint64_t cmp = 0;
    while (found < degree) {
        for (uint32_t i = 0; i < pool_len; ++i) {
            if (found >= degree) break;
            float occlude_factor = states[i].occlude_factor;
            uint16_t last_checked = states[i].last_checked;
            if (occlude_factor > current_alpha) continue;
            if (excluded && excluded[i]) {
                states[i].occlude_factor = std::numeric_limits<float>::max();
                continue;
            }
            while (last_checked != found) {
                uint32_t result_position = states[last_checked].neighbor;
                ++last_checked;
                if (result_position >= i) {
                    states[i].last_checked = last_checked;
                    continue;
                }
                float distance = (excluded && excluded[result_position])
                                     ? std::numeric_limits<float>::max()
                                     : pair_distance(idx, flavour, pool_ids[i], pool_ids[result_position]);
                ++cmp;
                occlude_factor = orc_update_occlude_factor(kind, pool_dists[i], distance,
                                                           occlude_factor, current_alpha);
                if (occlude_factor > current_alpha) break;
            }
            states[i].last_checked = last_checked;
            if (occlude_factor > current_alpha) {
                states[i].occlude_factor = occlude_factor;
                continue;
            }
            states[i].occlude_factor = std::numeric_limits<float>::max();
            states[found].neighbor = (uint16_t)i;
            ++found;
        }
        if (current_alpha == alpha) break;
        current_alpha = std::fmin(current_alpha * increment_factor, alpha);
    }
    for (uint32_t n = 0; n < found; ++n) out_pos[n] = states[n].neighbor;
    if (ncmp) *ncmp = cmp;
    return found;
}

// SortedNeighbors::new (graph/internal/sorted_neighbors.rs:26-44): `select_nth_unstable_by` at
// the last position, then `sort_unstable_by` of the prefix, by distance only.  The order of
// exactly tied candidates is whatever the Rust standard library's algorithms leave; the parts of
// them that are simple are followed here, because the lattice baselines are full of ties:
//   * selecting the last position swaps the FIRST maximum to the end (core::slice::select,
//     `index == len - 1`);
//   * a prefix of at most 20 elements is insertion-sorted, which is stable;
//   * a longer prefix that is already non-descending is left alone, a strictly descending one is
//     reversed (ipnsort's run detection);
//   * anything else goes through ipnsort's quicksort, whose tie order is NOT restated: a stable
//     sort stands in for it.

//
// The emulation is opt-in (orc_set_pool_tie_mode(1), used by the grid_insert golden test): the
// default stays the plain stable sort, so that the graphs the GPU parity tests are built on are
// the ones the kernels were validated with.
static int g_pool_tie_mode = 0;

void sort_pool(std::vector<Visit>& pool, size_t max) {
    auto less = [](const Visit& a, const Visit& b) { return a.dist < b.dist; };
    const size_t len = pool.size();
    if (len > max || g_pool_tie_mode == 0) {  // (never the case below MAX_OCCLUSION; kept for completeness)
        std::stable_sort(pool.begin(), pool.end(), less);
        if (len > max) pool.resize(max);
        return;
    }
    if (len < 2) return;
    size_t mx = 0;
    for (size_t i = 1; i < len; ++i)
        if (less(pool[mx], pool[i])) mx = i;
    std::swap(pool[mx], pool[len - 1]);
    const size_t n = len - 1;  // the prefix
    if (n < 2) return;
    if (n <= 20) {
        for (size_t i = 1; i < n; ++i) {
            Visit v = pool[i];
            size_t j = i;
            while (j > 0 && less(v, pool[j - 1])) {
                pool[j] = pool[j - 1];
                --j;
            }
            pool[j] = v;
        }
        return;
    }
    size_t run = 2;
    const bool descending = less(pool[1], pool[0]);
    if (descending) {
        while (run < n && less(pool[run], pool[run - 1])) ++run;
    } else {
        while (run < n && !less(pool[run], pool[run - 1])) ++run;
    }
    if (run == n) {
        if (descending) std::reverse(pool.begin(), pool.begin() + n);
        return;
    }
    std::stable_sort(pool.begin(), pool.begin() + n, less);
}

constexpr size_t MAX_OCCLUSION = 750;  // graph/config/defaults.rs:13

// occlude_list (index.rs:2565-2650) without saturation (defaults.rs SATURATE_AFTER_PRUNE=false)
void occlude_list(const orc_index* idx, std::vector<Visit>& pool, uint32_t location,
                  uint32_t degree, float alpha, int flavour, std::vector<uint32_t>& out) {
    out.clear();
    if (pool.empty()) return;
    std::vector<uint32_t> ids(pool.size()), pos(pool.size());
    std::vector<float> dists(pool.size());
    std::vector<uint8_t> excl(pool.size());
    for (size_t i = 0; i < pool.size(); ++i) {
        ids[i] = pool[i].id;
        dists[i] = pool[i].dist;
        excl[i] = pool[i].id == location;
    }
    uint32_t found = robust_prune(idx, ids.data(), dists.data(), excl.data(), (uint32_t)pool.size(),
                                  degree, alpha, flavour, pos.data(), nullptr);
    for (uint32_t n = 0; n < found; ++n) out.push_back(ids[pos[n]]);
}

}  // namespace

extern "C" {

// graph/config/mod.rs:80-103
float orc_update_occlude_factor(int kind, float d_ik, float d_jk, float cur, float alpha) {
    if (kind == 0) {
        if (d_jk == 0.0f) return std::numeric_limits<float>::max();
        return std::fmax(cur, d_ik / d_jk);  // f32::max
    }
    if (d_jk < alpha * d_ik) return alpha + 0.01f;  // OCCLUDING_MASK, config/mod.rs:62
    return cur;
}

uint32_t orc_robust_prune(const orc_index* idx, const uint32_t* pool_ids,
                          const float* pool_dists, const uint8_t* excluded, uint32_t pool_len,
                          uint32_t degree, float alpha, int flavour, uint32_t* out_pos,
                          uint64_t* out_ncmp) {
    return robust_prune(idx, pool_ids, pool_dists, excluded, pool_len, degree, alpha, flavour,
                        out_pos, out_ncmp);
}

uint32_t orc_search(const orc_index* idx, const void* query, uint32_t k, uint32_t l_search,
                    uint32_t beam_width, int flavour, uint32_t* out_ids, float* out_dists,
                    uint32_t* out_cmps, uint32_t* out_hops) {
    return search_one(idx, query, k, l_search, beam_width, flavour, out_ids, out_dists, out_cmps,
                      out_hops);
}

// benchmark-core/src/search/api.rs:400-434 (PartitionIter: contiguous ranges, the first
// nq % T ranges one longer).
static void search_batch_impl(const orc_index* idx, const void* queries, uint64_t query_stride,
                              uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                              int flavour, int n_threads, uint32_t* out_ids, float* out_dists,
                              uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops, bool rerank);

void orc_search_batch(const orc_index* idx, const void* queries, uint64_t query_stride,
                      uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                      int flavour, int n_threads, uint32_t* out_ids, float* out_dists,
                      uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops) {
    search_batch_impl(idx, queries, query_stride, nq, k, l_search, beam_width, flavour, n_threads, out_ids, out_dists,
                      out_counts, out_cmps, out_hops, false);
}

void orc_search_batch_rerank(const orc_index* idx, const void* queries, uint64_t query_stride,
                             uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                             int flavour, int n_threads, uint32_t* out_ids, float* out_dists,
                             uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops) {
    search_batch_impl(idx, queries, query_stride, nq, k, l_search, beam_width, flavour, n_threads, out_ids, out_dists,
                      out_counts, out_cmps, out_hops, true);
}

static void search_batch_impl(const orc_index* idx, const void* queries, uint64_t query_stride,
                              uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                              int flavour, int n_threads, uint32_t* out_ids, float* out_dists,
                              uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops, bool rerank) {
    if (n_threads < 1) n_threads = 1;
    if ((uint32_t)n_threads > nq) n_threads = nq ? (int)nq : 1;
    auto work = [&](uint32_t lo, uint32_t hi) {
        for (uint32_t i = lo; i < hi; ++i) {
            uint32_t c = 0, h = 0;
            uint32_t cnt = search_one(idx, (const char*)queries + (size_t)i * query_stride, k,
                                      l_search, beam_width, flavour, out_ids + (size_t)i * k,
                                      out_dists + (size_t)i * k, &c, &h, rerank);
            if (out_counts) out_counts[i] = cnt;
            if (out_cmps) out_cmps[i] = c;
            if (out_hops) out_hops[i] = h;
        }
    };
    if (n_threads == 1) {
        work(0, nq);
        return;
    }
    std::vector<std::thread> ts;
    uint32_t base = nq / n_threads, extra = nq % n_threads, lo = 0;
    for (int t = 0; t < n_threads; ++t) {
        uint32_t len = base + ((uint32_t)t < extra ? 1 : 0);
        ts.emplace_back(work, lo, lo + len);
        lo += len;
    }
    for (auto& t : ts) t.join();
}

// DiskANNIndex::insert for i = 0..n_points (index.rs:226-341), add_edge_and_prune
// (index.rs:2264-2341), robust_prune_list (index.rs:2397-2454).  max_backedges defaults to
// pruned_degree (config/mod.rs:292-306).
// provider-level write counters of the last orc_build (the reference's test provider reports the
// same two numbers as `set_neighbors` / `append_neighbors`, test/provider.rs Metrics)
static uint64_t g_build_sets = 0, g_build_appends = 0;

void orc_build(int dtype, int metric, uint32_t dim, uint64_t n_points, uint32_t n_start,
               const void* vectors, uint64_t row_stride, uint32_t pruned_degree,
               uint32_t max_degree, uint32_t l_build, float alpha, uint32_t* adj,
               uint32_t adj_stride) {
    orc_index idx;
    std::memset(&idx, 0, sizeof(idx));
    idx.dtype = dtype;
    idx.metric = metric;
    idx.dim = dim;
    idx.n_points = n_points;
    idx.n_start = n_start;
    idx.vectors = vectors;
    idx.row_stride = row_stride;
    idx.adj = adj;
    idx.adj_stride = adj_stride;
    const int flavour = ORC_FLAVOUR_AVX2;
    auto row = [&](uint32_t id) { return adj + (size_t)id * adj_stride; };
    auto set_neighbors = [&](uint32_t id, const std::vector<uint32_t>& v) {
        uint32_t* r = row(id);
        r[0] = (uint32_t)v.size();
        for (size_t j = 0; j < v.size(); ++j) r[1 + j] = v[j];
    };
    std::vector<Visit> record, pool;
    std::vector<uint32_t> new_neighbors, pruned, list;
    g_build_sets = g_build_appends = 0;
    for (uint64_t p = 0; p < n_points; ++p) {
        uint32_t id = (uint32_t)p;
        const void* vec = (const char*)vectors + (size_t)id * row_stride;
        QueryDist qd(&idx, vec, flavour);
        Queue best((size_t)l_build + n_start);
        uint32_t cmps = 0, hops = 0;
        record.clear();
        search_internal(&idx, qd, l_build, 1, best, &cmps, &hops, &record);
        sort_pool(record, MAX_OCCLUSION);
        occlude_list(&idx, record, id, pruned_degree, alpha, flavour, new_neighbors);
        set_neighbors(id, new_neighbors);
        ++g_build_sets;
        size_t nb = std::min<size_t>(new_neighbors.size(), pruned_degree);
        for (size_t s = 0; s < nb; ++s) {
            uint32_t source = new_neighbors[s];
            uint32_t* r = row(source);
            uint32_t deg = r[0];
            bool present = false;
            for (uint32_t j = 0; j < deg; ++j) present |= r[1 + j] == id;
            if (present) continue;
            if (deg + 1 <= max_degree) {
                r[1 + deg] = id;
                r[0] = deg + 1;
                ++g_build_appends;
                continue;
            }
            list.assign(r + 1, r + 1 + deg);
            list.push_back(id);
            pool.clear();
            for (uint32_t other : list)
                if (other != source) pool.push_back(Visit{other, pair_distance(&idx, flavour, source, other)});
            sort_pool(pool, MAX_OCCLUSION);
            occlude_list(&idx, pool, source, pruned_degree, alpha, flavour, pruned);
            set_neighbors(source, pruned);
            ++g_build_sets;
        }
    }
}

// DiskANNIndex::multi_insert (index.rs:815-1050) with intra_batch_candidates = None and the bootstrap
// branch not taken (it is meant for the first batches of ~128 items and costs O(batch^2) distances;
// the device build grows its batches instead, see orc_build_batch_size), one batch at a time:
//   * candidate generation (search_and_prune, index.rs:341-430): every item is searched against the
//     graph AS IT WAS BEFORE THE BATCH with a VisitedSearchRecord and pruned (robust_prune_with without
//     extras); nothing is written yet;
//   * aggregate_backedges (index.rs:123-143): target -> sources, sources sorted (index.rs:986-992);
//   * set_neighbors_bulk of the new out-lists;
//   * add_edge_and_prune(sorted sources, target) (index.rs:2264-2341): ALL new sources are appended
//     (extend_from_slice skips the ones already present); if the list still fits max_degree it is
//     kept, otherwise robust_prune_list runs ONCE over the whole extended list.
// Batch size 1 is exactly DiskANNIndex::insert, i.e. orc_build.
uint32_t orc_build_batch_size(uint32_t batch_size, uint64_t n_points, uint64_t inserted) {
    if (batch_size == 0) batch_size = (uint32_t)std::max<uint64_t>(1024, std::min<uint64_t>(65536, n_points / 16));
    // batches grow with the graph so that early points are not all inserted blind
    uint64_t b = std::min<uint64_t>(batch_size, std::max<uint64_t>(1, inserted / 8));
    return (uint32_t)std::min<uint64_t>(b, n_points - inserted);
}

// multi_insert's bootstrap routine (index.rs:589-747, triggered at :917-937): when the batch's back-edges reach few distinct
// targets (ceil(#targets / 8) <= batch length — always the case while the graph is smaller than eight batches) every
// pending edge list is re-pruned against its own edges plus ALL other members of the batch, with saturation
// (multi_insert_bootstrap_leaf: robust_prune_list with force_saturate), and the back-edges are aggregated again.
// Off by default: the device build grows its batches and does not run it (DESIGN.md); the reference's batch-insert
// baselines need it (tests/test_oracle_golden.py).  0: never, 1: under the reference's condition.
static int g_bootstrap = 0;
void orc_set_multi_insert_bootstrap(int mode) { g_bootstrap = mode; }
static uint64_t g_bootstrap_batches = 0, g_bootstrap_would = 0;
void orc_last_bootstrap_counts(uint64_t* ran, uint64_t* condition_held) {
    *ran = g_bootstrap_batches;
    *condition_held = g_bootstrap_would;
}

void orc_build_batched(int dtype, int metric, uint32_t dim, uint64_t n_points, uint32_t n_start,
                       const void* vectors, uint64_t row_stride, uint32_t pruned_degree,
                       uint32_t max_degree, uint32_t l_build, float alpha, uint32_t batch_size,
                       uint32_t* adj, uint32_t adj_stride) {
    orc_index idx;
    std::memset(&idx, 0, sizeof(idx));
    idx.dtype = dtype;
    idx.metric = metric;
    idx.dim = dim;
    idx.n_points = n_points;
    idx.n_start = n_start;
    idx.vectors = vectors;
    idx.row_stride = row_stride;
    idx.adj = adj;
    idx.adj_stride = adj_stride;
    const int flavour = ORC_FLAVOUR_AVX2;
    auto row = [&](uint32_t id) { return adj + (size_t)id * adj_stride; };
    std::vector<Visit> record, pool;
    std::vector<uint32_t> pruned, list;
    std::vector<std::vector<uint32_t>> edges;
    std::vector<std::pair<uint32_t, uint32_t>> back;  // (target, source)
    uint64_t inserted = 0;
    g_bootstrap_batches = g_bootstrap_would = 0;
    g_build_sets = g_build_appends = 0;  // provider writes: one set per inserted point (set_neighbors_bulk), then one
                                         // append or set per back-edge target (add_edge_and_prune)
    while (inserted < n_points) {
        // (with the bootstrap on, the reference's own drivers feed fixed chunks: no growth rule)
        const uint32_t b = g_bootstrap ? (uint32_t)std::min<uint64_t>(batch_size ? batch_size : 1, n_points - inserted)
                                       : orc_build_batch_size(batch_size, n_points, inserted);
        edges.assign(b, {});
        for (uint32_t i = 0; i < b; ++i) {
            const uint32_t id = (uint32_t)(inserted + i);
            const void* vec = (const char*)vectors + (size_t)id * row_stride;
            QueryDist qd(&idx, vec, flavour);
            Queue best((size_t)l_build + n_start);
            uint32_t cmps = 0, hops = 0;
            record.clear();
            search_internal(&idx, qd, l_build, 1, best, &cmps, &hops, &record);
            sort_pool(record, MAX_OCCLUSION);
            occlude_list(&idx, record, id, pruned_degree, alpha, flavour, edges[i]);
        }
        auto aggregate = [&]() {
            back.clear();
            for (uint32_t i = 0; i < b; ++i)
                for (uint32_t t : edges[i]) back.emplace_back(t, (uint32_t)(inserted + i));
            std::sort(back.begin(), back.end());
        };
        aggregate();
        {
            // aggregate_backedges(...).len() = distinct targets; intra_batch_candidates = None resolves to max(0, 1) = 1
            size_t targets = 0;
            for (size_t e = 0; e < back.size(); ++e)
                if (e == 0 || back[e].first != back[e - 1].first) ++targets;
            const bool cond = 1 < b && (targets + 7) / 8 <= b;
            if (cond) ++g_bootstrap_would;
            if (cond && g_bootstrap) {
                ++g_bootstrap_batches;
                std::vector<std::vector<uint32_t>> next(b);
                for (uint32_t i = 0; i < b; ++i) {
                    const uint32_t id = (uint32_t)(inserted + i);
                    // AdjacencyList::from_iter_untrusted(current.edges ++ other batch sources): duplicates dropped
                    list.assign(edges[i].begin(), edges[i].end());
                    for (uint32_t o = 0; o < b; ++o) {
                        const uint32_t other = (uint32_t)(inserted + o);
                        if (other != id && std::find(list.begin(), list.end(), other) == list.end()) list.push_back(other);
                    }
                    // robust_prune_list (index.rs:2397-2454): distances from the source, sorted pool, occlude, saturate
                    pool.clear();
                    for (uint32_t other : list)
                        if (other != id) pool.push_back(Visit{other, pair_distance(&idx, flavour, id, other)});
                    sort_pool(pool, MAX_OCCLUSION);
                    occlude_list(&idx, pool, id, pruned_degree, alpha, flavour, next[i]);
                    for (const Visit& v : pool) {  // force_saturate (index.rs:2637-2650)
                        if (next[i].size() >= pruned_degree) break;
                        if (v.id != id && std::find(next[i].begin(), next[i].end(), v.id) == next[i].end()) next[i].push_back(v.id);
                    }
                }
                edges.swap(next);
                aggregate();
            }
        }
        for (uint32_t i = 0; i < b; ++i) {
            uint32_t* r = row((uint32_t)(inserted + i));
            r[0] = (uint32_t)edges[i].size();
            for (size_t j = 0; j < edges[i].size(); ++j) r[1 + j] = edges[i][j];
            ++g_build_sets;
        }
        for (size_t e = 0; e < back.size();) {
            const uint32_t target = back[e].first;
            uint32_t* r = row(target);
            list.assign(r + 1, r + 1 + r[0]);
            size_t added = 0;
            for (; e < back.size() && back[e].first == target; ++e) {
                const uint32_t src = back[e].second;
                if (std::find(list.begin(), list.end(), src) == list.end()) {
                    list.push_back(src);
                    ++added;
                }
            }
            if (added == 0) continue;
            if (list.size() <= max_degree) {
                r[0] = (uint32_t)list.size();
                for (size_t j = 0; j < list.size(); ++j) r[1 + j] = list[j];
                ++g_build_appends;
                continue;
            }
            pool.clear();
            for (uint32_t other : list)
                if (other != target) pool.push_back(Visit{other, pair_distance(&idx, flavour, target, other)});
            sort_pool(pool, MAX_OCCLUSION);
            occlude_list(&idx, pool, target, pruned_degree, alpha, flavour, pruned);
            ++g_build_sets;
            r[0] = (uint32_t)pruned.size();
            for (size_t j = 0; j < pruned.size(); ++j) r[1 + j] = pruned[j];
        }
        inserted += b;
    }
}

void orc_set_pool_tie_mode(int mode) { g_pool_tie_mode = mode; }

void orc_last_build_counts(uint64_t* set_neighbors, uint64_t* append_neighbors) {
    *set_neighbors = g_build_sets;
    *append_neighbors = g_build_appends;
}

// ------------------------------------------------------------------ queue C API
struct orc_queue {
    Queue q;
    explicit orc_queue(uint32_t cap) : q(cap) {}
};
orc_queue* orc_queue_new(uint32_t capacity) { return new orc_queue(capacity); }
void orc_queue_free(orc_queue* q) { delete q; }
void orc_queue_insert(orc_queue* q, uint32_t id, float dist) { q->q.insert(id, dist); }
int orc_queue_has_notvisited(const orc_queue* q) { return q->q.has_notvisited() ? 1 : 0; }
int orc_queue_closest_notvisited(orc_queue* q, uint32_t* id, float* dist) {
    return q->q.closest_notvisited(id, dist) ? 1 : 0;
}
uint32_t orc_queue_size(const orc_queue* q) { return (uint32_t)q->q.size; }
void orc_queue_get(const orc_queue* q, uint32_t i, uint32_t* id, float* dist, int* visited) {
    *id = q->q.ids[i];
    *dist = q->q.dists[i];
    *visited = q->q.visited[i];
}

// ------------------------------------------------------------------ measurement helpers
void orc_bruteforce_knn(int dtype, int metric, uint32_t dim, const void* base, uint64_t n,
                        uint64_t row_stride, const void* queries, uint64_t query_stride,
                        uint32_t nq, uint32_t k, int n_threads, uint32_t* out_ids,
                        float* out_dists) {
    if (n_threads < 1) n_threads = 1;
    auto work = [&](uint32_t lo, uint32_t hi) {
        std::vector<std::pair<float, uint32_t>> heap;
        std::vector<float> widened(dim);
        for (uint32_t qi = lo; qi < hi; ++qi) {
            const void* q = (const char*)queries + (size_t)qi * query_stride;
            int dq = dtype;
            if (dtype == ORC_F16) {
                for (uint32_t j = 0; j < dim; ++j) widened[j] = orc_f16_to_f32(((const uint16_t*)q)[j]);
                q = widened.data();
                dq = ORC_F32;
            }
            heap.clear();
            for (uint64_t i = 0; i < n; ++i) {
                float d = orc_distance(ORC_FLAVOUR_AVX2, dq, dtype, metric, q,
                                       (const char*)base + i * row_stride, dim, nullptr);
                if (d != d) continue;  // NaN is never a neighbour (neighbor/queue.rs:131-134)
                std::pair<float, uint32_t> e(d, (uint32_t)i);
                if (heap.size() < k) {
                    heap.push_back(e);
                    std::push_heap(heap.begin(), heap.end());
                } else if (e < heap.front()) {
                    std::pop_heap(heap.begin(), heap.end());
                    heap.back() = e;
                    std::push_heap(heap.begin(), heap.end());
                }
            }
            std::sort_heap(heap.begin(), heap.end());
            for (uint32_t j = 0; j < k; ++j) {
                out_ids[(size_t)qi * k + j] = j < heap.size() ? heap[j].second : 0xFFFFFFFFu;
                out_dists[(size_t)qi * k + j] =
                    j < heap.size() ? heap[j].first : std::numeric_limits<float>::infinity();
            }
        }
    };
    std::vector<std::thread> ts;
    uint32_t per = (nq + n_threads - 1) / n_threads;
    for (int t = 0; t < n_threads; ++t) {
        uint32_t lo = std::min<uint32_t>(nq, t * per), hi = std::min<uint32_t>(nq, lo + per);
        if (lo < hi) ts.emplace_back(work, lo, hi);
    }
    for (auto& t : ts) t.join();
}

// benchmark-core/src/recall.rs:146-236 (fixed-size ground truth, no distance ties):
// integer hit counts over all queries divided once by nq * k.
double orc_recall(const uint32_t* gt, uint32_t gt_stride, const uint32_t* res,
                  uint32_t res_stride, const uint32_t* res_counts, uint32_t nq, uint32_t k,
                  uint32_t n) {
    uint64_t hits = 0;
    for (uint32_t q = 0; q < nq; ++q) {
        const uint32_t* g = gt + (size_t)q * gt_stride;
        const uint32_t* r = res + (size_t)q * res_stride;
        uint32_t rn = res_counts ? std::min(res_counts[q], n) : n;
        for (uint32_t i = 0; i < k; ++i)
            for (uint32_t j = 0; j < rn; ++j)
                if (g[i] == r[j]) {
                    ++hits;
                    break;
                }
    }
    return nq ? (double)hits / ((double)nq * (double)k) : 0.0;
}

int orc_hardware_threads(void) {
    unsigned n = std::thread::hardware_concurrency();
    return n ? (int)n : 1;
}

}  // extern "C"
