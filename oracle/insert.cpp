// insert.cpp — CPU restatement of DiskANNIndex::multi_insert over ids of the caller's choosing, on a graph that already
// exists: what dab_insert links (test infrastructure only).
//
// DiskANNIndex::insert (diskann/src/graph/index.rs:226-341) and multi_insert (:815-1030) with intra_batch_candidates = None
// and the bootstrap routine not run, one chunk at a time:
//   * candidate generation (search_and_prune, index.rs:341-430): every member of the chunk is searched against the graph
//     AS IT WAS BEFORE THE CHUNK (search_internal, index.rs:1933-2000, beam 1, with a VisitedSearchRecord) and its record
//     pruned (SortedNeighbors::new, then occlude_list without saturation); nothing is written yet;
//   * set_neighbors_bulk of the new out-lists;
//   * aggregate_backedges (index.rs:123-143): target -> sources, sources sorted (index.rs:986-992);
//   * add_edge_and_prune(sorted sources, target) (index.rs:2264-2341): every new source is appended; if the list still
//     fits max_degree it is kept, otherwise robust_prune_list (index.rs:2397-2454) runs once over the whole list.
// The arithmetic is liboracle's: orc_distance (Distance<T,T>, the f16 query widened first), its NeighborPriorityQueue
// (orc_queue_*) and its robust_prune (orc_robust_prune).  This is the loop orc_build_batched runs over its id ranges,
// restated over an id list; tests/test_insert.py holds the two equal over the device build's schedule, equal to
// orc_build at chunk size 1, and to the reference's single-insert lattice baseline.
//
// Built on its own into liboracle_insert.so (oracle/insert.mk), linked against liboracle.so.
// C ABI (declared here, bound by tests/insert_oracle.py):
//   void orc_insert_batched(int dtype, int metric, uint32_t dim, uint64_t n_points, uint32_t n_start, const void* vectors,
//                           uint64_t row_stride, uint32_t pruned_degree, uint32_t max_degree, uint32_t l_build, float alpha,
//                           const uint32_t* ids, uint64_t n, uint32_t batch_size, int tie_mode, uint32_t* adj,
//                           uint32_t adj_stride, uint64_t* out_sets, uint64_t* out_appends);
//   ids: data points, cut into consecutive chunks of batch_size (0: 65536) in the given order; vectors already hold the
//   new rows; adj ((n_points + n_start) rows of adj_stride words, [len, ids...]) is read and written.  tie_mode 1 orders
//   exactly tied prune candidates the way oracle/graph.cpp's opt-in emulation of the Rust standard library does, 0 by a
//   stable sort.  out_sets / out_appends (may be NULL): the provider writes, set_neighbors and append_neighbors.
#include "oracle.h"

#include <algorithm>
#include <cstring>
#include <unordered_set>
#include <utility>
#include <vector>

namespace {

constexpr size_t kMaxOcclusion = 750;  // graph/config/defaults.rs:13
constexpr int kFlavour = ORC_FLAVOUR_AVX2;

struct Visit {
    uint32_t id;
    float dist;
};

const char* row_of(const orc_index& idx, uint32_t id) { return (const char*)idx.vectors + (size_t)id * idx.row_stride; }

float pair_distance(const orc_index& idx, uint32_t a, uint32_t b) {
    return orc_distance(kFlavour, idx.dtype, idx.dtype, idx.metric, row_of(idx, a), row_of(idx, b), idx.dim, nullptr);
}

// search_internal with beam 1 and a VisitedSearchRecord: the nodes expanded, in order, with their distances
void search_record(const orc_index& idx, const uint32_t* adj, uint32_t id, uint32_t l_build, std::vector<Visit>& record) {
    const void* q = row_of(idx, id);
    int dq = idx.dtype;
    std::vector<float> widened;
    if (idx.dtype == ORC_F16) {  // layers/full.rs:421-423
        widened.resize(idx.dim);
        for (uint32_t k = 0; k < idx.dim; ++k) widened[k] = orc_f16_to_f32(((const uint16_t*)q)[k]);
        q = widened.data();
        dq = ORC_F32;
    }
    auto dist = [&](uint32_t v) { return orc_distance(kFlavour, dq, idx.dtype, idx.metric, q, row_of(idx, v), idx.dim, nullptr); };
    const uint64_t total = idx.n_points + idx.n_start;
    orc_queue* best = orc_queue_new(l_build + idx.n_start);  // scratch.rs:195-208
    std::unordered_set<uint32_t> visited;
    for (uint32_t s = 0; s < idx.n_start; ++s) {  // start_point_distances (diskann-inmem/src/provider.rs:406-433)
        const uint32_t sid = (uint32_t)(idx.n_points + s);
        visited.insert(sid);
        orc_queue_insert(best, sid, dist(sid));
    }
    std::vector<uint32_t> list;
    std::vector<Visit> found;
    uint32_t node;
    float d;
    while (orc_queue_closest_notvisited(best, &node, &d)) {
        record.push_back(Visit{node, d});
        // expand_beam (provider.rs:436-479): unvisited, in-bounds neighbours in list order, then their distances
        list.clear();
        const uint32_t* r = adj + (size_t)node * idx.adj_stride;
        for (uint32_t j = 0; j < r[0]; ++j) {
            const uint32_t v = r[1 + j];
            if (!visited.insert(v).second) continue;
            if (v >= total) continue;
            list.push_back(v);
        }
        found.clear();
        for (uint32_t v : list) found.push_back(Visit{v, dist(v)});
        for (const Visit& f : found) orc_queue_insert(best, f.id, f.dist);
    }
    orc_queue_free(best);
}

// SortedNeighbors::new (graph/internal/sorted_neighbors.rs:26-44), as oracle/graph.cpp's sort_pool restates it
void sort_pool(std::vector<Visit>& pool, int tie_mode) {
    auto less = [](const Visit& a, const Visit& b) { return a.dist < b.dist; };
    const size_t len = pool.size();
    if (len > kMaxOcclusion || tie_mode == 0) {
        std::stable_sort(pool.begin(), pool.end(), less);
        if (len > kMaxOcclusion) pool.resize(kMaxOcclusion);
        return;
    }
    if (len < 2) return;
    size_t mx = 0;  // select_nth_unstable_by at the last position swaps the first maximum to the end
    for (size_t i = 1; i < len; ++i)
        if (less(pool[mx], pool[i])) mx = i;
    std::swap(pool[mx], pool[len - 1]);
    const size_t n = len - 1;  // the prefix: insertion sort up to 20, else ipnsort's run detection, else a stable sort
    if (n < 2) return;
    if (n <= 20) {
        for (size_t i = 1; i < n; ++i) {
            const Visit v = pool[i];
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

// occlude_list (index.rs:2565-2650) without saturation: `location` is excluded from its own pool
void occlude_list(const orc_index& idx, const std::vector<Visit>& pool, uint32_t location, uint32_t degree, float alpha,
                  std::vector<uint32_t>& out) {
    out.clear();
    if (pool.empty()) return;
    const size_t n = pool.size();
    std::vector<uint32_t> ids(n), pos(n);
    std::vector<float> dists(n);
    std::vector<uint8_t> excl(n);
    for (size_t i = 0; i < n; ++i) {
        ids[i] = pool[i].id;
        dists[i] = pool[i].dist;
        excl[i] = pool[i].id == location;
    }
    const uint32_t found = orc_robust_prune(&idx, ids.data(), dists.data(), excl.data(), (uint32_t)n, degree, alpha, kFlavour, pos.data(), nullptr);
    for (uint32_t f = 0; f < found; ++f) out.push_back(ids[pos[f]]);
}

// one multi_insert over the b ids of `chunk`
void multi_insert(const orc_index& idx, uint32_t* adj, const uint32_t* chunk, uint32_t b, uint32_t pruned_degree, uint32_t max_degree,
                  uint32_t l_build, float alpha, int tie_mode, uint64_t& sets, uint64_t& appends) {
    auto row = [&](uint32_t id) { return adj + (size_t)id * idx.adj_stride; };
    std::vector<std::vector<uint32_t>> edges(b);
    std::vector<Visit> record, pool;
    for (uint32_t i = 0; i < b; ++i) {
        record.clear();
        search_record(idx, adj, chunk[i], l_build, record);
        sort_pool(record, tie_mode);
        occlude_list(idx, record, chunk[i], pruned_degree, alpha, edges[i]);
    }
    std::vector<std::pair<uint32_t, uint32_t>> back;  // (target, source)
    for (uint32_t i = 0; i < b; ++i)
        for (uint32_t t : edges[i]) back.emplace_back(t, chunk[i]);
    std::sort(back.begin(), back.end());
    for (uint32_t i = 0; i < b; ++i) {
        uint32_t* r = row(chunk[i]);
        r[0] = (uint32_t)edges[i].size();
        for (size_t j = 0; j < edges[i].size(); ++j) r[1 + j] = edges[i][j];
        ++sets;
    }
    std::vector<uint32_t> list, pruned;
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
            ++appends;
            continue;
        }
        pool.clear();
        for (uint32_t other : list)
            if (other != target) pool.push_back(Visit{other, pair_distance(idx, target, other)});
        sort_pool(pool, tie_mode);
        occlude_list(idx, pool, target, pruned_degree, alpha, pruned);
        ++sets;
        r[0] = (uint32_t)pruned.size();
        for (size_t j = 0; j < pruned.size(); ++j) r[1 + j] = pruned[j];
    }
}

}  // namespace

extern "C" {

void orc_insert_batched(int dtype, int metric, uint32_t dim, uint64_t n_points, uint32_t n_start, const void* vectors, uint64_t row_stride,
                        uint32_t pruned_degree, uint32_t max_degree, uint32_t l_build, float alpha, const uint32_t* ids, uint64_t n,
                        uint32_t batch_size, int tie_mode, uint32_t* adj, uint32_t adj_stride, uint64_t* out_sets, uint64_t* out_appends) {
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
    if (batch_size == 0) batch_size = 65536;
    uint64_t sets = 0, appends = 0;
    for (uint64_t first = 0; first < n; first += batch_size) {
        const uint32_t b = (uint32_t)std::min<uint64_t>(batch_size, n - first);
        multi_insert(idx, adj, ids + first, b, pruned_degree, max_degree, l_build, alpha, tie_mode, sets, appends);
    }
    if (out_sets) *out_sets = sets;
    if (out_appends) *out_appends = appends;
}

}  // extern "C"
