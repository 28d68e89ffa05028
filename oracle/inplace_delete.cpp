// inplace_delete.cpp — CPU restatement of DiskANNIndex::inplace_delete, multi_inplace_delete and drop_deleted_neighbors:
// what dab_inplace_delete and dab_drop_deleted_neighbors compute (test infrastructure only).
//
// Written from diskann/src/graph/index.rs:
//   * the candidate routines (:1139-1336): OneHop, TwoHopAndOneHop, VisitedAndTopK.  VisitedAndTopK's search is
//     search_internal (:1933-2000) with the member's own row as the query (the f16 row widened first, layers/full.rs),
//     beam 1 and a best list of l_value + #start (scratch.rs:195-208); RemoveDeletedIdsAndCopy then drops deleted ids from
//     the whole list, start points kept (inmem/full_precision.rs:596-630), and the first l_value are taken;
//   * inplace_delete_inner (:1585-1749): edges[c] for each in-neighbour, then the appends for each live neighbour;
//   * inplace_delete (:1527-1581) and multi_inplace_delete (:1338-1520), with add_edge_and_prune (:2264-2341) and
//     robust_prune_list (:2397-2454);
//   * drop_deleted_neighbors (:1756-1816).
// Where the reference leaves an order open, the order is the one dab_inplace_delete documents: every member of a chunk
// is marked deleted before any work list is read, and exact distance ties (and the cut at num_to_replace) go by
// position in the replace candidates.  An id >= n_points + n_start in a list counts as deleted with no neighbours; list
// lengths above max_degree are read as max_degree; such an id kept in a list that add_edge_and_prune prunes is left out
// of the prune pool.
// The arithmetic is liboracle's: orc_distance (Distance<T,T>), its NeighborPriorityQueue (orc_queue_*) and its
// robust_prune (orc_robust_prune).
//
// Built on its own into liboracle_inplace_delete.so (oracle/inplace_delete.mk), linked against liboracle.so.
// C ABI (bound by tests/inplace_delete_oracle.py):
//   void orc_inplace_delete(int dtype, int metric, uint32_t dim, uint64_t n_points, uint32_t n_start, const void* vectors,
//                           uint64_t row_stride, uint32_t max_degree, uint32_t* adj, uint32_t adj_stride, uint32_t* deleted,
//                           const uint32_t* ids, uint64_t n, int method, uint32_t num_to_replace, uint32_t k_value,
//                           uint32_t l_value, uint32_t pruned_degree, float alpha, uint32_t batch_size, int single);
//     adj ((n_points + n_start) rows of adj_stride words, [len, ids...]) and the deletion bitmap `deleted` ((n_total + 31)
//     / 32 words) are read and written.  single = 0: multi_inplace_delete over chunks of batch_size (0: all n); single =
//     1: inplace_delete called id by id (batch_size ignored).
//   uint64_t orc_drop_deleted_neighbors(uint64_t n_points, uint32_t n_start, uint32_t max_degree, uint32_t* adj,
//                                       uint32_t adj_stride, const uint32_t* deleted, uint32_t pruned_degree,
//                                       int only_orphans);  returns the lists written
#include "oracle.h"

#include <algorithm>
#include <cstring>
#include <map>
#include <unordered_set>
#include <utility>
#include <vector>

namespace {

constexpr size_t kMaxOcclusion = 750;  // graph/config/defaults.rs:13
constexpr int kFlavour = ORC_FLAVOUR_AVX2;
enum { VISITED_AND_TOPK = 0, TWO_HOP_AND_ONE_HOP = 1, ONE_HOP = 2 };

struct Visit {
    uint32_t id;
    float dist;
};

struct Graph {
    orc_index idx;
    uint32_t max_degree;
    uint32_t* adj;
    uint32_t* deleted;
    uint64_t total() const { return idx.n_points + idx.n_start; }
    std::vector<uint32_t> list(uint32_t id) const {  // get_neighbors
        const uint32_t* r = adj + (size_t)id * idx.adj_stride;
        return std::vector<uint32_t>(r + 1, r + 1 + std::min(r[0], max_degree));
    }
    void set(uint32_t id, const std::vector<uint32_t>& l) {  // set_neighbors
        uint32_t* r = adj + (size_t)id * idx.adj_stride;
        r[0] = (uint32_t)l.size();
        std::copy(l.begin(), l.end(), r + 1);
    }
    // deleted, or a status lookup that fails
    bool dead(uint32_t id) const { return id >= total() || (deleted[id >> 5] >> (id & 31) & 1u); }
    void mark(uint32_t id) { deleted[id >> 5] |= 1u << (id & 31); }
    const char* row(uint32_t id) const { return (const char*)idx.vectors + (size_t)id * idx.row_stride; }
    float distance(uint32_t a, uint32_t b) const {
        return orc_distance(kFlavour, idx.dtype, idx.dtype, idx.metric, row(a), row(b), idx.dim, nullptr);
    }
    std::vector<uint32_t> live_neighbors(uint32_t id) const {
        std::vector<uint32_t> out;
        for (uint32_t v : list(id))
            if (!dead(v)) out.push_back(v);
        return out;
    }
    bool holds(uint32_t c, uint32_t id) const {
        const std::vector<uint32_t> l = list(c);
        return std::find(l.begin(), l.end(), id) != l.end();
    }
};

// search_internal from row `id`, beam 1: the whole best list, start points included
std::vector<uint32_t> search_list(const Graph& g, uint32_t id, uint32_t l_value) {
    const orc_index& idx = g.idx;
    const void* q = g.row(id);
    int dq = idx.dtype;
    std::vector<float> widened;
    if (idx.dtype == ORC_F16) {  // layers/full.rs:421-423
        widened.resize(idx.dim);
        for (uint32_t k = 0; k < idx.dim; ++k) widened[k] = orc_f16_to_f32(((const uint16_t*)q)[k]);
        q = widened.data();
        dq = ORC_F32;
    }
    auto dist = [&](uint32_t v) { return orc_distance(kFlavour, dq, idx.dtype, idx.metric, q, g.row(v), idx.dim, nullptr); };
    orc_queue* best = orc_queue_new(l_value + idx.n_start);
    std::unordered_set<uint32_t> visited;
    for (uint32_t s = 0; s < idx.n_start; ++s) {
        const uint32_t sid = (uint32_t)(idx.n_points + s);
        visited.insert(sid);
        orc_queue_insert(best, sid, dist(sid));
    }
    std::vector<Visit> found;
    uint32_t node;
    float d;
    while (orc_queue_closest_notvisited(best, &node, &d)) {
        found.clear();
        for (uint32_t v : g.list(node)) {
            if (!visited.insert(v).second) continue;
            if (v >= g.total()) continue;
            found.push_back(Visit{v, 0.0f});
        }
        for (Visit& f : found) f.dist = dist(f.id);
        for (const Visit& f : found) orc_queue_insert(best, f.id, f.dist);
    }
    std::vector<uint32_t> out;
    for (uint32_t i = 0; i < orc_queue_size(best); ++i) {
        uint32_t v;
        float dv;
        int vis;
        orc_queue_get(best, i, &v, &dv, &vis);
        out.push_back(v);
    }
    orc_queue_free(best);
    return out;
}

// the num_to_replace candidates nearest to x, x excluded: (distance, position) order
std::vector<uint32_t> nearest(const Graph& g, uint32_t x, const std::vector<uint32_t>& rc, uint32_t num_to_replace) {
    std::vector<std::pair<Visit, size_t>> pool;
    for (size_t i = 0; i < rc.size(); ++i)
        if (rc[i] != x) pool.push_back({Visit{rc[i], g.distance(x, rc[i])}, i});
    std::stable_sort(pool.begin(), pool.end(), [](const auto& a, const auto& b) { return a.first.dist < b.first.dist; });
    std::vector<uint32_t> out;
    for (size_t i = 0; i < pool.size() && i < num_to_replace; ++i) out.push_back(pool[i].first.id);
    return out;
}

// inplace_delete_inner after the delete: the member's edges, in-neighbour entries first.  A std::map keyed by source
// stands for the HashMap; the order of its keys does not matter, each key's vector does.
std::map<uint32_t, std::vector<uint32_t>> edges_of(const Graph& g, uint32_t id, int method, uint32_t num_to_replace, uint32_t k_value,
                                                   uint32_t l_value) {
    const std::vector<uint32_t> one_hop = g.live_neighbors(id);
    std::vector<uint32_t> rc, in;
    if (method == VISITED_AND_TOPK) {
        std::vector<uint32_t> undeleted;
        for (uint32_t v : search_list(g, id, l_value))
            if (!(v < g.idx.n_points && g.dead(v)) && undeleted.size() < l_value) undeleted.push_back(v);
        for (uint32_t c : undeleted)
            if (g.holds(c, id)) in.push_back(c);
        rc.assign(undeleted.begin(), undeleted.begin() + std::min<size_t>(undeleted.size(), k_value));
    } else if (method == TWO_HOP_AND_ONE_HOP) {
        rc = one_hop;
        std::unordered_set<uint32_t> two_hop;
        for (uint32_t a : one_hop) {
            two_hop.insert(a);
            for (uint32_t b : g.list(a)) two_hop.insert(b);
        }
        for (uint32_t c : two_hop)
            if (!g.dead(c) && g.holds(c, id)) in.push_back(c);
    } else {
        rc = one_hop;
        for (uint32_t c : one_hop)
            if (g.holds(c, id)) in.push_back(c);
    }
    std::map<uint32_t, std::vector<uint32_t>> edges;
    for (uint32_t c : in) edges[c] = nearest(g, c, rc, num_to_replace);
    for (uint32_t a : one_hop)
        for (uint32_t r : nearest(g, a, rc, num_to_replace)) edges[r].push_back(a);
    return edges;
}

// add_edge_and_prune(targets, source, to_remove)
void add_edge_and_prune(Graph& g, const std::vector<uint32_t>& targets, uint32_t source, const std::unordered_set<uint32_t>& to_remove,
                        uint32_t pruned_degree, float alpha) {
    std::vector<uint32_t> list;
    bool did_remove = false;
    for (uint32_t v : g.list(source)) {
        if (to_remove.count(v))
            did_remove = true;
        else
            list.push_back(v);
    }
    size_t added = 0;
    for (uint32_t t : targets)
        if (std::find(list.begin(), list.end(), t) == list.end()) {
            list.push_back(t);
            ++added;
        }
    if (added == 0 && !did_remove) return;
    if (list.size() <= g.max_degree) {
        g.set(source, list);
        return;
    }
    // robust_prune_list: Distance<T,T>(source, id) for the list without source, sorted (stable), cut to 750, occlude_list
    // robust_prune_list's fill finds no row for an id >= n_total: it is left out of the pool
    std::vector<Visit> pool;
    for (uint32_t v : list)
        if (v != source && v < g.total()) pool.push_back(Visit{v, g.distance(source, v)});
    std::stable_sort(pool.begin(), pool.end(), [](const Visit& a, const Visit& b) { return a.dist < b.dist; });
    if (pool.size() > kMaxOcclusion) pool.resize(kMaxOcclusion);
    std::vector<uint32_t> ids(pool.size()), pos(pool.size());
    std::vector<float> dists(pool.size());
    std::vector<uint8_t> excl(pool.size(), 0);
    for (size_t i = 0; i < pool.size(); ++i) ids[i] = pool[i].id, dists[i] = pool[i].dist;
    const uint32_t found = pool.empty() ? 0
                                        : orc_robust_prune(&g.idx, ids.data(), dists.data(), excl.data(), (uint32_t)pool.size(), pruned_degree,
                                                           alpha, kFlavour, pos.data(), nullptr);
    std::vector<uint32_t> out;
    for (uint32_t f = 0; f < found; ++f) out.push_back(ids[pos[f]]);
    g.set(source, out);
}

void multi_inplace_delete(Graph& g, const uint32_t* chunk, uint32_t b, int method, uint32_t num_to_replace, uint32_t k_value,
                          uint32_t l_value, uint32_t pruned_degree, float alpha) {
    std::unordered_set<uint32_t> to_remove(chunk, chunk + b);
    for (uint32_t i = 0; i < b; ++i) g.mark(chunk[i]);  // every member deleted before any list is read
    std::vector<std::map<uint32_t, std::vector<uint32_t>>> maps;
    for (uint32_t i = 0; i < b; ++i) maps.push_back(edges_of(g, chunk[i], method, num_to_replace, k_value, l_value));
    std::map<uint32_t, std::vector<uint32_t>> sources;  // source -> targets concatenated in chunk order
    for (const auto& m : maps)
        for (const auto& [src, t] : m) {
            std::vector<uint32_t>& all = sources[src];
            all.insert(all.end(), t.begin(), t.end());
        }
    for (const auto& [src, t] : sources) add_edge_and_prune(g, t, src, to_remove, pruned_degree, alpha);
    for (uint32_t i = 0; i < b; ++i) g.set(chunk[i], {});
}

void inplace_delete(Graph& g, uint32_t id, int method, uint32_t num_to_replace, uint32_t k_value, uint32_t l_value, uint32_t pruned_degree,
                    float alpha) {
    g.mark(id);
    const std::unordered_set<uint32_t> to_remove{id};
    for (const auto& [src, t] : edges_of(g, id, method, num_to_replace, k_value, l_value))
        add_edge_and_prune(g, t, src, to_remove, pruned_degree, alpha);
    g.set(id, {});
}

Graph make_graph(int dtype, int metric, uint32_t dim, uint64_t n_points, uint32_t n_start, const void* vectors, uint64_t row_stride,
                 uint32_t max_degree, uint32_t* adj, uint32_t adj_stride, uint32_t* deleted) {
    Graph g;
    std::memset(&g.idx, 0, sizeof(g.idx));
    g.idx.dtype = dtype;
    g.idx.metric = metric;
    g.idx.dim = dim;
    g.idx.n_points = n_points;
    g.idx.n_start = n_start;
    g.idx.vectors = vectors;
    g.idx.row_stride = row_stride;
    g.idx.adj = adj;
    g.idx.adj_stride = adj_stride;
    g.max_degree = max_degree;
    g.adj = adj;
    g.deleted = deleted;
    return g;
}

}  // namespace

extern "C" {

void orc_inplace_delete(int dtype, int metric, uint32_t dim, uint64_t n_points, uint32_t n_start, const void* vectors, uint64_t row_stride,
                        uint32_t max_degree, uint32_t* adj, uint32_t adj_stride, uint32_t* deleted, const uint32_t* ids, uint64_t n, int method,
                        uint32_t num_to_replace, uint32_t k_value, uint32_t l_value, uint32_t pruned_degree, float alpha, uint32_t batch_size,
                        int single) {
    Graph g = make_graph(dtype, metric, dim, n_points, n_start, vectors, row_stride, max_degree, adj, adj_stride, deleted);
    if (single) {
        for (uint64_t i = 0; i < n; ++i) inplace_delete(g, ids[i], method, num_to_replace, k_value, l_value, pruned_degree, alpha);
        return;
    }
    const uint64_t cap = batch_size ? batch_size : std::max<uint64_t>(n, 1);
    for (uint64_t first = 0; first < n; first += cap)
        multi_inplace_delete(g, ids + first, (uint32_t)std::min(cap, n - first), method, num_to_replace, k_value, l_value, pruned_degree, alpha);
}

uint64_t orc_drop_deleted_neighbors(uint64_t n_points, uint32_t n_start, uint32_t max_degree, uint32_t* adj, uint32_t adj_stride,
                                    const uint32_t* deleted, uint32_t pruned_degree, int only_orphans) {
    Graph g = make_graph(ORC_F32, 0, 0, n_points, n_start, nullptr, 0, max_degree, adj, adj_stride, const_cast<uint32_t*>(deleted));
    uint64_t rewritten = 0;
    for (uint64_t v = 0; v < g.total(); ++v) {
        if (g.dead((uint32_t)v)) continue;
        std::vector<uint32_t> pool, dead_nbrs;
        for (uint32_t u : g.list((uint32_t)v)) (g.dead(u) ? dead_nbrs : pool).push_back(u);
        if (only_orphans)
            for (uint32_t u : dead_nbrs)
                if (u < g.total() && !g.list(u).empty()) pool.push_back(u);
        if (dead_nbrs.empty() && pool.size() <= pruned_degree) continue;
        g.set((uint32_t)v, pool);
        ++rewritten;
    }
    return rewritten;
}

}  // extern "C"
