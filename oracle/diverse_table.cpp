// diverse_table.cpp — the reference's Diverse::search over any traversal distance (test infrastructure only).
//
// Diverse::search (diskann/src/graph/search/diverse_search.rs:189-234) is generic over the search strategy: it runs
// search_internal (diskann/src/graph/index.rs:1933-2000) with the strategy's accessor and hands best.iter().take(L) to
// the strategy's post-processor.  Here the accessor's distances come from a table the caller fills (a quantized
// store's distances to every id), and the post-processor is either the default one (start points and deleted ids
// dropped, the first k kept) or, for the quantized in-memory strategies, Pipeline<FilterStartPoints, Rerank>
// (diskann-providers/.../inmem/product.rs:391-400, full_precision.rs:356-399).  The DiverseNeighborQueue is the one of
// liboracle_diverse_search.so (oracle/diverse_search.cpp), driven through its C ABI, so both searches share one queue.
//
// Built on its own into liboracle_diverse_table.so (oracle/diverse_table.mk).  C ABI (bound by tests/diverse_table_oracle.py):
//   void orc_search_batch_diverse_table(const orc_index* idx, const float* dists, const void* queries, uint64_t query_stride,
//                                       uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width, uint32_t diverse_k,
//                                       const uint32_t* attr_values, const uint8_t* attr_present, const uint32_t* deleted,
//                                       int rerank, int flavour, uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
//                                       uint32_t* out_cmps, uint32_t* out_hops, uint64_t* failed_removals);
//     The traversal distance of query q to id i is dists[q * (n_points + n_start) + i].  attr_values / attr_present /
//     deleted / failed_removals as orc_search_batch_diverse.  rerank != 0: every entry of the post-processed list that is
//     neither a start point nor deleted gets its full-precision Distance<T, T> to the query (queries: index dtype), the
//     entries are sorted stably by it and the first k kept.  queries may be NULL without rerank.
#include "oracle.h"

#include <algorithm>
#include <limits>
#include <unordered_set>
#include <utility>
#include <vector>

// the DiverseNeighborQueue of liboracle_diverse_search.so
extern "C" {
struct orc_dq;
orc_dq* orc_diverse_queue_new(uint32_t l_value, uint32_t k_value, uint32_t diverse_k, const uint32_t* values, const uint8_t* present,
                              uint64_t n_ids);
void orc_diverse_queue_free(orc_dq*);
void orc_diverse_queue_insert(orc_dq*, uint32_t id, float dist);
void orc_diverse_queue_post_process(orc_dq*);
void orc_diverse_queue_clear(orc_dq*);
uint32_t orc_diverse_queue_size(const orc_dq*);
void orc_diverse_queue_get(const orc_dq*, uint32_t i, uint32_t* id, float* dist, int* visited);
int orc_diverse_queue_has_notvisited(const orc_dq*);
int orc_diverse_queue_closest_notvisited(orc_dq*, uint32_t* id, float* dist);
uint64_t orc_diverse_queue_failed_removals(const orc_dq*);
}

namespace {

bool is_deleted(const uint32_t* deleted, uint32_t id) { return deleted && (deleted[id >> 5] >> (id & 31) & 1u); }

// one query: search_internal over the queue (cleared first), post_process, then the post-processor; returns the count
uint32_t search_one(const orc_index* idx, orc_dq* best, const float* dist, const void* query, uint32_t k, uint32_t l_search,
                    uint32_t beam_width, const uint32_t* deleted, bool rerank, int flavour, uint32_t* out_ids, float* out_dists,
                    uint32_t* out_cmps, uint32_t* out_hops) {
    orc_diverse_queue_clear(best);
    std::unordered_set<uint32_t> visited;
    uint32_t cmps = 0, hops = 0;
    const uint64_t total = idx->n_points + idx->n_start;
    // start_point_distances (diskann-inmem/src/provider.rs:406-433)
    for (uint32_t s = 0; s < idx->n_start; ++s) {
        const uint32_t id = (uint32_t)(idx->n_points + s);
        visited.insert(id);
        orc_diverse_queue_insert(best, id, dist[id]);
        ++cmps;
    }
    if (beam_width == 0) beam_width = 1;
    std::vector<uint32_t> beam, list;
    while (orc_diverse_queue_has_notvisited(best)) {
        beam.clear();
        uint32_t id;
        float d;
        while (beam.size() < beam_width && orc_diverse_queue_closest_notvisited(best, &id, &d)) beam.push_back(id);
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
        for (uint32_t n : list) orc_diverse_queue_insert(best, n, dist[n]);
        cmps += (uint32_t)list.size();
        hops += (uint32_t)beam.size();
    }
    orc_diverse_queue_post_process(best);
    // best.iter().take(L) without start points and deleted ids
    std::vector<std::pair<float, uint32_t>> cand;
    const uint32_t n = std::min(orc_diverse_queue_size(best), l_search);
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t id;
        float d;
        int v;
        orc_diverse_queue_get(best, i, &id, &d, &v);
        if (id >= idx->n_points || is_deleted(deleted, id)) continue;
        if (rerank) {
            const char* row = (const char*)idx->vectors + (size_t)id * idx->row_stride;
            d = orc_distance(flavour, idx->dtype, idx->dtype, idx->metric, query, row, idx->dim, nullptr);
        }
        cand.emplace_back(d, id);
    }
    // Rerank: sorted by full-precision distance, ties in list order
    if (rerank) std::stable_sort(cand.begin(), cand.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
    const uint32_t count = (uint32_t)std::min<size_t>(k, cand.size());
    for (uint32_t i = 0; i < k; ++i) {
        out_ids[i] = i < count ? cand[i].second : 0xFFFFFFFFu;
        out_dists[i] = i < count ? cand[i].first : std::numeric_limits<float>::infinity();
    }
    *out_cmps = cmps;
    *out_hops = hops;
    return count;
}

}  // namespace

extern "C" {

void orc_search_batch_diverse_table(const orc_index* idx, const float* dists, const void* queries, uint64_t query_stride, uint32_t nq,
                                    uint32_t k, uint32_t l_search, uint32_t beam_width, uint32_t diverse_k, const uint32_t* attr_values,
                                    const uint8_t* attr_present, const uint32_t* deleted, int rerank, int flavour, uint32_t* out_ids,
                                    float* out_dists, uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops,
                                    uint64_t* failed_removals) {
    const uint64_t total = idx->n_points + idx->n_start;
    // Diverse::create_scratch (diverse_search.rs:149-177): a queue of L entries, one per batch, cleared per query
    orc_dq* best = orc_diverse_queue_new(l_search, k, diverse_k, attr_values, attr_present, total);
    for (uint32_t q = 0; q < nq; ++q) {
        const uint64_t failed_before = orc_diverse_queue_failed_removals(best);
        const void* query = queries ? (const char*)queries + (size_t)q * query_stride : nullptr;
        out_counts[q] = search_one(idx, best, dists + (size_t)q * total, query, k, l_search, beam_width, deleted, rerank != 0, flavour,
                                   out_ids + (size_t)q * k, out_dists + (size_t)q * k, out_cmps + q, out_hops + q);
        if (failed_removals) failed_removals[q] = orc_diverse_queue_failed_removals(best) - failed_before;
    }
    orc_diverse_queue_free(best);
}

}  // extern "C"
