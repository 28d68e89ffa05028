// minmax_search.cpp — CPU restatement of KNN::search through the MinMax store of an index (test infrastructure only).
//
// MinMaxElement<NBITS> as the index's VectorRepr (diskann-providers/src/common/minmax_repr.rs:167-336): every search
// distance is MinMax{Cosine, IP, L2Squared, CosineNormalized} between the query, compressed by the store's quantizer
// into a row like the stored ones (query: &[MinMaxElement<N>]), and the stored row (orc_minmax_distance).  The loop is
// search_internal (diskann/src/graph/index.rs:1933-2000) over liboracle's NeighborPriorityQueue (orc_queue_*); the
// post-processing is the quant-only copy of the first k non-start entries or Pipeline<FilterStartPoints, Rerank>
// (full_precision.rs:356-399) with the full-precision query and rows, as in oracle/graph.cpp.
//
// Built on its own into liboracle_minmax_search.so (oracle/minmax_search.mk), linked against liboracle.so.
// C ABI (declared here, bound by tests/test_minmax_search.py):
//   void orc_search_batch_minmax(const orc_index* idx, const void* queries, uint64_t query_stride, const uint8_t* mm_rows,
//                                int mm_nbits, const uint8_t* mm_queries, uint32_t nq, uint32_t k, uint32_t l_search,
//                                uint32_t beam_width, int rerank, int flavour, uint32_t* out_ids, float* out_dists,
//                                uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops);
//   mm_rows: (n_points + n_start) canonical-front Data<NBITS> rows, mm_queries: nq rows of the same width; the row size
//   follows from the dim word of the first query row.
#include "oracle.h"

#include <algorithm>
#include <cstring>
#include <limits>
#include <unordered_set>
#include <vector>

namespace {

struct Visit {
    uint32_t id;
    float dist;
};

uint32_t search_one(const orc_index* idx, const void* query, const uint8_t* mm_rows, int nbits, size_t row_bytes, const uint8_t* mm_query,
                    uint32_t k, uint32_t l_search, uint32_t beam_width, bool rerank, int flavour, uint32_t* out_ids, float* out_dists,
                    uint32_t* out_cmps, uint32_t* out_hops) {
    auto dist = [&](uint32_t id) { return orc_minmax_distance(idx->metric, nbits, nbits, mm_query, mm_rows + (size_t)id * row_bytes); };
    // scratch.rs:195-208: queue capacity = L + number of start points
    orc_queue* best = orc_queue_new(l_search + idx->n_start);
    std::unordered_set<uint32_t> visited;
    uint32_t cmps = 0, hops = 0;
    const uint64_t total = idx->n_points + idx->n_start;
    // start_point_distances (diskann-inmem/src/provider.rs:406-433)
    for (uint32_t s = 0; s < idx->n_start; ++s) {
        const uint32_t id = (uint32_t)(idx->n_points + s);
        visited.insert(id);
        orc_queue_insert(best, id, dist(id));
        ++cmps;
    }
    if (beam_width == 0) beam_width = 1;
    std::vector<uint32_t> beam, list;
    while (orc_queue_has_notvisited(best)) {
        beam.clear();
        uint32_t id;
        float d;
        while (beam.size() < beam_width && orc_queue_closest_notvisited(best, &id, &d)) beam.push_back(id);
        // expand_beam (provider.rs:436-479): unvisited, in-bounds neighbours of the beam in adjacency order, then their
        // distances in that order
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
        std::vector<Visit> neighbors;
        for (uint32_t n : list) neighbors.push_back(Visit{n, dist(n)});
        for (const Visit& v : neighbors) orc_queue_insert(best, v.id, v.dist);
        cmps += (uint32_t)neighbors.size();
        hops += (uint32_t)beam.size();
    }
    const uint32_t size = std::min(orc_queue_size(best), l_search + idx->n_start);
    std::vector<Visit> cand;
    for (uint32_t i = 0; i < size; ++i) {
        uint32_t id;
        float d;
        int v;
        orc_queue_get(best, i, &id, &d, &v);
        if (id >= idx->n_points) continue;  // FilterStartPoints / no external id
        if (rerank) d = orc_distance(flavour, idx->dtype, idx->dtype, idx->metric, query,
                                     (const char*)idx->vectors + (size_t)id * idx->row_stride, idx->dim, nullptr);
        cand.push_back(Visit{id, d});
    }
    orc_queue_free(best);
    // Rerank sorts with sort_unstable_by (ties unspecified in the reference; here they keep their traversal order)
    if (rerank) std::stable_sort(cand.begin(), cand.end(), [](const Visit& a, const Visit& b) { return a.dist < b.dist; });
    const uint32_t count = (uint32_t)std::min<size_t>(k, cand.size());
    for (uint32_t i = 0; i < k; ++i) {
        out_ids[i] = i < count ? cand[i].id : 0xFFFFFFFFu;
        out_dists[i] = i < count ? cand[i].dist : std::numeric_limits<float>::infinity();
    }
    *out_cmps = cmps;
    *out_hops = hops;
    return count;
}

}  // namespace

extern "C" {

void orc_search_batch_minmax(const orc_index* idx, const void* queries, uint64_t query_stride, const uint8_t* mm_rows, int mm_nbits,
                             const uint8_t* mm_queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width, int rerank,
                             int flavour, uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops) {
    if (nq == 0) return;
    uint32_t dim;
    memcpy(&dim, mm_queries, 4);
    const size_t row_bytes = orc_minmax_row_bytes(dim, mm_nbits);
    for (uint32_t q = 0; q < nq; ++q) {
        uint32_t c = 0, h = 0;
        out_counts[q] = search_one(idx, (const char*)queries + (size_t)q * query_stride, mm_rows, mm_nbits, row_bytes,
                                   mm_queries + (size_t)q * row_bytes, k, l_search, beam_width, rerank != 0, flavour,
                                   out_ids + (size_t)q * k, out_dists + (size_t)q * k, &c, &h);
        out_cmps[q] = c;
        out_hops[q] = h;
    }
}

}  // extern "C"
