// search_diverse.cuh — parameter block and host entry points of the diversity-aware traversal (search_diverse.cu), run
// as one kind of the search job (SlotJob, search_kernel.cu).
#pragma once

#include "dab_common.cuh"
#include "search_host.cuh"
#include "search_source.cuh"

namespace dab {

constexpr int kDivWarps = 4;
// the longest list a diverse search keeps (its L): the list, its attributes and the candidates of a hop live in shared
// memory
constexpr uint32_t kDiverseMaxL = 1024;

struct SearchParamsDiverse {
    const uint32_t* adj;
    uint32_t adj_stride;
    uint64_t n_points;
    uint32_t n_start;
    uint32_t dim;
    uint32_t max_degree;
    const uint8_t* vectors;
    size_t row_stride;
    const void* queries;
    const uint32_t* query_list;
    uint32_t n_work;
    uint32_t k, cap, beam;  // cap: the list's L
    uint32_t* out_ids;
    float* out_dists;
    uint32_t *out_counts, *out_cmps, *out_hops;
    uint32_t* tables;
    uint32_t n_buckets;
    uint32_t* counters;
    uint32_t* overflow_list;
    // the attribute table (dab_upload_attributes): values [n_total], presence bits [(n_total + 31) / 32]
    const uint32_t* attr_values;
    const uint32_t* attr_present;
    uint32_t diverse_k;
    uint32_t local_cap;  // every local queue's capacity: diverse_k * L / k
    // the local queues of every warp the pass launches: pool_cap entries of {attribute, distance, id, insertion number},
    // four arrays of pool_cap words per warp
    uint32_t* pools;
    uint32_t pool_cap;
    uint32_t warp_smem, off_gd, off_gi, off_ga, off_cid, off_cd, off_beam;
    StoreParams store;  // the quantized traversals (diverse_kernel_quant)
    // with rerank: the post-processed list of every query (at most L ids) for launch_rerank
    uint32_t* list_ids;     // [nq][list_cap]
    uint32_t* list_counts;  // [nq]
    uint32_t list_cap;
};

// A CTA's shared memory may not pass this: kDivWarps x (the query area of query_area_bytes, 3 x L list words,
// 2 x beam_width x max_degree candidate words, the beam)
constexpr size_t kDiverseMaxSmem = 200 * 1024;
// "<api>: ... need N B shared memory per CTA" unless (L, beam_width) fit kDiverseMaxSmem on this index for a traversal
// over `store` (-1: full precision, else a QuantStore); no device work
int diverse_check_smem(const dab_index* idx, const char* api, uint32_t l_search, uint32_t beam, int store = -1);

// The kernel of this index's schema (store -1) or of `store`, and its shape in CTAs of kDivWarps warps; fills p's
// shared-memory offsets
int diverse_plan(const dab_index* idx, uint32_t l_search, uint32_t beam, int store, SearchParamsDiverse& p, WarpPlan<SearchParamsDiverse>& plan);
// Local-queue entries per warp in the first pass at L (tests may ask for fewer), and after a pass where a query's
// entries outgrew them
uint64_t diverse_pool_first(const dab_index* idx, uint32_t l_search);
uint64_t diverse_pool_grow(const dab_index* idx, uint64_t pool);

}  // namespace dab
