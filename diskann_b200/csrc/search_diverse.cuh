// search_diverse.cuh — parameter block and host entry points of the diversity-aware traversal (search_diverse.cu), run
// as one kind of the search job (SlotJob, search_kernel.cu).
#pragma once

#include "dab_common.cuh"

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
    // the quantized traversals (diverse_kernel_quant), named as in SearchParamsPq for the per-candidate code
    // (quant_device.cuh).  Fields of the full-precision kernel come first, so that its parameter offsets stay as they were.
    int dtype;
    const float* pivots;  // PQ: the table, [n_centers][dim]
    const uint32_t* offsets;
    const uint8_t* codes;  // [n_total][n_chunks]
    uint32_t n_chunks, n_centers;
    int ip_table, direct_cosine;
    float* luts;  // PQ tables (TableL2 / TableIP): n_chunks x n_centers f32 for every warp of the grid
    const uint8_t* row_codes;  // SQ / MinMax: the store's rows and the batch's staged queries
    const float* row_meta;
    uint32_t code_stride, code_dim;
    int code_nbits, code_metric;
    float sq_scale_squared, sq_shift_square_norm;
    const uint8_t* query_codes;  // [nq][code_stride]
    const float4* query_meta;    // [nq]
    // with rerank: the post-processed list of every query (at most L ids) for launch_rerank
    uint32_t* list_ids;     // [nq][list_cap]
    uint32_t* list_counts;  // [nq]
    uint32_t list_cap;
};

// A CTA's shared memory may not pass this: kDivWarps x (the query, 3 x L list words, 2 x beam_width x max_degree
// candidate words, the beam).  The query area is the query itself over full-precision rows (i8 / u8: its bytes rounded
// up to 16; floats: dim f32), the f32 query for PQ, and the query's code row plus 16 bytes of compensations for SQ and
// MinMax.
constexpr size_t kDiverseMaxSmem = 200 * 1024;
// "<api>: ... need N B shared memory per CTA" unless (L, beam_width) fit kDiverseMaxSmem on this index for a traversal
// over `store` (-1: full precision, else a QuantStore); no device work
int diverse_check_smem(const dab_index* idx, const char* api, uint32_t l_search, uint32_t beam, int store = -1);

// The kernel of this index's schema and its shape: `grid` CTAs of kDivWarps warps are resident, each with `smem_block`
// bytes of shared memory.  Fills p's shared-memory offsets.
struct DiversePlan {
    void (*kern)(const SearchParamsDiverse) = nullptr;
    int grid = 0;
    size_t smem_block = 0;
};
int diverse_plan(const dab_index* idx, uint32_t l_search, uint32_t beam, int store, SearchParamsDiverse& p, DiversePlan& plan);
// One pass over p.n_work queries, queued on `stream`
int diverse_launch(const SearchParamsDiverse& p, const DiversePlan& plan, cudaStream_t stream);
// Local-queue entries per warp in the first pass at L (tests may ask for fewer), and after a pass where a query's
// entries outgrew them
uint64_t diverse_pool_first(const dab_index* idx, uint32_t l_search);
uint64_t diverse_pool_grow(const dab_index* idx, uint64_t pool);

}  // namespace dab
