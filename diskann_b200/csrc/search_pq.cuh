// search_pq.cuh — parameter block shared by the quantized-traversal kernels (search_kernel_pq.cu: per-warp table in
// global memory, DirectCosine, the SQ and MinMax stores; search_kernel_pqs.cu: pivots resident in shared memory), and
// the query staging of the two packed-code stores.
#pragma once

#include "dab_common.cuh"

namespace dab {

constexpr int kPqWarps = 4;

struct SearchParamsPq {
    const uint32_t* adj;
    uint32_t adj_stride;
    uint64_t n_points;
    uint32_t n_start;
    uint32_t dim;
    uint32_t max_degree;
    int dtype;
    const void* queries;
    const uint32_t* query_list;
    uint32_t n_work;
    uint32_t k, cap, beam;
    const float* pivots;
    const uint32_t* offsets;
    const uint8_t* codes;
    uint32_t n_chunks, n_centers;
    int ip_table;  // 1: TableIP (entries -dot), 0: TableL2
    int direct_cosine;  // 1: Metric::Cosine -> QueryComputer::DirectCosine (no table): resumable cosine over the gathered pivot chunks
    float* luts;   // [warps][n_chunks * n_centers]
    uint32_t* out_ids;
    float* out_dists;
    uint32_t* out_counts;
    uint32_t* out_cmps;
    uint32_t* out_hops;
    uint32_t* tables;
    uint32_t n_buckets;
    uint32_t* counters;
    uint32_t* overflow_list;
    // optional: the whole candidate list (best.iter()) for the rerank stage
    uint32_t* list_ids;     // [nq][list_cap]
    uint32_t* list_counts;  // [nq]
    uint32_t list_cap;
    uint32_t warp_smem, off_q, off_qd, off_qi, off_cid, off_cd, off_beam, off_qc, off_nrow;
    // search_kernel_pqs: the pivot table of the CTA in shared memory
    uint32_t piv_stride;  // floats between pivot rows (odd multiple of 4: rows of different centres start in different 16-byte bank groups)
    uint32_t piv_bytes;   // n_centers * piv_stride * 4, the per-warp slices follow
    // MODE 1 (SQ) and MODE 2 (MinMax): the store's rows and the batch's queries, staged into the same layout.  The order of
    // these fields steers ptxas's register allocation of search_kernel_pq MODE 1 / 2: check -res-usage when moving them.
    const float* row_meta;  // SQ: [n_total] compensations; MinMax: [n_total][4] {b, n, a, norm_squared}
    float sq_scale_squared, sq_shift_square_norm;  // MODE 1: the quantizer's constants
    uint32_t code_dim;           // codes per row
    const uint8_t* row_codes;    // [n_total][code_stride], dense N-bit codes, zero padded to 16 B
    const uint8_t* query_codes;  // [nq][code_stride]
    const float4* query_meta;    // [nq] SQ: {compensation, -, -, -}; MinMax: {b, n, a, norm_squared}
    uint32_t code_stride;
    int code_nbits, code_metric;
};

// search_kernel_pq.cu
using PqKernel = void (*)(const SearchParamsPq);
// search_kernel_pq's instantiation for lists of `cap` entries over `store`; `keep_starts`: the one whose results keep
// start points (search_kernel_pq_starts)
PqKernel pq_kernel(uint32_t cap, QuantStore store, bool keep_starts = false);
// A quantized call's rerank can run: the full-precision vectors are uploaded (reported under `api`) and the rerank of
// lists of list_cap entries fits a CTA of this index's schema
int check_rerank(const dab_index* idx, const char* api, uint32_t list_cap);
// Reranks each query's list (d_list [nq][list_cap], d_list_n [nq]) by full-precision distance, the start points and the ids
// `deleted` marks (may be NULL) dropped: the first k into d_ids / d_dists [nq][k] and d_counts, queued on `stream`
int launch_rerank(const dab_index* idx, cudaStream_t stream, const void* d_queries, uint32_t nq, uint32_t k, uint32_t list_cap,
                  const uint32_t* d_list, const uint32_t* d_list_n, uint32_t* d_ids, float* d_dists, uint32_t* d_counts,
                  const uint32_t* deleted);

// search_kernel_pqs.cu — the shape of one launch of the shared-memory-pivot kernel
struct PqsPlan {
    int warps;         // warps (= queries in flight) per CTA, one CTA per SM
    int grid;
    size_t smem;       // dynamic shared memory per CTA
    uint32_t piv_stride, piv_bytes;
    int chunk_len;     // 4 / 8: every chunk has this length (float4 loads, folded arithmetic); 0: generic
};
// false: this index / call does not fit the kernel (pivot table too large for shared memory, > 32 chunks, ...)
bool pqs_plan(const dab_index* idx, uint32_t warp_smem, uint32_t nq, PqsPlan* out);
int pqs_launch(const SearchParamsPq& p, const PqsPlan& plan, uint32_t cap, cudaStream_t stream);

// The query side of the packed-code traversals: the nq queries d_queries (index dtype, device memory) are compressed by
// the store's own quantizer on `stream` into codes [nq][stride] and one float4 per query in the store's layout, in the
// staging scratch `stage` (stage_query_buffers).  Nothing waits.
// sq_index.cu: as_f32, the InnerProduct rescale, ScalarQuantizer::compress; the compensation in .x.  A NaN packs as 0.
int sq_stage_queries(const dab_index* idx, cudaStream_t stream, Scratch& stage, const void* d_queries, uint32_t nq, const uint8_t** d_qcodes,
                     const float4** d_qmeta);
// minmax_index.cu: as_f32, the store's transform, its compressor; {b, n, a, norm_squared}.  The index of the first query
// whose transformed vector holds a NaN (~0 if none) is copied to *h_first_nan (pinned host memory) on `stream`: it is
// valid once the stream has passed this point.
int minmax_stage_queries(const dab_index* idx, cudaStream_t stream, Scratch& stage, const void* d_queries, uint32_t nq,
                         unsigned long long* h_first_nan, const uint8_t** d_qcodes, const float4** d_qmeta);
// the staging scratch each of the two needs for nq queries, reserved before anything of a batch is queued
size_t sq_stage_bytes(const dab_index* idx, uint32_t nq);
size_t minmax_stage_bytes(const dab_index* idx, uint32_t nq);


}  // namespace dab
