// search_host.cuh — the host side every graph search shares (defined in search_kernel.cu): argument checks, the size of
// the per-warp visited tables in global memory, the parameter fields every traversal takes from the index, the query
// area, CTA cap, PQ tables, kernel choice, plan and launch of the one-query-per-warp traversals (paged, diverse,
// filtered, range), the staging of SQ / MinMax queries, the one-shot search batch and the slots of batches in flight.
#pragma once

#include "dab_common.cuh"
#include "distance_device.cuh"

#include <algorithm>
#include <type_traits>

namespace dab {

// k, L and beam of a search call; `need_vectors`: the search reads the full-precision rows (the quantized traversal
// reads only the graph and its codes)
int check_search_args(const dab_index* idx, uint32_t k, uint32_t l_search, uint32_t beam, bool need_vectors = true);

// Ids a warp's visited table holds in the first global-table pass at (L, beam, mode): the reference's estimate, or less
// where `hint` has seen the visited sets of this (or a larger) L and beam.  A default VisitedHint is no hint.
uint64_t table_slots(const dab_index* idx, const VisitedHint& hint, uint32_t l_search, uint32_t beam, QuantStore mode);
// After a global-table pass `pass` that overflowed: the table of the next one, or DAB_ERR_VISITED_OVERFLOW after six
int grow_visited_tables(const dab_index* idx, int& pass, uint64_t& slots);

// The grid of a pass of persistent one-query warps over n_work queries, where resident_ctas CTAs of warps_per_cta warps
// fit the device: every resident warp runs the same number of queries (10K queries on 3108 resident warps would
// otherwise pay for 4 full rounds with the last one 22 % full)
inline int balanced_grid(uint64_t n_work, int resident_ctas, int warps_per_cta) {
    const uint64_t max_warps = (uint64_t)resident_ctas * warps_per_cta;
    const uint64_t rounds = (n_work + max_warps - 1) / max_warps;
    const uint64_t need = (n_work + rounds - 1) / rounds;
    return (int)((need + warps_per_cta - 1) / warps_per_cta);
}

// f(std::integral_constant<int, QT>) for the merge tile QT (merge_any, search_common.cuh) of a list of `cap` entries
template <class F>
auto visit_list_tile(uint32_t cap, F&& f) {
    if (cap <= 128) return f(std::integral_constant<int, 4>{});
    if (cap <= 256) return f(std::integral_constant<int, 8>{});
    if (cap <= 512) return f(std::integral_constant<int, 16>{});
    return f(std::integral_constant<int, 32>{});
}

// A quantized traversal's store is ready: the PQ table and codes, or the SQ / MinMax rows (and the SQ store's metric,
// SQStore::distance_computer, providers inmem/scalar.rs:214-226).  `who` names the entry point in the message.
// `upload_first`: a store that was never set up is reported as "<upload call> has not been called" (the paged calls)
// instead of as missing codes or rows (the batch calls).
int check_quant_store(const dab_index* idx, QuantStore store, const char* who, bool upload_first);

// The graph fields every traversal's parameter block (SearchParamsV2, SearchParamsV3, SearchParamsPq, PagedParams) takes
// from the index
template <class P>
void set_graph_params(const dab_index* idx, P& p) {
    p.adj = idx->d_adj;
    p.adj_stride = idx->adj_stride;
    p.n_points = idx->n_points;
    p.n_start = idx->n_start;
    p.dim = idx->dim;
    p.max_degree = idx->max_degree;
}

// The 16-bit quotient tags of a visited table in shared memory (Tag16Map, search_common.cuh) cover ids < 2^K
inline uint32_t tag_id_bits(uint64_t n_total) {
    uint32_t K = 8;
    while (((uint64_t)1 << K) < n_total) ++K;
    return K;
}
// The tag map of a table of `n_buckets` buckets of 16 tags over this index's ids into p.tag_kmask / tag_shift / tag_magic;
// false (nothing set) when a tag, the id's quotient by n_buckets, needs more than 14 bits or the id and its bucket more
// than 32
template <class P>
bool set_tag_map(const dab_index* idx, uint64_t n_buckets, P& p) {
    const uint32_t K = tag_id_bits(idx->n_total());
    uint32_t sbits = 0;
    while (((uint64_t)1 << sbits) < n_buckets) ++sbits;
    if (((((uint64_t)1 << K) + 16383) >> 14) > n_buckets || K + sbits > 32) return false;
    p.tag_kmask = (uint32_t)(((uint64_t)1 << K) - 1);
    p.tag_shift = K + sbits;
    p.tag_magic = (uint32_t)((((uint64_t)1 << (K + sbits)) + n_buckets - 1) / n_buckets);
    return true;
}

// The fields a quantized traversal's parameter block (SearchParamsPq, or the StoreParams of the others) takes from the
// index and the store it reads
template <class P>
void set_store_params(const dab_index* idx, QuantStore store, P& p) {
    p.dtype = idx->dtype;
    if (store == STORE_PQ) {
        p.pivots = idx->d_pivots;
        p.offsets = idx->d_offsets;
        p.codes = idx->d_codes;
        p.n_chunks = idx->pq_chunks;
        p.n_centers = idx->pq_centers;
        p.ip_table = idx->metric == DAB_INNER_PRODUCT ? 1 : 0;  // L2 and CosineNormalized use TableL2 (dynamic.rs:80-85)
        p.direct_cosine = idx->metric == DAB_COSINE ? 1 : 0;
        return;
    }
    const CodeStore& cs = store == STORE_SQ ? idx->sq : idx->mm;
    p.row_codes = cs.d_codes;
    p.row_meta = cs.d_meta;
    p.code_stride = cs.stride;
    p.code_dim = cs.dim;
    p.code_nbits = cs.nbits;
    p.code_metric = idx->metric;  // MinMaxElement::query_distance: all four metrics (minmax_repr.rs)
    if (store == STORE_SQ) {
        p.sq_scale_squared = idx->sq_scale * idx->sq_scale;  // AsFunctor (scalar/quantizer.rs:316-335)
        p.sq_shift_square_norm = idx->sq_shift_square_norm;
    }
}

// The query area at the front of a warp's shared memory in a traversal over `store` (-1: full precision, else a
// QuantStore): the query itself over full-precision rows (i8 / u8: its bytes rounded up to 16; floats: dim f32), the f32
// query for PQ, and the query's code row plus 16 bytes of compensations for SQ and MinMax
inline size_t query_area_bytes(const dab_index* idx, int store) {
    if (store == STORE_SQ || store == STORE_MINMAX) return round_up((size_t)(store == STORE_SQ ? idx->sq : idx->mm).stride + 16, 16);
    const bool is_int = idx->dtype == DAB_I8 || idx->dtype == DAB_U8;
    return is_int && store < 0 ? round_up(round_up((size_t)idx->dim, 4), 16) : round_up((size_t)idx->dim * 4, 16);
}

// The most CTAs per SM of a traversal over `store` (-1: full precision, else a QuantStore): with a PQ table metric every
// resident warp owns a table (pq_table_bytes) that its lookups read through L2, and the cap of search_kernel_pq keeps
// them L2-resident; no cap otherwise
inline int store_ctas_cap(const dab_index* idx, int store) { return store == STORE_PQ && idx->metric != DAB_COSINE ? 6 : INT32_MAX; }

// The PQ tables of `warps` warps over `store`: n_chunks x n_centers f32 each for a PQ table metric, else 0 bytes
// (`cosine_too`: search_kernel_pq's reservation, which keeps them under DirectCosine as well)
inline size_t pq_table_bytes(const dab_index* idx, int store, uint64_t warps, bool cosine_too = false) {
    return store == STORE_PQ && (cosine_too || idx->metric != DAB_COSINE) ? (size_t)warps * idx->pq_chunks * idx->pq_centers * 4 : 0;
}

// A kind's kernel over `store` into `kern`: quant(integral_constant<int, MODE>) over a store, MODE being the store
// (STORE_PQ / SQ / MINMAX = 0 / 1 / 2), or full(S) for the index's distance schema S over full-precision rows (-1)
template <class P, class F>
int full_kernel(const dab_index* idx, F&& full, void (*&kern)(const P)) {
    return visit_schema<OPS_QUERY>(idx->dtype, idx->metric, [&](auto sc) -> int {
        kern = full(sc);
        return DAB_OK;
    });
}
template <class P, class Q, class F>
int traversal_kernel(const dab_index* idx, int store, Q&& quant, F&& full, void (*&kern)(const P)) {
    if (store < 0) return full_kernel(idx, full, kern);
    kern = store == STORE_PQ ? quant(std::integral_constant<int, STORE_PQ>{})
           : store == STORE_SQ ? quant(std::integral_constant<int, STORE_SQ>{})
                               : quant(std::integral_constant<int, STORE_MINMAX>{});
    return DAB_OK;
}

// A one-query-per-warp kernel and its shape: CTAs of `warps` warps and smem_block bytes, `grid` of them resident
template <class P>
struct WarpPlan {
    void (*kern)(const P) = nullptr;
    int warps = 0;
    int grid = 0;
    size_t smem_block = 0;
    int pass_grid(uint64_t n_work) const { return balanced_grid(n_work, grid, warps); }  // a pass over n_work queries
};

// plan.kern's shape over `store`: CTAs of `warps` warps of warp_smem bytes each, at most store_ctas_cap per SM.  Returns
// plan.grid: 0 when no CTA fits or smem_block passes max_smem, which the caller reports.
template <class P>
int plan_warps(const dab_index* idx, int store, int warps, size_t warp_smem, size_t max_smem, WarpPlan<P>& plan) {
    plan.warps = warps;
    plan.smem_block = warp_smem * warps;
    const int per_sm = plan.smem_block > max_smem ? 0 : ctas_per_sm(plan.kern, warps * 32, plan.smem_block);
    plan.grid = std::min(per_sm, store_ctas_cap(idx, store)) * idx->sm_count;
    return plan.grid;
}

// One pass of plan.kern in `grid` CTAs (plan.pass_grid, or fewer), queued on `stream`; the shared-memory attribute is set
// at every launch because it belongs to the kernel, which plans of other shapes share
template <class P>
int warp_launch(const P& p, const WarpPlan<P>& plan, int grid, cudaStream_t stream) {
    DAB_CUDA(cudaFuncSetAttribute(plan.kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan.smem_block));
    plan.kern<<<grid, plan.warps * 32, plan.smem_block, stream>>>(p);
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    return DAB_OK;
}

// Where a batch's results go: ids and dists [nq][k]; counts, cmps and hops [nq], optional
struct SearchOut {
    uint32_t* ids;
    float* dists;
    uint32_t *counts, *cmps, *hops;
};

// RemoveDeletedIdsAndCopy over whole lists (delete_kernels.cu): the traversal wrote each query's entries below `bound`
// (n_points: no start points; n_total: all), list order, into ids / dists [nq][cap] (padded with UINT32_MAX); the first
// k below `bound` that `deleted` does not mark go to `out` ([nq][k], padded UINT32_MAX / +inf; counts = how many), queued
// on `stream`.  cmps and hops are not touched.
int queue_drop_deleted(const dab_index* idx, cudaStream_t stream, const uint32_t* deleted, const uint32_t* ids, const float* dists,
                       uint32_t cap, uint32_t nq, uint32_t k, const SearchOut& out, uint64_t bound);

// SQ and MinMax: a batch's queries as the store's quantizer compressed them (search_pq.cuh), in the handle's staging
// scratch until the next call that stages
struct StagedQueries {
    const uint8_t* codes;
    const float4* meta;
};

// SQ / MinMax: the nq queries compressed into `stage` on `stream` (nothing otherwise).  MinMax: staged_first_nan reads
// the first query holding a NaN after the transform from h_counters (pinned, 24 bytes) once the stream has passed.
int stage_store_queries(const dab_index* idx, cudaStream_t stream, Scratch& stage, int store, const void* d_queries, uint32_t nq,
                        uint32_t* h_counters, StagedQueries& out);
inline unsigned long long staged_first_nan(const uint32_t* h_counters) { return *(const unsigned long long*)(h_counters + 4); }

// Searches whose queries are rows of the index (the build's insert searches, in-place deletes): they ignore deletions
// and teach the visited tables nothing.  With `ids` each records the nodes it expanded; with `keep_starts` its results
// are the list's entries with start points kept (the caller filters them).  `keep_deleted`, for queries that are not
// rows (the first phase of range search): the results keep deleted ids too, and the caller filters them.  `staged`
// (NULL: not wanted) receives an SQ or MinMax batch's compressed queries, for a caller that reads them after the search.
struct SearchRecord {
    const uint32_t* query_rows;  // [nq] row ids of the queries
    uint32_t* ids;               // [nq][cap] expanded nodes, [nq] counts (NULL: no record)
    float* dists;
    uint32_t* counts;
    uint32_t cap;
    bool keep_starts;
    bool keep_deleted;
    StagedQueries* staged;
};

// One batch on the handle's stream and scratch, device pointers only.  `store`: -1 full precision, else the QuantStore the
// traversal reads; `rerank` (quantized) reorders each list by full-precision distances.  Returns once the traversal is
// complete; a full-precision batch also has its deleted ids filtered, while a quantized batch's rerank or filter may still
// run.  `rec` (full precision): searches over rows of the index, which ignore deletions and teach the visited tables
// nothing.
int run_search(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam, const SearchOut& d,
               int store, bool rerank, const SearchRecord* rec = nullptr);

// ---- batches in flight ---------------------------------------------------------------------------------------------
// A batch of any kind (full precision, PQ, SQ, MinMax) as a resumable job (search_kernel.cu)
struct SlotJob;

// A host-buffer call's results: where the kernels write them and where the caller wants them
struct HostCopy {
    SearchOut dev, host;
    uint32_t nq, k;
};

// A slot of batches in flight: its own stream and grow-only scratch, so that nothing a batch in flight touches is
// shared with another slot or with the synchronous calls on the handle's stream.
struct SearchSlot {
    cudaStream_t stream = nullptr;
    Scratch tables, counters, queries, out, stats, h_counters;
    Scratch stage, luts;  // the quantized traversals: staged queries, per-warp LUTs
    Scratch lists;        // the rerank's candidate lists, or the whole lists a search filters deleted ids from
    SlotJob* job = nullptr;
    HostCopy host_out{};  // the pending call's result copies (host_out.host.ids null: device buffers)
};

}  // namespace dab
