// search_kernel_pq.cu — batched greedy search whose traversal distances come from a quantized store:
// PQ ADC lookups (MODE 0), scalar-quantized codes (MODE 1) or MinMax codes (MODE 2; see the notes below).
//
// Restates the providers' quant accessor (diskann-providers/src/model/graph/provider/async_/
// inmem/product.rs:311-340: expand_beam with `computer.evaluate_similarity(aux_vectors[i])`)
// around the same search_internal loop (diskann/src/graph/index.rs:1933-2000):
//   * QueryComputer::new (pq/distance/dynamic.rs:63-87): L2 and CosineNormalized -> TableL2,
//     InnerProduct -> TableIP (entries are -dot); the query is converted to f32 first;
//   * the warp builds its query's table once (n_chunks x n_centers f32, entries in the
//     reference's SIMD order for the chunk length, fixed_chunk_pq_table.rs:152-187) into a
//     per-warp global scratch that stays in L2;
//   * per hop every lane owns one surviving neighbour: coalesced 16 B code loads, one table
//     gather per chunk, and the sum is accumulated in chunk order from 0.0
//     (pq_dist_lookup_single, fixed_chunk_pq_table.rs:82-98) -> bit-identical ADC distances;
//   * visited set, sorted list and post-processing are the shared exact helpers; the per-candidate distances live in
//     quant_device.cuh, shared with the paged sessions (search_paged.cu).
// No tensor cores: LUT gather + byte loads, HBM traffic is n_chunks code bytes per candidate.
//
// MODE 1 and MODE 2 — the two stores of dense N-bit code rows (bits/slice.rs:261-323), 16 B aligned, compensations
// apart.  Before the launch the batch's queries are compressed by the store's own quantizer into the rows' layout
// (sq_stage_queries, minmax_stage_queries); the warp copies its query's code words to shared memory.  Per candidate,
// one lane runs the exact integer core over the packed words (bits/distances.rs:397, 979 — here vabsdiffu4 + dp4a on
// masked fields, popc for 1 bit) with 16 B code loads, then the store's f32 epilogue:
//   * MODE 1, the scalar-quantized accessor (providers inmem/scalar.rs:449-570; the query from SQStore::query_computer,
//     :227-253): sq_finish, Compensated{SquaredL2, IP, CosineNormalized} (scalar/vectors.rs:206-460).  Traffic is
//     ceil(dim * N / 8) bytes per candidate (+ 4 B compensation for InnerProduct).
//   * MODE 2, the MinMax store (minmax_index.cu; providers common/minmax_repr.rs:167-336, garnet provider.rs:1170-1358;
//     the query is &[MinMaxElement<N>] behind the store's transform): minmax_finish, the MinMax distance of the index
//     metric from the codes' inner product (vectors.rs:206-228, all four metrics).  Traffic is ceil(dim * N / 8) code
//     bytes + 16 B of compensations per candidate.
#include "dab_common.cuh"
#include "quant_device.cuh"
#include "search_common.cuh"
#include "search_host.cuh"
#include "search_pq.cuh"
#include "search_smem.cuh"

#include <algorithm>
#include <type_traits>

namespace dab {

template <int QT, int MODE>
__global__ void __launch_bounds__(kPqWarps * 32) search_kernel_pq(const SearchParamsPq p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    uint8_t* base = smem + (size_t)wib * p.warp_smem;
    float* qf = reinterpret_cast<float*>(base + p.off_q);
    float* qd = reinterpret_cast<float*>(base + p.off_qd);
    uint32_t* qi = reinterpret_cast<uint32_t*>(base + p.off_qi);
    uint32_t* cid = reinterpret_cast<uint32_t*>(base + p.off_cid);
    float* cd = reinterpret_cast<float*>(base + p.off_cd);
    uint32_t* beam_ids = reinterpret_cast<uint32_t*>(base + p.off_beam);
    uint32_t* qc = reinterpret_cast<uint32_t*>(base + p.off_qc);  // MODE 1 / 2: the query's packed codes
    float q_comp = 0.0f;

    const uint32_t warp_slot = blockIdx.x * kPqWarps + wib;
    const uint32_t nbk = p.n_buckets;
    uint32_t* table = p.tables + (size_t)warp_slot * nbk * 8;
    const uint32_t hlimit = nbk * 7;
    const uint64_t n_total = p.n_points + p.n_start;
    const uint32_t entries = p.n_chunks * p.n_centers;
    float* lut = p.luts + (size_t)warp_slot * entries;
    const int dim = (int)p.dim;

    // quantized distances of candidates cid[0..n) -> cd[]: one lane per candidate
    auto adc = [&](uint32_t n) {
        for (uint32_t c0 = 0; c0 < n; c0 += 32) {
            const uint32_t c = c0 + lane;
            if (MODE != 0) {
                if (c < n) cd[c] = packed_code_distance<MODE>(p, qc, q_comp, cid[c]);
            } else if (p.direct_cosine) {
                if (c < n) cd[c] = pq_direct_cosine(p, qf, dim, cid[c]);
            } else if (c < n) {
                cd[c] = pq_table_distance(p, lut, cid[c]);
            }
        }
        __syncwarp();
    };

    for (uint32_t qidx; next_query(p.counters, p.n_work, p.query_list, lane, qidx);) {
        // ---- query -> f32 (T: Into<f32>), table build, visited clear
        __syncwarp();
        if (MODE == 0) widen_query(p.dtype, p.queries, qidx, dim, qf, lane);
        for (uint32_t i = lane; i < nbk; i += 32) store_empty_bucket(table + (size_t)i * 8);
        __syncwarp();
        if (MODE != 0) {
            load_query_codes<MODE>(p.query_codes + (size_t)qidx * p.code_stride, p.query_meta + qidx, p.code_stride >> 2, qc, q_comp, lane);
            __syncwarp();
        }
        for (uint32_t t = lane; MODE == 0 && !p.direct_cosine && t < entries; t += 32) __stcg(lut + t, pq_table_entry(p, qf, dim, t));
        __syncwarp();

        uint32_t size = 0, cursor_lo = 0, cmps = 0, hops = 0, nvisited = 0;
        bool overflow = false;

        // ---- start points
        for (uint32_t s0 = 0; s0 < p.n_start; s0 += 32) {
            const uint32_t n = min(32u, p.n_start - s0);
            if ((uint32_t)lane < n) {
                const uint32_t id = (uint32_t)p.n_points + s0 + lane;
                cid[lane] = id;
                visit_global(table, nbk, id);
            }
            __syncwarp();
            adc(n);
            merge_any<QT>(qd, qi, p.cap, size, cursor_lo, cid, cd, 0, n, lane);
            nvisited += n;
            cmps += n;
        }

        // ---- greedy loop
        for (;;) {
            const uint32_t lim = min(p.cap, size);
            const uint32_t nb = pick_beam(qi, lim, p.beam, cursor_lo, beam_ids, lane);
            if (nb == 0) break;
            uint32_t ncand = 0;
            for (uint32_t b = 0; b < nb; ++b) {
                const uint32_t node = beam_ids[b];
                const uint32_t* row = p.adj + (size_t)node * p.adj_stride;
                const uint32_t deg = min(__ldg(row), p.max_degree);
                for (uint32_t c0 = 0; c0 < deg + 1; c0 += 32) {
                    const uint32_t j = c0 + lane;
                    const uint32_t word = j < p.adj_stride ? __ldg(row + j) : kEmptyV2;
                    const bool inserted = j >= 1 && j <= deg && visit_global(table, nbk, word);
                    push_new(inserted, inserted && word < n_total, word, cid, ncand, nvisited, lane);
                }
                if (nvisited + p.max_degree > hlimit) {
                    overflow = true;
                    break;
                }
            }
            if (overflow) break;
            __syncwarp();
            adc(ncand);
            for (uint32_t c0 = 0; c0 < ncand; c0 += 32)
                merge_any<QT>(qd, qi, p.cap, size, cursor_lo, cid, cd, c0, min(32u, ncand - c0), lane);
            cmps += ncand;
            hops += nb;
        }

        if (overflow) {
            report_overflow(p.counters, p.overflow_list, qidx, lane);
            continue;
        }
        const uint32_t n = min(p.cap, size);
        if (p.list_ids) write_list(qi, n, p.list_ids, p.list_counts, p.list_cap, qidx, lane);
        const uint32_t count = write_results(qi, qd, n, p.n_points, p.k, p.out_ids, p.out_dists, qidx, lane);
        write_stats(p.counters, nvisited, p.out_counts, p.out_cmps, p.out_hops, qidx, count, cmps, hops, lane);
    }
}

// ---- Rerank (diskann-providers/.../inmem/full_precision.rs:356-399 behind FilterStartPoints,
// product.rs:391-400): every candidate of best.iter() that is not a start point gets its
// full-precision Distance<T, T> to the query; the list is ordered by that distance (ties keep
// their traversal order: the reference's sort_unstable_by leaves them unspecified) and the
// first k are returned.  One warp per query; rows are gathered with the wide-load loops of
// search_smem.cuh (f32 x f32 has the query x row association; i8 / u8 are exact).
constexpr int kRerankWarps = 4;
struct RerankParams {
    const uint8_t* vectors;
    size_t row_stride;
    uint64_t n_points;
    uint32_t dim;
    const void* queries;  // index dtype
    uint32_t nq, k, list_cap;
    const uint32_t* list_ids;
    const uint32_t* list_counts;
    uint32_t* out_ids;
    float* out_dists;
    uint32_t* out_counts;
    const uint32_t* deleted;  // the deletion table, or NULL: its ids are dropped with the start points
    uint32_t warp_smem, off_ids, off_d;
};

// NA = 4: the wide-load loops (f32 rows, L2 / InnerProduct / CosineNormalized; integers).  NA = 2: the schemas with two
// accumulators — f16 x f16 (Strategy2x4, simd.rs:424-483: both sides widened to f32 lanes, so the f32 copy of the query
// in shared memory is the same operand) and Metric::Cosine over float rows — one team of 16 lanes per row.
template <typename TD, int KIND, int POST, int NA = 4>
__global__ void __launch_bounds__(kRerankWarps * 32) rerank_kernel(const RerankParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    constexpr bool kInt = std::is_same<TD, int8_t>::value || std::is_same<TD, uint8_t>::value;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    uint8_t* base = smem + (size_t)wib * p.warp_smem;
    float* qf = reinterpret_cast<float*>(base);
    uint32_t* cid = reinterpret_cast<uint32_t*>(base + p.off_ids);
    float* cd = reinterpret_cast<float*>(base + p.off_d);
    const int dim = (int)p.dim;
    for (uint32_t q = blockIdx.x * kRerankWarps + wib; q < p.nq; q += gridDim.x * kRerankWarps) {
        __syncwarp();
        load_query(reinterpret_cast<const TD*>(p.queries) + (size_t)q * dim, dim, 16, qf, lane);
        const uint32_t n = min(p.list_counts[q], p.list_cap);
        uint32_t m = 0;  // candidates that are neither start points nor deleted, traversal order kept
        for (uint32_t b = 0; b < n; b += 32) {
            const uint32_t i = b + lane;
            const uint32_t id = i < n ? p.list_ids[(size_t)q * p.list_cap + i] : kEmptyV2;
            const bool keep = i < n && id < p.n_points && !(p.deleted && (__ldg(p.deleted + (id >> 5)) >> (id & 31) & 1u));
            const unsigned mk = __ballot_sync(kFull, keep);
            if (keep) cid[m + __popc(mk & ((1u << lane) - 1u))] = id;
            m += __popc(mk);
        }
        __syncwarp();
        if constexpr (kInt) {
            int qq = 0;
            if (KIND != KIND_IP) qq = warp_int_self<std::is_same<TD, int8_t>::value>(reinterpret_cast<const uint8_t*>(qf), dim, lane);
            wide_distances_int<std::is_same<TD, int8_t>::value, KIND, POST, 4>(reinterpret_cast<const uint8_t*>(qf), qq, p.vectors, p.row_stride,
                                                                             cid, m, cd, dim, lane);
        } else if constexpr (NA == 2) {
            constexpr int S = 16, U = 2;
            const int team = lane / S, slot = lane % S;
            for (uint32_t c0 = 0; c0 < m; c0 += 2 * U) {  // every lane takes part in the team shuffles: uniform trip count
                const TD* rows[U];
#pragma unroll
                for (int u = 0; u < U; ++u)
                    rows[u] = reinterpret_cast<const TD*>(p.vectors + (size_t)cid[min(c0 + team * U + u, m - 1)] * p.row_stride);
                float r[U];
                team_float_multi<2, KIND, U>(qf, rows, dim, slot, r);
#pragma unroll
                for (int u = 0; u < U; ++u)
                    if (slot == 0 && c0 + team * U + u < m) cd[c0 + team * U + u] = post_op<POST>(r[u]);
            }
        } else {
            wide_distances<TD, KIND, POST, 2, 4>(qf, p.vectors, p.row_stride, cid, m, cd, dim, lane);
        }
        __syncwarp();
        for (uint32_t i = lane; i < m; i += 32) {
            const float di = cd[i];
            uint32_t r = 0;
            for (uint32_t j = 0; j < m; ++j) {
                const float dj = cd[j];
                r += (dj < di || (dj == di && j < i)) ? 1u : 0u;
            }
            if (r < p.k) {
                p.out_ids[(size_t)q * p.k + r] = cid[i];
                p.out_dists[(size_t)q * p.k + r] = di;
            }
        }
        const uint32_t count = min(m, p.k);
        pad_results(p.out_ids, p.out_dists, q, p.k, count, lane);
        if (lane == 0 && p.out_counts) p.out_counts[q] = count;
    }
}

// shared memory of one rerank_kernel warp: the query (i8 / u8 rows: as they are; float rows: f32), the list's ids and
// distances
static size_t rerank_warp_smem(bool is_int, uint32_t dim, uint32_t list_cap) {
    return (is_int ? round_up((size_t)dim, 16) : round_up((size_t)dim * 4, 16)) + 2 * round_up((size_t)list_cap * 4, 16);
}

// the rerank of lists of list_cap entries fits a CTA of this index's schema
static int check_rerank(const dab_index* idx, uint32_t list_cap) {
    return visit_schema<OPS_ROW>(idx->dtype, idx->metric, [&](auto s) -> int {
        const size_t smem = rerank_warp_smem(decltype(s)::IS_INT, idx->dim, list_cap) * kRerankWarps;
        if (smem > 200 * 1024) return fail(DAB_ERR_INVALID_ARGUMENT, "rerank: configuration needs %zu B shared memory per CTA", smem);
        return DAB_OK;
    });
}

static int launch_rerank(const dab_index* idx, cudaStream_t stream, const void* d_queries, uint32_t nq, uint32_t k, uint32_t list_cap,
                         const uint32_t* d_list, const uint32_t* d_list_n, uint32_t* d_ids, float* d_dists, uint32_t* d_counts,
                         const uint32_t* deleted) {
    RerankParams p;
    memset(&p, 0, sizeof(p));
    p.vectors = idx->d_vectors;
    p.row_stride = idx->row_stride;
    p.n_points = idx->n_points;
    p.dim = idx->dim;
    p.queries = d_queries;
    p.nq = nq;
    p.k = k;
    p.list_cap = list_cap;
    p.list_ids = d_list;
    p.list_counts = d_list_n;
    p.out_ids = d_ids;
    p.out_dists = d_dists;
    p.out_counts = d_counts;
    p.deleted = deleted;
    const int grid = (int)std::min<uint64_t>(((uint64_t)nq + kRerankWarps - 1) / kRerankWarps, (uint64_t)idx->sm_count * 8);
    const int rc = visit_schema<OPS_ROW>(idx->dtype, idx->metric, [&](auto s) -> int {
        using S = decltype(s);
        const size_t off = S::IS_INT ? round_up((size_t)idx->dim, 16) : round_up((size_t)idx->dim * 4, 16);
        p.off_ids = (uint32_t)off;
        p.off_d = (uint32_t)(off + round_up((size_t)list_cap * 4, 16));
        p.warp_smem = (uint32_t)rerank_warp_smem(S::IS_INT, idx->dim, list_cap);
        const size_t smem = (size_t)p.warp_smem * kRerankWarps;
        if (smem > 200 * 1024) return fail(DAB_ERR_INVALID_ARGUMENT, "rerank: configuration needs %zu B shared memory per CTA", smem);
        auto kern = rerank_kernel<typename S::TD, S::KIND, S::POST, S::NA>;
        DAB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, kRerankWarps * 32, smem, stream>>>(p);
        return DAB_OK;
    });
    if (rc) return rc;
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    return DAB_OK;
}

// The checks of a quantized search that need no plan: arguments, the store, the metric, the list length
static int check_pq_args(const dab_index* idx, uint32_t k, uint32_t l_search, uint32_t beam, QuantStore mode) {
    int rc;
    // every entry point of a store reports under its synchronous host-buffer call's name
    const char* who = mode == STORE_PQ ? "dab_search_batch_pq" : mode == STORE_SQ ? "dab_search_batch_sq" : "dab_search_batch_minmax";
    if ((rc = check_search_args(idx, k, l_search, beam, false)) || (rc = check_quant_store(idx, mode, who, false))) return rc;
    if (l_search + idx->n_start > 1024)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: L + #start must be <= 1024", mode == STORE_MINMAX ? "dab_search_batch_minmax" : "dab_search_batch_pq");
    return DAB_OK;
}

// ---- one quantized batch as a resumable job --------------------------------------------------
// The quantized counterpart of SearchJob (search_kernel.cu).  `prepare` plans the batch (check_pq_args has passed),
// makes the checks of the plan and reserves every buffer the first pass needs (nothing is queued); `launch` queues the staging of the queries (SQ, MinMax), the first traversal pass, the
// read-back of its counters (and the MinMax NaN flag) into pinned memory and, optimistically, the rerank; `finish`
// waits for the counters, learns the visited-set size, re-runs the queries whose visited set outgrew its table on
// larger tables and then queues the rerank of the whole batch again.  The synchronous entry points run prepare, launch
// and finish on the handle's stream and scratch; the *_async calls on a slot's.  A re-run reads the store the batch was
// planned on: if a quantized store was replaced since (retire_quantized_stores), finish fails instead.
struct PqSearchJob : SlotJob {
    dab_index* idx = nullptr;
    cudaStream_t stream = nullptr;
    Scratch *tables = nullptr, *counters = nullptr, *stage = nullptr, *luts = nullptr, *lists = nullptr;
    uint32_t* h_counters = nullptr;  // pinned: the four counters of a pass, then (u64 at word 4) the MinMax NaN flag

    QuantStore mode = STORE_PQ;
    bool rerank = false;
    const void* d_queries = nullptr;
    uint32_t nq = 0, k = 0, l_search = 0, beam = 0, cap = 0;
    SearchParamsPq p;
    PqsPlan plan;
    bool use_pqs = false;
    void (*kern)(const SearchParamsPq) = nullptr;
    int grid = 0;
    size_t smem_block = 0;
    uint64_t slots = 0;
    int pass = 0;
    Scratch retry;
    cudaEvent_t counted = nullptr;  // recorded after the read-back of a pass's counters
    uint64_t stores_version = 0;    // idx->stores_version when the batch was planned
    // some id is deleted: the rerank drops deleted ids; without rerank the traversal writes every non-start entry of a
    // list (k = L + #start) to `lists` and the filter takes the first k live ones into `filtered`, the caller's buffers
    const uint32_t* deleted = nullptr;
    SearchOut filtered{};

    int prepare(const void* d_queries_, uint32_t nq_, uint32_t k_, uint32_t l_search_, uint32_t beam_, const SearchOut& d, bool rerank_, QuantStore mode_);
    int stage_queries();
    int launch_traversal();
    int launch() override;
    int finish() override;
    int launch_pass();
    int launch_post();
    int reserve_tables();
    unsigned long long first_nan() const { return *(const unsigned long long*)(h_counters + 4); }
    int nan_error() const {
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_search_batch_minmax: query %llu contains NaN after the transform (InputContainsNaN)", first_nan());
    }
    ~PqSearchJob() override {
        retry.release();
        if (counted) cudaEventDestroy(counted);
    }
};

int PqSearchJob::prepare(const void* d_queries_, uint32_t nq_, uint32_t k_, uint32_t l_search_, uint32_t beam_, const SearchOut& d,
                         bool rerank_, QuantStore mode_) {
    d_queries = d_queries_, nq = nq_, k = k_, l_search = l_search_, beam = beam_, rerank = rerank_, mode = mode_;
    stores_version = idx->stores_version;
    int rc;
    cap = l_search + idx->n_start;
    memset(&p, 0, sizeof(p));
    p.adj = idx->d_adj;
    p.adj_stride = idx->adj_stride;
    p.n_points = idx->n_points;
    p.n_start = idx->n_start;
    p.dim = idx->dim;
    p.max_degree = idx->max_degree;
    p.dtype = idx->dtype;
    p.queries = d_queries;
    p.k = k;
    p.cap = cap;
    p.beam = beam;
    set_store_params(idx, mode, p);
    p.out_ids = d.ids;
    p.out_dists = d.dists;
    p.out_counts = d.counts;
    p.out_cmps = d.cmps;
    p.out_hops = d.hops;
    deleted = deleted_filter(idx);
    if (deleted && !rerank) {
        if ((rc = lists->reserve((size_t)nq * cap * 8))) return rc;
        filtered = d;
        p.k = cap;
        p.out_ids = (uint32_t*)lists->p;
        p.out_dists = (float*)(p.out_ids + (size_t)nq * cap);
    }

    size_t off = 0;
    p.off_q = 0;
    off += round_up((size_t)idx->dim * 4, 16);
    const size_t cap_pad = round_up(cap, 32) + 32;
    p.off_qd = (uint32_t)off;
    off += cap_pad * 4;
    p.off_qi = (uint32_t)off;
    off += cap_pad * 4;
    const size_t ncand_max = std::max<size_t>((size_t)beam * idx->max_degree, idx->n_start);
    p.off_cid = (uint32_t)off;
    off += round_up(ncand_max * 4, 16);
    p.off_cd = (uint32_t)off;
    off += round_up(ncand_max * 4, 16);
    p.off_beam = (uint32_t)off;
    off += round_up((size_t)beam * 4, 16);
    p.off_qc = (uint32_t)off;
    if (mode == STORE_SQ) off += p.code_stride;
    if (mode == STORE_MINMAX) off += p.code_stride + 16;  // the query's code row and its four compensations
    off = round_up(off, 16);
    p.off_nrow = (uint32_t)off;  // search_kernel_pqs: the adjacency row copied one hop ahead
    if (mode == STORE_PQ) off += 96 * 4;
    p.warp_smem = (uint32_t)round_up(off, 16);
    // table metrics with a pivot table that fits shared memory: search_kernel_pqs (pivots resident per SM, entries
    // computed on the fly); everything else — SQ, DirectCosine, wide pivots, > 32 chunks — the per-warp kernel below
    memset(&plan, 0, sizeof(plan));
    use_pqs = mode == STORE_PQ && !p.direct_cosine && pqs_plan(idx, p.warp_smem, nq, &plan);
    smem_block = (size_t)p.warp_smem * kPqWarps;
    uint32_t warps;
    if (use_pqs) {
        p.piv_stride = plan.piv_stride;
        p.piv_bytes = plan.piv_bytes;
        grid = plan.grid;
        warps = (uint32_t)plan.grid * (uint32_t)plan.warps;
    } else {
        if (smem_block > 200 * 1024) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_search_batch_pq: configuration needs %zu B shared memory per CTA", smem_block);
        kern = visit_list_tile(cap, [&](auto qt) {
            constexpr int QT = decltype(qt)::value;
            return mode == STORE_MINMAX ? search_kernel_pq<QT, STORE_MINMAX> : mode == STORE_SQ ? search_kernel_pq<QT, STORE_SQ> : search_kernel_pq<QT, STORE_PQ>;
        });
        DAB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_block));
        int per_sm = 0;
        DAB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kPqWarps * 32, smem_block));
        if (per_sm < 1) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_search_batch_pq: kernel does not fit");
        // every resident warp owns a LUT (n_chunks x n_centers f32: 32 KB at 32 x 256) and a visited table in
        // global memory; ADC terms and probes are L2 hits only while all of them stay L2-resident
        // (the SQ kernel has no LUT: it keeps the occupancy the shared memory allows)
        if (mode == STORE_PQ) per_sm = std::min(per_sm, 6);
        grid = (int)std::min<uint64_t>((uint64_t)per_sm * idx->sm_count, ((uint64_t)nq + kPqWarps - 1) / kPqWarps);
        warps = (uint32_t)grid * kPqWarps;
    }

    if ((rc = counters->reserve(16 + (size_t)nq * 4))) return rc;
    p.counters = (uint32_t*)counters->p;
    p.overflow_list = p.counters + 4;
    const size_t lut_bytes = mode == STORE_PQ && !use_pqs ? (size_t)warps * idx->pq_chunks * idx->pq_centers * 4 : 16;
    if ((rc = luts->reserve(lut_bytes))) return rc;
    p.luts = (float*)luts->p;
    p.n_work = nq;
    if (rerank) {
        if (!idx->vectors_ready) return fail(DAB_ERR_NOT_READY, "dab_search_batch_pq: rerank needs the full-precision vectors");
        if ((rc = check_rerank(idx, cap))) return rc;
        if ((rc = lists->reserve(((size_t)nq * cap + nq) * 4))) return rc;
        p.list_ids = (uint32_t*)lists->p;
        p.list_counts = p.list_ids + (size_t)nq * cap;
        p.list_cap = cap;
    }
    // global-table passes: the overflowed queries of one are re-run on larger tables in the next
    slots = table_slots(idx, idx->pq_hint, l_search, beam, mode);
    pass = 0;
    if ((rc = reserve_tables())) return rc;
    if ((rc = stage->reserve(mode == STORE_SQ ? sq_stage_bytes(idx, nq) : mode == STORE_MINMAX ? minmax_stage_bytes(idx, nq) : 0))) return rc;
    DAB_CUDA(cudaEventCreateWithFlags(&counted, cudaEventDisableTiming));
    return DAB_OK;
}

// SQ and MinMax: the batch's queries compressed by the store's quantizer (MinMax: the NaN flag read back into h_counters)
int PqSearchJob::stage_queries() {
    if (mode == STORE_SQ) return sq_stage_queries(idx, stream, *stage, d_queries, nq, &p.query_codes, &p.query_meta);
    if (mode == STORE_MINMAX) return minmax_stage_queries(idx, stream, *stage, d_queries, nq, (unsigned long long*)(h_counters + 4), &p.query_codes, &p.query_meta);
    return DAB_OK;
}

// a visited table of `slots` ids per resident warp
int PqSearchJob::reserve_tables() {
    int rc;
    p.n_buckets = (uint32_t)((slots + 7) / 8);
    const size_t warps = use_pqs ? (size_t)plan.grid * plan.warps : (size_t)grid * kPqWarps;
    if ((rc = tables->reserve(warps * p.n_buckets * 32))) return rc;
    p.tables = (uint32_t*)tables->p;
    return DAB_OK;
}

// one traversal pass over p.n_work queries (tables reserved) and the read-back of its counters
int PqSearchJob::launch_pass() {
    int rc;
    DAB_CUDA(cudaMemsetAsync(p.counters, 0, 16, stream));
    if (use_pqs) {
        if ((rc = pqs_launch(p, plan, cap, stream))) return rc;
    } else {
        kern<<<grid, kPqWarps * 32, smem_block, stream>>>(p);
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
    }
    DAB_CUDA(cudaMemcpyAsync(h_counters, p.counters, 16, cudaMemcpyDeviceToHost, stream));
    DAB_CUDA(cudaEventRecord(counted, stream));
    return DAB_OK;
}

// the post-processing of the whole batch: the rerank, or the filter of deleted ids
int PqSearchJob::launch_post() {
    if (rerank) return launch_rerank(idx, stream, d_queries, nq, k, cap, p.list_ids, p.list_counts, p.out_ids, p.out_dists, p.out_counts, deleted);
    if (deleted) return queue_drop_deleted(idx, stream, deleted, p.out_ids, p.out_dists, cap, nq, k, filtered);
    return DAB_OK;
}

// the first pass and, optimistically, the post-processing
int PqSearchJob::launch_traversal() {
    int rc;
    if ((rc = launch_pass())) return rc;
    return launch_post();
}

int PqSearchJob::launch() {
    int rc;
    if ((rc = stage_queries())) return rc;
    return launch_traversal();
}

int PqSearchJob::finish() {
    DAB_CUDA(cudaEventSynchronize(counted));
    if (mode == STORE_MINMAX && first_nan() != ~0ull) return nan_error();
    for (;;) {
        learn_visited(idx->pq_hint, l_search, beam, mode, h_counters[2]);
        const uint32_t n_over = h_counters[1];
        if (n_over == 0) break;
        // the store the batch was planned on has been freed: its overflowed queries cannot be re-run
        if (idx->stores_version != stores_version)
            return fail(DAB_ERR_INVALID_ARGUMENT, "dab_wait: a quantized store was replaced while the batch was in flight; "
                                                  "%u of its queries could not be re-run", n_over);
        int rc;
        if ((rc = take_overflow_list(stream, p.overflow_list, n_over, retry)) || (rc = grow_visited_tables(idx, pass, slots)) ||
            (rc = reserve_tables()))
            return rc;
        p.query_list = (const uint32_t*)retry.p;
        p.n_work = n_over;
        reran = true;
        if ((rc = launch_pass())) return rc;
        DAB_CUDA(cudaEventSynchronize(counted));
    }
    // the rerank or filter queued by launch read lists that the re-runs have since rewritten
    return reran ? launch_post() : DAB_OK;
}

// The synchronous calls: the job on the handle's stream and scratch.  A MinMax batch with a NaN query fails before any
// traversal is launched.  Device pointers only; returns once the traversal is complete (the rerank may still run).
static int run_search_pq(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam,
                         const SearchOut& d, bool rerank, QuantStore mode) {
    int rc;
    if ((rc = idx->h_counters.reserve(24))) return rc;
    PqSearchJob job;
    job.idx = idx;
    job.stream = idx->stream;
    job.tables = &idx->s_tables, job.counters = &idx->s_counters, job.stage = &idx->s_stage, job.luts = &idx->s_out2, job.lists = &idx->s_ids;
    job.h_counters = (uint32_t*)idx->h_counters.p;
    if ((rc = check_pq_args(idx, k, l_search, beam, mode)) || (rc = job.prepare(d_queries, nq, k, l_search, beam, d, rerank, mode))) return rc;
    if ((rc = job.stage_queries())) return rc;
    if (mode == STORE_MINMAX) {
        DAB_CUDA(cudaStreamSynchronize(idx->stream));
        if (job.first_nan() != ~0ull) return job.nan_error();
    }
    if ((rc = job.launch_traversal())) return rc;
    return job.finish();
}

static int search_pq_host(dab_index* idx, const char* api, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                          uint32_t beam_width, const SearchOut& out, bool rerank, QuantStore mode) {
    return search_host_buffers(idx, api, queries, nq, k, out, [&](const void* d_queries, const SearchOut& d) {
        return run_search_pq(idx, d_queries, nq, k, l_search, beam_width, d, rerank, mode);
    });
}

static int search_pq_device(dab_index* idx, const char* api, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                            uint32_t beam_width, const SearchOut& d, bool rerank, QuantStore mode) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", api);
    if (nq == 0) return DAB_OK;
    if (!d_queries || !d.ids || !d.dists) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL argument", api);
    DAB_CUDA(cudaSetDevice(idx->device));
    return run_search_pq(idx, d_queries, nq, k, l_search, beam_width, d, rerank, mode);
}

// The *_async calls: the job on the slot's stream and scratch
static int search_pq_async(dab_index* idx, const char* api, uint32_t slot, bool host, const void* queries, uint32_t nq, uint32_t k,
                           uint32_t l_search, uint32_t beam_width, const SearchOut& out, bool rerank, QuantStore mode) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", api);
    if (nq && (!queries || !out.ids || !out.dists)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL argument", api);
    int rc;
    if ((rc = check_pq_args(idx, k, l_search, beam_width, mode))) return rc;  // before the slot rules, as the full-precision call
    return slot_submit(idx, api, slot, host, queries, nq, k, out, [&](SearchSlot* s, const void* d_queries, const SearchOut& d, SlotJob** out_job) {
        int rc2;
        if ((rc2 = s->h_counters.reserve(24))) return rc2;
        PqSearchJob* job = new PqSearchJob();
        *out_job = job;
        job->idx = idx;
        job->stream = s->stream;
        job->tables = &s->tables, job->counters = &s->counters, job->stage = &s->stage, job->luts = &s->luts, job->lists = &s->lists;
        job->h_counters = (uint32_t*)s->h_counters.p;
        return job->prepare(d_queries, nq, k, l_search, beam_width, d, rerank, mode);
    });
}

}  // namespace dab

using namespace dab;

extern "C" {

int dab_search_batch_pq(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                        uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops) {
    return search_pq_host(idx, "dab_search_batch_pq", queries, nq, k, l_search, beam_width,
                          SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, false, STORE_PQ);
}

int dab_search_batch_pq_rerank(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                               uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops) {
    return search_pq_host(idx, "dab_search_batch_pq_rerank", queries, nq, k, l_search, beam_width,
                          SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, true, STORE_PQ);
}

int dab_search_batch_pq_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                               int rerank, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts, uint32_t* d_out_cmps,
                               uint32_t* d_out_hops) {
    return search_pq_device(idx, "dab_search_batch_pq_device", d_queries, nq, k, l_search, beam_width,
                            SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, rerank != 0, STORE_PQ);
}

int dab_search_batch_sq(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                        int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops) {
    return search_pq_host(idx, "dab_search_batch_sq", queries, nq, k, l_search, beam_width,
                          SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, rerank != 0, STORE_SQ);
}

int dab_search_batch_sq_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                               int rerank, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts, uint32_t* d_out_cmps,
                               uint32_t* d_out_hops) {
    return search_pq_device(idx, "dab_search_batch_sq_device", d_queries, nq, k, l_search, beam_width,
                            SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, rerank != 0, STORE_SQ);
}

int dab_search_batch_minmax(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                            int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops) {
    return search_pq_host(idx, "dab_search_batch_minmax", queries, nq, k, l_search, beam_width,
                          SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, rerank != 0, STORE_MINMAX);
}

int dab_search_batch_minmax_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                                   int rerank, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts, uint32_t* d_out_cmps,
                                   uint32_t* d_out_hops) {
    return search_pq_device(idx, "dab_search_batch_minmax_device", d_queries, nq, k, l_search, beam_width,
                            SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, rerank != 0, STORE_MINMAX);
}

// ---- asynchronous batches (see dab_search_batch_async): the same jobs on a slot, joined by dab_wait ----
int dab_search_batch_pq_async(dab_index* idx, uint32_t slot, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                              uint32_t beam_width, int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                              uint32_t* out_cmps, uint32_t* out_hops) {
    return search_pq_async(idx, "dab_search_batch_pq_async", slot, true, queries, nq, k, l_search, beam_width,
                           SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, rerank != 0, STORE_PQ);
}

int dab_search_batch_pq_device_async(dab_index* idx, uint32_t slot, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                     uint32_t beam_width, int rerank, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts,
                                     uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    return search_pq_async(idx, "dab_search_batch_pq_device_async", slot, false, d_queries, nq, k, l_search, beam_width,
                           SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, rerank != 0, STORE_PQ);
}

int dab_search_batch_sq_async(dab_index* idx, uint32_t slot, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                              uint32_t beam_width, int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                              uint32_t* out_cmps, uint32_t* out_hops) {
    return search_pq_async(idx, "dab_search_batch_sq_async", slot, true, queries, nq, k, l_search, beam_width,
                           SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, rerank != 0, STORE_SQ);
}

int dab_search_batch_sq_device_async(dab_index* idx, uint32_t slot, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                     uint32_t beam_width, int rerank, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts,
                                     uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    return search_pq_async(idx, "dab_search_batch_sq_device_async", slot, false, d_queries, nq, k, l_search, beam_width,
                           SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, rerank != 0, STORE_SQ);
}

int dab_search_batch_minmax_async(dab_index* idx, uint32_t slot, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                  uint32_t beam_width, int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                                  uint32_t* out_cmps, uint32_t* out_hops) {
    return search_pq_async(idx, "dab_search_batch_minmax_async", slot, true, queries, nq, k, l_search, beam_width,
                           SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, rerank != 0, STORE_MINMAX);
}

int dab_search_batch_minmax_device_async(dab_index* idx, uint32_t slot, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                         uint32_t beam_width, int rerank, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts,
                                         uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    return search_pq_async(idx, "dab_search_batch_minmax_device_async", slot, false, d_queries, nq, k, l_search, beam_width,
                           SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, rerank != 0, STORE_MINMAX);
}

}  // extern "C"
