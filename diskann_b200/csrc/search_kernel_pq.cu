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

// One warp's share of a pass.  KEEP_STARTS: the results are the list's first k entries with start points kept (the
// first phase of range search, which filters them itself).
template <int QT, int MODE, bool KEEP_STARTS>
__device__ __forceinline__ void pq_queries(const SearchParamsPq& p) {
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
        const uint32_t count = write_results(qi, qd, n, KEEP_STARTS ? n_total : p.n_points, p.k, p.out_ids, p.out_dists, qidx, lane);
        write_stats(p.counters, nvisited, p.out_counts, p.out_cmps, p.out_hops, qidx, count, cmps, hops, lane);
    }
}

template <int QT, int MODE>
__global__ void __launch_bounds__(kPqWarps * 32) search_kernel_pq(const SearchParamsPq p) {
    pq_queries<QT, MODE, false>(p);
}

template <int QT, int MODE>
__global__ void __launch_bounds__(kPqWarps * 32) search_kernel_pq_starts(const SearchParamsPq p) {
    pq_queries<QT, MODE, true>(p);
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
        rerank_distances<TD, KIND, POST, NA>(qf, p.vectors, p.row_stride, cid, m, cd, dim, lane);
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

int check_rerank(const dab_index* idx, const char* api, uint32_t list_cap) {
    if (!idx->vectors_ready) return fail(DAB_ERR_NOT_READY, "%s: rerank needs the full-precision vectors", api);
    return visit_schema<OPS_ROW>(idx->dtype, idx->metric, [&](auto s) -> int {
        const size_t smem = rerank_warp_smem(decltype(s)::IS_INT, idx->dim, list_cap) * kRerankWarps;
        if (smem > 200 * 1024) return fail(DAB_ERR_INVALID_ARGUMENT, "rerank: configuration needs %zu B shared memory per CTA", smem);
        return DAB_OK;
    });
}

int launch_rerank(const dab_index* idx, cudaStream_t stream, const void* d_queries, uint32_t nq, uint32_t k, uint32_t list_cap,
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

PqKernel pq_kernel(uint32_t cap, QuantStore store, bool keep_starts) {
    return visit_list_tile(cap, [&](auto qt) -> PqKernel {
        constexpr int QT = decltype(qt)::value;
        if (keep_starts)
            return store == STORE_MINMAX ? search_kernel_pq_starts<QT, STORE_MINMAX>
                   : store == STORE_SQ  ? search_kernel_pq_starts<QT, STORE_SQ>
                                        : search_kernel_pq_starts<QT, STORE_PQ>;
        return store == STORE_MINMAX ? search_kernel_pq<QT, STORE_MINMAX> : store == STORE_SQ ? search_kernel_pq<QT, STORE_SQ> : search_kernel_pq<QT, STORE_PQ>;
    });
}

}  // namespace dab
