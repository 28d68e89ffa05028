// flat_kernels.cu — exhaustive scan (diskann/src/flat, ground truth for recall) with the
// same bit-exact distance arithmetic as the graph path, so ground-truth distances equal the
// search's distances bit for bit.
//
// Register-blocked: a warp owns an 8-query x 4-row tile.  Lane s owns SIMD slot s of every
// pair in the tile (the same sequential FMA chains as distance_device.cuh); the 32 partial
// accumulators are reduced with a transpose-butterfly — stage order xor 8, 16 (accumulator
// combine), remainder, xor 4, 2, 1 (sum_tree) — that keeps the reference's association for
// every value while needing 31 shuffles per 32 pairs instead of 160.  A CTA of 8 warps shares
// the same 4 rows (L1 hits) across 64 queries held transposed-free in shared memory.
// A second kernel folds each row block into the running per-query top-k.
#include "dab_common.cuh"
#include "distance_device.cuh"

#include <algorithm>

namespace dab {

constexpr int kFlatWarps = 8;
constexpr int kFQ = 8;   // queries per warp tile
constexpr int kFR = 4;   // rows per warp tile

// one transpose-butterfly stage over M live values
template <int M>
__device__ __forceinline__ void bfly_stage(float (&v)[32], int lane, int bit) {
    const bool up = (lane & bit) != 0;
#pragma unroll
    for (int i = 0; i < M / 2; ++i) {
        const float keep = up ? v[M / 2 + i] : v[i];
        const float send = up ? v[i] : v[M / 2 + i];
        v[i] = __fadd_rn(keep, __shfl_xor_sync(kFull, send, bit));
    }
}

// index of the value a lane ends up holding after the 5 stages (see header comment)
__device__ __forceinline__ int bfly_final_index(int lane) {
    return (((lane >> 3) & 1) << 4) | (((lane >> 4) & 1) << 3) | (lane & 7);
}

// float rows x f32-widened queries, NA = 4 kernels (L2 / IP).  out[q][r - r0], ld = out_ld.
template <typename TD, int KIND, int POST>
__global__ void __launch_bounds__(kFlatWarps * 32)
flat_float_kernel(const float* __restrict__ queries /*[nq][dim] f32*/, uint32_t nq, const uint8_t* __restrict__ vectors,
                  size_t row_stride, uint32_t r0, uint32_t r1, int dim, float* __restrict__ out, size_t out_ld,
                  uint32_t rows_per_cta) {
    extern __shared__ __align__(16) float sq[];  // [kFlatWarps * kFQ][dim]
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const uint32_t q_base = blockIdx.y * (kFlatWarps * kFQ);
    for (uint32_t i = threadIdx.x; i < (uint32_t)(kFlatWarps * kFQ) * dim; i += blockDim.x) {
        const uint32_t u = i / dim, e = i % dim;
        sq[i] = q_base + u < nq ? queries[(size_t)(q_base + u) * dim + e] : 0.0f;
    }
    __syncthreads();
    const float* myq = sq + (size_t)wib * kFQ * dim;
    const uint32_t my_q0 = q_base + wib * kFQ;
    const int full8 = dim & ~7, rem = dim & 7;
    const uint32_t rb0 = r0 + blockIdx.x * rows_per_cta;
    const uint32_t rb1 = min(r1, rb0 + rows_per_cta);
    for (uint32_t r = rb0; r < rb1; r += kFR) {
        const TD* rows[kFR];
#pragma unroll
        for (int j = 0; j < kFR; ++j)
            rows[j] = reinterpret_cast<const TD*>(vectors + (size_t)min(r + j, rb1 - 1) * row_stride);
        float v[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = 0.0f;
        for (int e = lane; e < full8; e += 32) {
            float y[kFR], x[kFQ];
#pragma unroll
            for (int j = 0; j < kFR; ++j) y[j] = ldg_elem(rows[j] + e);
#pragma unroll
            for (int u = 0; u < kFQ; ++u) x[u] = myq[u * dim + e];
#pragma unroll
            for (int j = 0; j < kFR; ++j)
#pragma unroll
                for (int u = 0; u < kFQ; ++u) {
                    if (KIND == KIND_L2) {
                        const float c = __fsub_rn(x[u], y[j]);
                        v[j * kFQ + u] = __fmaf_rn(c, c, v[j * kFQ + u]);
                    } else {
                        v[j * kFQ + u] = __fmaf_rn(x[u], y[j], v[j * kFQ + u]);
                    }
                }
        }
        bfly_stage<32>(v, lane, 8);
        bfly_stage<16>(v, lane, 16);
        if (rem) {
            // 8 live values: index i | b3 << 3 | b4 << 4 with b4 = lane bit 3, b3 = lane bit 4
            const int hi = (((lane >> 4) & 1) << 3) | (((lane >> 3) & 1) << 4);
            const int l = lane & 7;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int idx = i | hi, j = idx / kFQ, u = idx % kFQ;
                const float x = l < rem ? myq[u * dim + full8 + l] : 0.0f;
                const float y = l < rem ? ldg_elem(rows[j] + full8 + l) : 0.0f;
                if (KIND == KIND_L2) {
                    const float c = __fsub_rn(x, y);
                    v[i] = __fmaf_rn(c, c, v[i]);
                } else {
                    v[i] = __fmaf_rn(x, y, v[i]);
                }
            }
        }
        bfly_stage<8>(v, lane, 4);
        bfly_stage<4>(v, lane, 2);
        bfly_stage<2>(v, lane, 1);
        const int idx = bfly_final_index(lane), j = idx / kFQ, u = idx % kFQ;
        if (r + j < rb1 && my_q0 + u < nq) out[(size_t)(my_q0 + u) * out_ld + (r + j - r0)] = post_op<POST>(v[0]);
    }
}

// Generic (slow, no row reuse) path for the schemas not covered above: float cosine
// (Strategy2x4) and the integer types.  One warp per (query, 32-row tile).
template <typename TD, int NA, int KIND, int POST, bool IS_INT, bool SIGNED>
__global__ void __launch_bounds__(kFlatWarps * 32)
flat_generic_kernel(const void* __restrict__ queries, uint32_t nq, const uint8_t* __restrict__ vectors, size_t row_stride,
                    uint32_t r0, uint32_t r1, int dim, float* __restrict__ out, size_t out_ld) {
    extern __shared__ __align__(16) uint8_t smem[];
    constexpr int S = 8 * NA, TEAMS = IS_INT ? 1 : 32 / S;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int team = IS_INT ? 0 : lane / S, slot = IS_INT ? lane : lane % S;
    const size_t qbytes = IS_INT ? (size_t)((dim + 3) & ~3) : (size_t)dim * 4;
    uint8_t* qb = smem + (size_t)wib * ((qbytes + 15) & ~(size_t)15);
    float* qf = reinterpret_cast<float*>(qb);
    const uint32_t tiles = (r1 - r0 + 31) / 32;
    const uint64_t total = (uint64_t)nq * tiles;
    const uint64_t nwarps = (uint64_t)gridDim.x * kFlatWarps;
    for (uint64_t t = (uint64_t)blockIdx.x * kFlatWarps + wib; t < total; t += nwarps) {
        const uint32_t q = (uint32_t)(t / tiles);
        const uint32_t ra = r0 + (uint32_t)(t % tiles) * 32, rb = min(r1, ra + 32);
        __syncwarp();
        if constexpr (IS_INT) {
            const uint8_t* src = reinterpret_cast<const uint8_t*>(queries) + (size_t)q * dim;
            for (int e = lane; e < (int)qbytes; e += 32) qb[e] = e < dim ? src[e] : 0;
        } else {
            const float* src = reinterpret_cast<const float*>(queries) + (size_t)q * dim;
            for (int e = lane; e < dim; e += 32) qf[e] = src[e];
        }
        __syncwarp();
        int qq = 0;
        if constexpr (IS_INT && KIND != KIND_IP) qq = warp_int_self<SIGNED>(qb, dim, lane);
        for (uint32_t r = ra; r < rb; r += TEAMS) {
            const uint32_t rr = min(r + team, rb - 1);
            float res[1];
            if constexpr (IS_INT) {
                const uint8_t* rows[1] = {vectors + (size_t)rr * row_stride};
                warp_int_multi<SIGNED, KIND, 1>(qb, rows, dim, lane, qq, res);
            } else {
                const TD* rows[1] = {reinterpret_cast<const TD*>(vectors + (size_t)rr * row_stride)};
                team_float_multi<NA, KIND, 1>(qf, rows, dim, slot, res);
            }
            if (slot == 0 && r + team < rb) out[(size_t)q * out_ld + (r + team - r0)] = post_op<POST>(res[0]);
        }
    }
}

// widen a query batch to f32 (f16 -> f32 is exact, layers/full.rs:421-423)
__global__ void widen_f16_kernel(const __half* __restrict__ src, float* __restrict__ dst, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = __half2float(src[i]);
}

// Fold dist[q][0 .. nrows) (rows r0 ..) into the running top-k of query q: ascending distance,
// ties by lower id (rows arrive in increasing id, a new item goes AFTER equal distances).
// One warp per query; top-k lists live in global memory between row blocks.
__global__ void __launch_bounds__(kFlatWarps * 32)
flat_topk_kernel(const float* __restrict__ dist, size_t ld, uint32_t nq, uint32_t r0, uint32_t nrows, uint32_t k,
                 uint32_t* __restrict__ top_ids, float* __restrict__ top_d, uint32_t* __restrict__ top_n) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    float* td = reinterpret_cast<float*>(smem) + (size_t)wib * 2 * k;
    uint32_t* ti = reinterpret_cast<uint32_t*>(td + k);
    const uint32_t q = blockIdx.x * kFlatWarps + wib;
    if (q >= nq) return;
    uint32_t n = top_n[q];
    for (uint32_t i = lane; i < n; i += 32) {
        td[i] = top_d[(size_t)q * k + i];
        ti[i] = top_ids[(size_t)q * k + i];
    }
    __syncwarp();
    const float* row = dist + (size_t)q * ld;
    for (uint32_t b = 0; b < nrows; b += 32) {
        const uint32_t j = b + lane;
        const float d = j < nrows ? row[j] : __int_as_float(0x7FC00000);
        float worst = n == k ? td[k - 1] : __int_as_float(0x7F800000);
        // NaN never enters; candidate passes if the list is not full or d < worst
        unsigned m = __ballot_sync(kFull, j < nrows && d == d && (n < k || d < worst));
        while (m) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            const float dv = __shfl_sync(kFull, d, src);
            const uint32_t id = r0 + b + src;
            if (n == k && !(dv < td[k - 1])) continue;
            // upper bound: count of entries <= dv
            uint32_t pos = 0;
            for (uint32_t s = 0; s < n; s += 32) {
                const uint32_t i = s + lane;
                const unsigned le = __ballot_sync(kFull, i < n && td[i] <= dv);
                pos += __popc(le);
                if (le != kFull) break;
            }
            if (n == k) --n;
            if (pos < n) {
                for (int s = (int)((n - 1) & ~31u); s >= (int)(pos & ~31u); s -= 32) {
                    const uint32_t i = (uint32_t)s + lane;
                    const bool mv = i >= pos && i < n;
                    float v = 0.0f;
                    uint32_t w = 0;
                    if (mv) {
                        v = td[i];
                        w = ti[i];
                    }
                    __syncwarp();
                    if (mv) {
                        td[i + 1] = v;
                        ti[i + 1] = w;
                    }
                    __syncwarp();
                }
            }
            __syncwarp();  // orders the reads above against the write below when nothing was moved (racecheck)
            if (lane == 0) {
                td[pos] = dv;
                ti[pos] = id;
            }
            __syncwarp();
            ++n;
        }
    }
    __syncwarp();
    for (uint32_t i = lane; i < n; i += 32) {
        top_d[(size_t)q * k + i] = td[i];
        top_ids[(size_t)q * k + i] = ti[i];
    }
    for (uint32_t i = n + lane; i < k; i += 32) {
        top_d[(size_t)q * k + i] = __int_as_float(0x7F800000);
        top_ids[(size_t)q * k + i] = kNoId;
    }
    if (lane == 0) top_n[q] = n;
}

// The exact scan of nq queries already on the device (index dtype, packed rows) into the device top-k lists d_top_ids /
// d_top_d ([nq][k]).  dab_flat_knn and the queries dab_flat_knn_tc cannot certify both run it.  Its only scratch is
// s_out2, so a caller may keep its queries and results in the other buffers.
int flat_knn_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t* d_top_ids, float* d_top_d) {
    const int dim = (int)idx->dim;
    const uint32_t n = (uint32_t)idx->n_points;  // start points are not data
    cudaStream_t st = idx->stream;

    // row block sized so the distance tile stays around 1 GiB
    uint32_t rb = (uint32_t)std::min<uint64_t>(n, std::max<uint64_t>(1024, ((1ull << 30) / 4) / nq));
    rb = (rb + 31) & ~31u;
    // scratch: [f16 queries widened to f32 | per-query list lengths | distance tile]
    const size_t qf_bytes = idx->dtype == DAB_F16 ? round_up((size_t)nq * dim * 4, 256) : 0;
    const size_t tn_bytes = round_up((size_t)nq * 4, 256);
    int rc;
    if ((rc = idx->s_out2.reserve(qf_bytes + tn_bytes + (size_t)nq * rb * 4))) return rc;
    float* d_qf = (float*)idx->s_out2.p;
    uint32_t* d_top_n = (uint32_t*)((uint8_t*)idx->s_out2.p + qf_bytes);
    float* d_dist = (float*)((uint8_t*)d_top_n + tn_bytes);
    const void* d_q = d_queries;
    if (idx->dtype == DAB_F16) {  // floats widened to f32 once
        widen_f16_kernel<<<idx->sm_count * 4, 256, 0, st>>>((const __half*)d_queries, d_qf, (size_t)nq * dim);
        DAB_LAUNCHED();
        d_q = d_qf;
    }
    DAB_CUDA(cudaMemsetAsync(d_top_n, 0, (size_t)nq * 4, st));

    const bool fast_fits = (size_t)kFlatWarps * kFQ * dim * 4 <= 200 * 1024;
    for (uint32_t r0 = 0; r0 < n; r0 += rb) {
        const uint32_t r1 = std::min(n, r0 + rb);
        rc = visit_schema<OPS_QUERY>(idx->dtype, idx->metric, [&](auto s) -> int {
            using S = decltype(s);
            if constexpr (!S::IS_INT && S::KIND != KIND_COS) {
                if (fast_fits) {
                    const size_t smem = (size_t)kFlatWarps * kFQ * dim * 4;
                    const uint32_t qtiles = (nq + kFlatWarps * kFQ - 1) / (kFlatWarps * kFQ);
                    // enough CTAs along rows to fill the machine ~4x, at least 64 rows per CTA
                    uint32_t rsplit = std::max<uint32_t>(1, std::min<uint32_t>((r1 - r0 + 63) / 64, (idx->sm_count * 8 + qtiles - 1) / qtiles));
                    uint32_t rows_per_cta = ((r1 - r0 + rsplit - 1) / rsplit + kFR - 1) / kFR * kFR;
                    rsplit = (r1 - r0 + rows_per_cta - 1) / rows_per_cta;
                    dim3 grid(rsplit, qtiles);
                    auto kern = flat_float_kernel<typename S::TD, S::KIND, S::POST>;
                    DAB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                    kern<<<grid, kFlatWarps * 32, smem, st>>>((const float*)d_q, nq, idx->d_vectors, idx->row_stride, r0, r1, dim,
                                                              d_dist, rb, rows_per_cta);
                    return DAB_OK;
                }
            }
            const size_t qb = S::IS_INT ? round_up(dim, 4) : (size_t)dim * 4;
            const size_t smem = (size_t)kFlatWarps * round_up(qb, 16);
            const uint64_t tiles = (uint64_t)nq * ((r1 - r0 + 31) / 32);
            int grid = (int)std::min<uint64_t>((tiles + kFlatWarps - 1) / kFlatWarps, (uint64_t)idx->sm_count * 8);
            auto kern = flat_generic_kernel<KernelRow<S>, S::NA, S::KIND, S::POST, S::IS_INT, S::SIGNED>;
            DAB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            kern<<<grid, kFlatWarps * 32, smem, st>>>(d_q, nq, idx->d_vectors, idx->row_stride, r0, r1, dim, d_dist, rb);
            return DAB_OK;
        });
        if (rc) return rc;
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
        const size_t tsmem = (size_t)kFlatWarps * 2 * k * 4;
        DAB_CUDA(cudaFuncSetAttribute(flat_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tsmem));
        flat_topk_kernel<<<(nq + kFlatWarps - 1) / kFlatWarps, kFlatWarps * 32, tsmem, st>>>(d_dist, rb, nq, r0, r1 - r0, k, d_top_ids,
                                                                                          d_top_d, d_top_n);
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
    }
    return DAB_OK;
}

}  // namespace dab

using namespace dab;

extern "C" {

int dab_flat_knn(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t* out_ids, float* out_dists) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_flat_knn: idx is NULL");
    if (!idx->vectors_ready) return fail(DAB_ERR_NOT_READY, "dab_flat_knn: vectors not uploaded");
    if (nq == 0) return DAB_OK;
    if (!queries || !out_ids || !out_dists) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_flat_knn: NULL argument");
    if (k == 0 || k > 2048) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_flat_knn: k must be in [1, 2048]");
    DAB_CUDA(cudaSetDevice(idx->device));
    cudaStream_t st = idx->stream;
    const size_t qraw = (size_t)nq * idx->dim * elem_size(idx->dtype);
    int rc;
    if ((rc = idx->s_queries.reserve(qraw))) return rc;
    if ((rc = idx->s_out.reserve((size_t)nq * k * 8))) return rc;
    uint32_t* d_top_ids = (uint32_t*)idx->s_out.p;
    float* d_top_d = (float*)(d_top_ids + (size_t)nq * k);
    DAB_CUDA(cudaMemcpyAsync(idx->s_queries.p, queries, qraw, cudaMemcpyHostToDevice, st));
    if ((rc = flat_knn_device(idx, idx->s_queries.p, nq, k, d_top_ids, d_top_d))) return rc;
    DAB_CUDA(cudaMemcpyAsync(out_ids, d_top_ids, (size_t)nq * k * 4, cudaMemcpyDeviceToHost, st));
    DAB_CUDA(cudaMemcpyAsync(out_dists, d_top_d, (size_t)nq * k * 4, cudaMemcpyDeviceToHost, st));
    DAB_CUDA(cudaStreamSynchronize(st));
    return DAB_OK;
}

}  // extern "C"
