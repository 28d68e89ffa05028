// flat_tc.cu — exhaustive scan (diskann/src/flat, ground truth for recall) on the Hopper tensor
// cores: the query x base distance block is a dense contraction, so it runs as a wgmma GEMM with
// TMA-staged tiles and a fused norm expansion + per-row candidate selection
// (BASELINE.json north_star; SURVEY.md §8f.3).
//
//   * operands are bf16.  f32 / f16 rows are split x = hi + lo (hi = bf16(x), lo = bf16(x - hi)) and
//     the three significant products are obtained from ONE GEMM over a 3x longer K:
//     A' = [q_hi | q_hi | q_lo], B' = [b_hi | b_lo | b_hi]  =>  A'.B' = hi.hi + hi.lo + lo.hi
//     (relative error of the dot product ~2^-16; fp32 accumulation in registers).  i8 / u8 rows are
//     exact in bf16 and their products / sums are exact in fp32 (128 * 127^2 < 2^24): one segment.
//   * one CTA = 128 query rows x a range of base rows; per 128-column tile: K' / 64 pipeline stages
//     of (A k-block, B k-block) 128 x 64 bf16 tiles loaded by TMA (128-byte swizzle) into shared
//     memory by a producer warp, and 4 k-steps x 2 row halves of wgmma.m64n128k16 per stage issued by
//     one consumer warpgroup, whose 128 threads hold the 128 x 128 f32 accumulator tile (2 x 64
//     registers each); the producer runs up to a whole pipeline of stages ahead, so the loads of the
//     next tile overlap the epilogue of this one;
//   * epilogue (the consumer warpgroup): score = alpha[col] * dot + beta[col] (L2: ||b||^2 - 2 q.b, the
//     ||q||^2 term is constant per row; inner product: -q.b; cosine: -q.b / ||b||), transposed through
//     shared memory 32 columns at a time so that each thread owns one query row, which keeps the KP best
//     columns of the row in a small per-thread set;
//   * the KP candidates of every (query, base range) are then re-scored with the exact, reference-order
//     distance kernel (launch_frontier) and the final top-k is taken by (distance, id);
//   * every query is then certified (certify_kernel): the range's largest kept score W, less a rigorous bound E
//     on the approximate score's error, must map to a distance strictly above the query's exact k-th distance, so
//     no row the selection dropped can belong in the top-k.  The queries that fail (ill-conditioned data: a large
//     common offset, near-duplicates beyond the slack, fp32 sums past 2^24, norms that underflow, NaN / inf rows,
//     n < k) are re-run through the exact scan (flat_knn_device) and scattered back.  So the ids and the distance
//     bits always equal dab_flat_knn's.
//
// The error bound E (certify_kernel; u = 2^-24 is fp32 round-to-nearest, gamma(n, v) = n v / (1 - n v)).  For a
// query q and a row b of the range, with B^2 an upper bound of the range's ||b||^2:
//   * split residuals: x = hi + lo + r with |hi| <= (1 + 2^-8)|x|, |lo| <= 2^-8 (1 + 2^-8)|x|, |r| <= 2^-16 |x|.  The
//     three products hi.hi + hi.lo + lo.hi miss lo.lo + hi.r + r.hi + (smaller): at most 2^-14 |q_i b_i| per element,
//     2^-14 ||q|| ||b|| in all (Cauchy-Schwarz).  i8 / u8 rows are exact in bf16: no split error.
//   * accumulation: the bf16 products are exact in fp32; kp of them (3 dim for floats) are summed in fp32 by the
//     tensor cores in an unspecified order, assumed no better than truncation: gamma(kp, 2^-23) times the sum of
//     |products| <= 1.03 ||q|| ||b||.  For i8 / u8 every partial sum is an integer of magnitude <= ||q|| ||b||, so
//     the dot is exact while ||q|| B < 2^24.  Flushed subnormals cost at most kp 2^-125 (||q|| + ||b|| + 1).
//     Together: E_dot.
//   * epilogue: the row's ||b||^2 in `beta` is an fp32 sum (gamma(dim, u) relative), the fma rounds once (u), and
//     for cosine 1 / ||b|| comes from rsqrtf (2 ulp): rho = 2^-22 + gamma(dim, u) + u relative.
//   * the exact distance of the row, which is what the k-th distance is compared with, is itself an fp32 sum in
//     the reference's order: gamma(dim + 2, u) relative for L2, gamma(dim, u) ||q|| ||b|| for the dot, and
//     2 gamma(dim, u) + 7u absolute for cosine's sqrt / divide / clamp / 1 - x.
// Every row the selection dropped scored at least W (W = FLT_MAX when the range kept fewer than KP), so with D_k
// the exact k-th distance a query is certified when, for every range (a 1.01 factor covers the second-order terms):
//   L2:                        (||q||^2 + W - E)(1 - gamma(dim + 2, u)) > D_k,  E = 2 E_dot + (gamma(dim, u) + 2u)(B^2 + 2 ||q|| B)
//   IP:                        W - E > D_k,                                      E = E_dot + gamma(dim, u) ||q|| B
//   float CosineNormalized:    (1 + W - E) - 2u |1 + W - E| > D_k,              E as for IP
//   Cosine, int CosNormalized: 1 + (W - E) / ||q|| - (2 gamma(dim, u) + 7u) > D_k,  E = ||q|| ((e + 1) rho + e) + kp 2^-70 (||q|| + 1),
//                              with e the dot's relative term above (0 for exact integer dots)
// and the query has k finite distances, ||q||^2 + B^2 + 2 ||q|| B < 2^120 (no score can overflow) and, for cosine,
// ||q||^2 >= 2^-100.  A cosine row whose fp32 ||b||^2 lies in (0, 2^-100) makes its tile uncertifiable: the exact
// kernel may or may not treat its norm as zero.  A row whose ||b||^2 is 0 scores 0, which is its exact distance 1.
#include "dab_common.cuh"
#include "distance_device.cuh"

#include <cuda.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <vector>

namespace dab {

int launch_frontier(const dab_index* idx, const void* d_queries, uint32_t nq, const uint32_t* d_ids, uint32_t c, float* d_out);
int flat_knn_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t* d_top_ids, float* d_top_d);

namespace {

constexpr int kBM = 128, kBN = 128, kBK = 64;  // CTA tile; one k-block = 64 bf16 = one 128-byte swizzle row
constexpr int kStages = 5;                    // stages of (A k-block, B k-block)
constexpr int kTcThreads = 160;                // warps 0-3: MMA + epilogue warpgroup, warp 4: TMA
constexpr int kKP = 32;                        // largest candidate set per (query row, base range); k <= 10 uses 16
constexpr uint32_t kTileBytes = kBM * kBK * 2; // 16 KB per operand tile

// ---- PTX wrappers ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int32_t x, int32_t y) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
                 "l"(map), "r"(smem_u32(bar)), "r"(x), "r"(y)
                 : "memory");
}
// K-major operand tile [rows][64 bf16] written by TMA with the 128-byte swizzle: 8-row groups of
// 1024 bytes (SBO = 1024 B), LBO unused (1), layout type 1 = SWIZZLE_128B (PTX ISA, "Matrix Descriptor
// Format" of wgmma); a k-step of 16 elements advances the start address by 32 bytes inside the swizzle row
__device__ __forceinline__ uint64_t gmma_desc(const void* tile, uint32_t k_byte_offset) {
    const uint32_t addr = smem_u32(tile) + k_byte_offset;
    return (uint64_t)((addr >> 4) & 0x3FFFu) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// D[64 x 128] (+)= A[64 x 16] . B[128 x 16]^T, bf16 inputs from shared memory (both K-major), f32 accumulators.
// Fragment of thread t of the warpgroup: d[4j + r] is row 16 (t / 32) + (t % 32) / 4 + 8 (r / 2),
// column 8 j + 2 (t % 4) + (r % 2).
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, "
        "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
          "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),
          "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
          "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of the accumulators across the asynchronous MMAs
__device__ __forceinline__ void fence_operands(float (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---- operand preparation --------------------------------------------------------------------
// rows of the index dtype -> bf16 [n][kp]: f32 / f16: (hi, hi, lo) for queries, (hi, lo, hi) for base
// rows; i8 / u8: one exact segment.  Base rows also get their score coefficients.
template <typename T>
__device__ __forceinline__ float elem_f32(const T* p, uint32_t i) {
    if constexpr (sizeof(T) == 2) return __half2float(p[i]);
    else return (float)p[i];
}
template <typename T>
__global__ void prep_bf16_kernel(const uint8_t* __restrict__ rows, size_t row_stride, uint64_t n, uint32_t dim, uint32_t kp, int is_query,
                                 int score_kind /*0 L2, 1 IP, 2 cosine*/, __nv_bfloat16* __restrict__ out, float* __restrict__ alpha,
                                 float* __restrict__ beta, float* __restrict__ tile_nn) {
    constexpr bool kInt = sizeof(T) == 1;
    const int lane = threadIdx.x & 31;
    const uint64_t warp = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t r = warp; r < n; r += nwarps) {
        const T* row = reinterpret_cast<const T*>(rows + r * row_stride);
        __nv_bfloat16* o = out + r * kp;
        float nn = 0.0f;
        for (uint32_t d = lane; d < dim; d += 32) {
            const float x = elem_f32(row, d);
            nn = fmaf(x, x, nn);
            const __nv_bfloat16 hi = __float2bfloat16_rn(x);
            if constexpr (kInt) {
                o[d] = hi;
            } else {
                const __nv_bfloat16 lo = __float2bfloat16_rn(x - __bfloat162float(hi));
                o[d] = hi;
                o[dim + d] = is_query ? hi : lo;
                o[2 * dim + d] = is_query ? lo : hi;
            }
        }
        for (uint32_t d = (kInt ? dim : 3 * dim) + lane; d < kp; d += 32) o[d] = __float2bfloat16_rn(0.0f);
        if (!is_query) {
#pragma unroll
            for (int s = 16; s > 0; s >>= 1) nn += __shfl_xor_sync(0xFFFFFFFFu, nn, s);
            if (lane == 0) {
                if (score_kind == 0) {
                    alpha[r] = -2.0f;
                    beta[r] = nn;
                } else if (score_kind == 1) {
                    alpha[r] = -1.0f;
                    beta[r] = 0.0f;
                } else {
                    alpha[r] = nn > 0.0f ? -rsqrtf(nn) : 0.0f;
                    beta[r] = 0.0f;
                }
                // the largest fp32 ||b||^2 of the 128-row tile (certify_kernel); +inf marks a tile no query can be
                // certified against: a non-finite row, or a cosine row whose norm the exact kernel may take for zero
                const bool bad = !(nn <= 3.402823466e38f) || (score_kind == 2 && nn > 0.0f && nn < 0x1p-100f);
                atomicMax(reinterpret_cast<unsigned*>(tile_nn) + r / kBN, bad ? 0x7F800000u : __float_as_uint(nn));
            }
        }
    }
}

struct TcParams {
    uint32_t nq, n_base, kp;
    uint32_t tiles_per_split;  // 128-column tiles per base range
    uint32_t n_splits;
    const float* alpha;
    const float* beta;
    uint32_t* cand;            // [nq][n_splits][kKP]
    float* worst;              // [nq][n_splits]: the largest kept score, +inf when the range kept fewer than KP
};

template <int KP>
__global__ void __launch_bounds__(kTcThreads, 1)
flat_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const TcParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* sa = smem;                                                  // kStages x 16 KB
    uint8_t* sb = smem + kStages * kTileBytes;                           // kStages x 16 KB
    float* s_coef = reinterpret_cast<float*>(sb + kStages * kTileBytes);  // [alpha 128 | beta 128] of the current tile
    float* s_scores = s_coef + 2 * kBN;                                          // [128 query rows][33]: 32 scores per row
    float* s_cd = s_scores + 128 * 33;                                           // [KP][128]: candidate scores, entry-major (conflict-free)
    uint32_t* s_ci = reinterpret_cast<uint32_t*>(s_cd + KP * 128);               // [KP][128]: candidate ids
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_ci + KP * 128);               // offsets stay 8-byte aligned
    uint64_t* full = bars;                  // [kStages] TMA -> MMA
    uint64_t* empty = bars + kStages;       // [kStages] MMA -> TMA

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t m0 = blockIdx.y * kBM;
    const uint32_t split = blockIdx.x;
    const uint32_t n_tiles_total = (p.n_base + kBN - 1) / kBN;
    const uint32_t t0 = split * p.tiles_per_split, t1 = min(n_tiles_total, t0 + p.tiles_per_split);
    const uint32_t kblocks = p.kp / kBK;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) {
            mbar_init(full + s, 1);
            mbar_init(empty + s, 4);  // one arrival per consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
    }
    __syncthreads();

    if (warp == 4) {
        // ===== TMA producer (one lane) =====
        if (lane == 0) {
            uint32_t stage = 0, phase = 0;
            for (uint32_t t = t0; t < t1; ++t) {
                for (uint32_t kb = 0; kb < kblocks; ++kb) {
                    mbar_wait(empty + stage, phase ^ 1);
                    mbar_expect_tx(full + stage, 2 * kTileBytes);
                    tma_load_2d(&map_a, full + stage, sa + stage * kTileBytes, (int32_t)(kb * kBK), (int32_t)m0);
                    tma_load_2d(&map_b, full + stage, sb + stage * kTileBytes, (int32_t)(kb * kBK), (int32_t)(t * kBN));
                    if (++stage == kStages) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
    } else {
        // ===== consumer warpgroup: MMAs into registers, then the epilogue with one query row per thread =====
        const uint32_t row = threadIdx.x;  // 0..127: row of the 128-row tile this thread selects for
        const uint32_t q = m0 + row;
        float* my_scores = s_scores + row * 33;      // stride 33: conflict-free rows
        float* cd = s_cd + row;        // entry e of this thread: cd[e * 128]
        uint32_t* ci = s_ci + row;
        uint32_t cn = 0;
        float worst = -1.0f;   // largest kept score (valid when cn == KP)
        int worst_at = 0;
        float acc[2][64];      // rows [0, 64) and [64, 128) of the tile
        uint32_t stage = 0, phase = 0;
        for (uint32_t t = t0; t < t1; ++t) {
            {  // per-column score coefficients of this tile (the previous tile's readers passed the barriers below)
                const uint32_t col = t * kBN + row;
                s_coef[row] = col < p.n_base ? p.alpha[col] : 0.0f;
                s_coef[kBN + row] = col < p.n_base ? p.beta[col] : __int_as_float(0x7F800000);
            }
            for (uint32_t kb = 0; kb < kblocks; ++kb) {
                mbar_wait(full + stage, phase);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < kBK / 16; ++k) {
                    const uint64_t db = gmma_desc(sb + stage * kTileBytes, k * 32);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const uint64_t da = gmma_desc(sa + stage * kTileBytes + h * (kTileBytes / 2), k * 32);
                        wgmma_m64n128k16(acc[h], da, db, (kb | (uint32_t)k) != 0 ? 1u : 0u);
                    }
                }
                wgmma_commit();
                wgmma_wait_all();
                fence_operands(acc[0]);
                fence_operands(acc[1]);
                __syncwarp();
                if (lane == 0) mbar_arrive(empty + stage);  // this warp's MMAs have read the stage
                if (++stage == kStages) {
                    stage = 0;
                    phase ^= 1;
                }
            }
            asm volatile("bar.sync 1, 128;" ::: "memory");  // s_coef written by everyone
#pragma unroll
            for (int cc = 0; cc < kBN / 32; ++cc) {
                const int c0 = cc * 32;
                // the scores of columns [c0, c0 + 32) of this thread's accumulator fragment, into their rows' scratch
#pragma unroll
                for (int h = 0; h < 2; ++h) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
#pragma unroll
                        for (int r = 0; r < 4; ++r) {
                            const int fr = h * 64 + warp * 16 + (lane >> 2) + 8 * (r >> 1);
                            const int fc = 8 * j + 2 * (lane & 3) + (r & 1);
                            s_scores[fr * 33 + fc] = fmaf(acc[h][4 * (cc * 4 + j) + r], s_coef[c0 + fc], s_coef[kBN + c0 + fc]);
                        }
                    }
                }
                asm volatile("bar.sync 1, 128;" ::: "memory");
                // fast path, branch-free: a bit mask marks the scores that beat the current threshold (all of
                // them while the set fills)
                uint32_t mask = 0;
                const float thr = cn < (uint32_t)KP ? __int_as_float(0x7F800000) : worst;
#pragma unroll
                for (int j = 0; j < 32; ++j) mask |= my_scores[j] < thr ? (1u << j) : 0u;
                // slow path (rare once the threshold has settled): one candidate at a time
                while (mask) {
                    const int j = __ffs(mask) - 1;
                    mask &= mask - 1;
                    const float sc = my_scores[j];
                    const uint32_t id = t * kBN + c0 + j;
                    if (cn < (uint32_t)KP) {
                        cd[cn * 128] = sc;
                        ci[cn * 128] = id;
                        if (++cn < (uint32_t)KP) continue;
                    } else if (sc < worst) {
                        cd[worst_at * 128] = sc;
                        ci[worst_at * 128] = id;
                    } else {
                        continue;
                    }
                    // new threshold: the largest kept score (independent loads, then a max tree)
                    float v[KP];
#pragma unroll
                    for (int e = 0; e < KP; ++e) v[e] = cd[e * 128];
                    worst = v[0];
                    worst_at = 0;
#pragma unroll
                    for (int e = 1; e < KP; ++e)
                        if (v[e] > worst) worst = v[e], worst_at = e;
                }
                asm volatile("bar.sync 1, 128;" ::: "memory");  // scratch rows free for the next 32 columns
            }
        }
        if (q < p.nq) {
            uint32_t* out = p.cand + ((size_t)q * p.n_splits + split) * KP;
            for (uint32_t e = 0; e < (uint32_t)KP; ++e) out[e] = e < cn ? ci[e * 128] : kNoId;
            p.worst[(size_t)q * p.n_splits + split] = cn == (uint32_t)KP ? worst : __int_as_float(0x7F800000);
        }
    }
}

// exact distances of the candidates -> top-k by (distance, id); one warp per query
__global__ void __launch_bounds__(128) cand_topk_kernel(const uint32_t* __restrict__ cand, const float* __restrict__ dist, uint32_t nq, uint32_t c,
                                                        uint32_t k, uint32_t* __restrict__ out_ids, float* __restrict__ out_d) {
    extern __shared__ uint8_t sm[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    float* sd = reinterpret_cast<float*>(sm) + (size_t)wib * c;
    uint32_t* si = reinterpret_cast<uint32_t*>(reinterpret_cast<float*>(sm) + (size_t)(blockDim.x >> 5) * c) + (size_t)wib * c;
    const uint32_t q = blockIdx.x * (blockDim.x >> 5) + wib;
    if (q >= nq) return;
    for (uint32_t i = lane; i < c; i += 32) {
        const uint32_t id = cand[(size_t)q * c + i];
        const float d = dist[(size_t)q * c + i];
        si[i] = id;
        sd[i] = (id == kNoId || d != d) ? __int_as_float(0x7F800000) : d;  // NaN never enters (flat_topk_kernel)
        if (id != kNoId && d != d) si[i] = kNoId;
    }
    __syncwarp();
    for (uint32_t r = 0; r < k; ++r) {
        float bd = __int_as_float(0x7F800000);
        uint32_t bi = kNoId, bp = 0xFFFFFFFFu;
        for (uint32_t i = lane; i < c; i += 32) {
            const float d = sd[i];
            const uint32_t id = si[i];
            if (id != kNoId && (d < bd || (d == bd && id < bi))) bd = d, bi = id, bp = i;
        }
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) {
            const float od = __shfl_xor_sync(0xFFFFFFFFu, bd, s);
            const uint32_t oi = __shfl_xor_sync(0xFFFFFFFFu, bi, s), op = __shfl_xor_sync(0xFFFFFFFFu, bp, s);
            if (oi != kNoId && (bi == kNoId || od < bd || (od == bd && oi < bi))) bd = od, bi = oi, bp = op;
        }
        if (lane == 0) {
            out_ids[(size_t)q * k + r] = bi;
            out_d[(size_t)q * k + r] = bi == kNoId ? __int_as_float(0x7F800000) : bd;
            if (bp != 0xFFFFFFFFu) si[bp] = kNoId;
        }
        __syncwarp();
    }
}

__device__ __forceinline__ double gamma_n(double n, double v) { return n * v / (1.0 - n * v); }

// One warp per query: is the candidate top-k provably the exact one?  (E: see the header comment.)  Queries that are
// not certified are appended to redo[1..], redo[0] counting them.  kind: 0 L2, 1 IP, 2 float CosineNormalized,
// 3 cosine (-q.b / ||b||).
template <typename T>
__global__ void __launch_bounds__(128) certify_kernel(const uint8_t* __restrict__ queries, uint32_t nq, uint32_t dim, uint32_t kp, int kind,
                                                      const float* __restrict__ top_d, uint32_t k, const float* __restrict__ worst,
                                                      uint32_t n_splits, const float* __restrict__ tile_nn, uint32_t n_tiles,
                                                      uint32_t tiles_per_split, uint32_t* __restrict__ redo) {
    constexpr bool kInt = sizeof(T) == 1;
    const int lane = threadIdx.x & 31;
    const uint32_t q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (q >= nq) return;
    const T* row = reinterpret_cast<const T*>(queries + (size_t)q * dim * sizeof(T));
    double qq = 0.0;
    for (uint32_t d = lane; d < dim; d += 32) {
        const double x = elem_f32(row, d);
        qq += x * x;
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) qq += __shfl_xor_sync(0xFFFFFFFFu, qq, s);
    qq *= 1.0 + dim * 0x1p-52;  // the double sum (of exact squares), rounded up
    const double u = 0x1p-24, g_dim = gamma_n(dim, u), g_ex = gamma_n(dim + 2.0, u), g_kp = gamma_n(kp, 0x1p-23);
    const double qn = sqrt(qq) * (1.0 + 0x1p-50);
    const double dk = top_d[(size_t)q * k + k - 1];
    bool ok = isfinite(qq) && (kind != 3 || qq >= 0x1p-100);
    for (uint32_t i = lane; i < k; i += 32) ok = ok && isfinite(top_d[(size_t)q * k + i]);
    for (uint32_t r = lane; r < n_splits && ok; r += 32) {
        double b2 = 0.0;
        for (uint32_t t = r * tiles_per_split; t < min(n_tiles, (r + 1) * tiles_per_split); ++t) b2 = fmax(b2, (double)tile_nn[t]);
        b2 = (b2 + dim * 0x1p-149) / (1.0 - g_dim);  // bounds every exact ||b||^2 of the range
        const double B = sqrt(b2) * (1.0 + 0x1p-50);
        const float wf = worst[(size_t)q * n_splits + r];
        const double w = wf == __int_as_float(0x7F800000) ? 3.402823466e38 : (double)wf;
        // relative error of the dot per ||q|| ||b||, and its absolute floor
        const double e = kInt ? (qn * B < 0x1p24 ? 0.0 : 1.03 * g_kp) : 0x1p-14 + 1.03 * g_kp;
        const double e_abs = kInt ? 0.0 : kp * 0x1p-125 * (qn + B + 1.0);
        const double e_dot = e * qn * B + e_abs;
        double lb;
        if (kind == 0) {
            lb = (qq + w - 1.01 * (2.0 * e_dot + (g_dim + 2.0 * u) * (b2 + 2.0 * qn * B))) * (1.0 - g_ex);
        } else if (kind == 1) {
            lb = w - 1.01 * (e_dot + g_dim * qn * B);
        } else if (kind == 2) {
            const double x = 1.0 + w - 1.01 * (e_dot + g_dim * qn * B);
            lb = x - 2.0 * u * fabs(x);
        } else {
            const double rho = 0x1p-22 + g_dim + u;
            const double ec = qn * ((e + 1.0) * rho + e) + (kInt ? 0.0 : kp * 0x1p-70 * (qn + 1.0));
            lb = 1.0 + (w - 1.01 * ec) / qn - 1.01 * (2.0 * g_dim + 7.0 * u);
        }
        ok = isfinite(b2) && qq + b2 + 2.0 * qn * B < 0x1p120 && lb > dk;
    }
    ok = __all_sync(0xFFFFFFFFu, ok);
    if (lane == 0 && !ok) redo[1 + atomicAdd(redo, 1u)] = q;
}

// the raw rows of the queries listed in redo[1..], packed in list order (one block per query)
__global__ void gather_rows_kernel(const uint8_t* __restrict__ src, size_t row_bytes, const uint32_t* __restrict__ redo, uint8_t* __restrict__ dst) {
    const uint8_t* s = src + (size_t)redo[1 + blockIdx.x] * row_bytes;
    uint8_t* d = dst + (size_t)blockIdx.x * row_bytes;
    for (size_t b = threadIdx.x; b < row_bytes; b += blockDim.x) d[b] = s[b];
}

// their exact top-k lists back into the rows of the whole batch
__global__ void scatter_topk_kernel(const uint32_t* __restrict__ redo, uint32_t k, const uint32_t* __restrict__ ids, const float* __restrict__ d,
                                    uint32_t* __restrict__ out_ids, float* __restrict__ out_d) {
    const size_t q = redo[1 + blockIdx.x];
    for (uint32_t i = threadIdx.x; i < k; i += blockDim.x) {
        out_ids[q * k + i] = ids[(size_t)blockIdx.x * k + i];
        out_d[q * k + i] = d[(size_t)blockIdx.x * k + i];
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int make_map(CUtensorMap* map, void* base, uint64_t rows, uint32_t kp) {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) != cudaSuccess || !p)
            return fail(DAB_ERR_CUDA, "flat_tc: cuTensorMapEncodeTiled is not available from this driver");
        fn = (EncodeTiledFn)p;
    }
    const cuuint64_t dims[2] = {kp, rows};
    const cuuint64_t strides[1] = {(cuuint64_t)kp * 2};
    const cuuint32_t box[2] = {(cuuint32_t)kBK, (cuuint32_t)kBM};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(DAB_ERR_CUDA, "flat_tc: cuTensorMapEncodeTiled failed (%d)", (int)r);
    return DAB_OK;
}

template <typename... A>
void launch_prep(int dtype, int grid, cudaStream_t st, A... a) {
    switch (dtype) {
        case DAB_F32: prep_bf16_kernel<float><<<grid, 256, 0, st>>>(a...); break;
        case DAB_F16: prep_bf16_kernel<__half><<<grid, 256, 0, st>>>(a...); break;
        case DAB_I8: prep_bf16_kernel<int8_t><<<grid, 256, 0, st>>>(a...); break;
        default: prep_bf16_kernel<uint8_t><<<grid, 256, 0, st>>>(a...); break;
    }
}

template <typename... A>
void launch_certify(int dtype, int grid, cudaStream_t st, A... a) {
    switch (dtype) {
        case DAB_F32: certify_kernel<float><<<grid, 128, 0, st>>>(a...); break;
        case DAB_F16: certify_kernel<__half><<<grid, 128, 0, st>>>(a...); break;
        case DAB_I8: certify_kernel<int8_t><<<grid, 128, 0, st>>>(a...); break;
        default: certify_kernel<uint8_t><<<grid, 128, 0, st>>>(a...); break;
    }
}

}  // namespace

void tc_release(dab_index* idx) {
    cudaFree(idx->d_tc_base);
    cudaFree(idx->d_tc_coef);
    idx->d_tc_base = nullptr;
    idx->d_tc_coef = nullptr;
}

}  // namespace dab

using namespace dab;

extern "C" {

int dab_flat_knn_tc(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t* out_ids, float* out_dists) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_flat_knn_tc: idx is NULL");
    if (!idx->vectors_ready) return fail(DAB_ERR_NOT_READY, "dab_flat_knn_tc: vectors not uploaded");
    if (nq == 0) return DAB_OK;
    if (!queries || !out_ids || !out_dists) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_flat_knn_tc: NULL argument");
    if (k == 0 || k + 8 > (uint32_t)kKP) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_flat_knn_tc: k must be in [1, %d] (use dab_flat_knn beyond)", kKP - 8);
    DAB_CUDA(cudaSetDevice(idx->device));
    cudaStream_t st = idx->stream;
    const bool is_int = idx->dtype == DAB_I8 || idx->dtype == DAB_U8;
    const uint32_t dim = idx->dim;
    const uint32_t kp = (uint32_t)round_up((size_t)(is_int ? dim : 3 * dim), kBK);
    const uint64_t n = idx->n_points;  // start points are not data
    const int score_kind = idx->metric == DAB_L2 ? 0 : idx->metric == DAB_COSINE ? 2 : (is_int && idx->metric == DAB_COSINE_NORMALIZED) ? 2 : 1;
    const int cert_kind = score_kind == 0 ? 0 : score_kind == 2 ? 3 : idx->metric == DAB_INNER_PRODUCT ? 1 : 2;
    // geometry: queries padded to whole 128-row tiles; base ranges: enough CTAs to fill the machine, whole 128-column
    // tiles each (at most 48 ranges: the exact re-scoring handles splits x kKP candidates per query)
    const uint32_t m_tiles = (nq + kBM - 1) / kBM;
    const uint32_t n_tiles = (uint32_t)((n + kBN - 1) / kBN);
    uint32_t splits = std::max<uint32_t>(1, std::min<uint32_t>(std::min<uint32_t>(n_tiles, 48), (uint32_t)(idx->sm_count * 2 + m_tiles - 1) / m_tiles));
    const uint32_t tiles_per_split = (n_tiles + splits - 1) / splits;
    splits = (n_tiles + tiles_per_split - 1) / tiles_per_split;
    const uint32_t kp_sel = k <= 10 ? 16u : (uint32_t)kKP;  // per-range candidates: k plus slack for the approximate scores
    const uint32_t c = splits * kp_sel;
    const size_t tsmem = (size_t)4 * c * 8;
    if (tsmem > 200 * 1024) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_flat_knn_tc: %u candidates per query do not fit the selection kernel", c);
    int rc;
    // base operand (bf16 split rows + score coefficients + per-tile norm bounds): built once per uploaded snapshot
    if (!idx->d_tc_base || idx->tc_version != idx->vectors_version) {
        tc_release(idx);
        DAB_CUDA(cudaMalloc(&idx->d_tc_base, n * (size_t)kp * 2));
        DAB_CUDA(cudaMalloc(&idx->d_tc_coef, (n * 2 + n_tiles) * sizeof(float)));
        DAB_CUDA(cudaMemsetAsync((float*)idx->d_tc_coef + 2 * n, 0, n_tiles * sizeof(float), st));
        launch_prep(idx->dtype, idx->sm_count * 8, st, (const uint8_t*)idx->d_vectors, idx->row_stride, n, dim, kp, 0, score_kind,
                    (__nv_bfloat16*)idx->d_tc_base, (float*)idx->d_tc_coef, (float*)idx->d_tc_coef + n, (float*)idx->d_tc_coef + 2 * n);
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
        idx->tc_version = idx->vectors_version;
    }
    // queries: raw copy (exact re-scoring) + bf16 operand
    const size_t qrow = (size_t)dim * elem_size(idx->dtype);
    const size_t qraw = (size_t)nq * qrow;
    const size_t qop = (size_t)m_tiles * kBM * kp * 2;
    if ((rc = idx->s_queries.reserve(round_up(qraw, 256) + qop))) return rc;
    uint8_t* d_qraw = (uint8_t*)idx->s_queries.p;
    __nv_bfloat16* d_qop = (__nv_bfloat16*)(d_qraw + round_up(qraw, 256));
    DAB_CUDA(cudaMemcpyAsync(d_qraw, queries, qraw, cudaMemcpyHostToDevice, st));
    DAB_CUDA(cudaMemsetAsync(d_qop, 0, qop, st));
    launch_prep(idx->dtype, idx->sm_count * 4, st, (const uint8_t*)d_qraw, qrow, (uint64_t)nq, dim, kp, 1, score_kind, d_qop, (float*)nullptr,
                (float*)nullptr, (float*)nullptr);
    DAB_LAUNCHED();
    // s_ids: [candidates nq x c | W nq x splits | redo: count, query ids | redo queries' rows | their exact top-k]
    const size_t o_worst = round_up((size_t)nq * c * 4, 256), o_redo = o_worst + round_up((size_t)nq * splits * 4, 256);
    const size_t o_rows = o_redo + round_up(((size_t)nq + 1) * 4, 256), o_top = o_rows + round_up(qraw, 256);
    if ((rc = idx->s_ids.reserve(o_top + (size_t)nq * k * 8))) return rc;
    if ((rc = idx->s_out2.reserve((size_t)nq * c * 4))) return rc;
    if ((rc = idx->s_out.reserve((size_t)nq * k * 8))) return rc;
    uint8_t* ids_base = (uint8_t*)idx->s_ids.p;
    uint32_t* d_cand = (uint32_t*)ids_base;
    float* d_worst = (float*)(ids_base + o_worst);
    uint32_t* d_redo = (uint32_t*)(ids_base + o_redo);
    CUtensorMap map_a, map_b;
    if ((rc = make_map(&map_a, d_qop, (uint64_t)m_tiles * kBM, kp))) return rc;
    if ((rc = make_map(&map_b, idx->d_tc_base, n, kp))) return rc;
    TcParams p;
    p.nq = nq;
    p.n_base = (uint32_t)n;
    p.kp = kp;
    p.tiles_per_split = tiles_per_split;
    p.n_splits = splits;
    p.alpha = (const float*)idx->d_tc_coef;
    p.beta = (const float*)idx->d_tc_coef + n;
    p.cand = d_cand;
    p.worst = d_worst;
    const size_t smem = 1024 + 2 * (size_t)kStages * kTileBytes + 2 * kBN * 4 + 128 * 33 * 4 + 2 * (size_t)kp_sel * 128 * 4 + 2 * (size_t)kStages * 8;
    auto kern = kp_sel == 16 ? flat_tc_kernel<16> : flat_tc_kernel<32>;
    DAB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<dim3(splits, m_tiles), kTcThreads, smem, st>>>(map_a, map_b, p);
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    // exact distances of the candidates in the reference's SIMD order, then the final top-k
    if ((rc = launch_frontier(idx, d_qraw, nq, d_cand, c, (float*)idx->s_out2.p))) return rc;
    uint32_t* d_top_ids = (uint32_t*)idx->s_out.p;
    float* d_top_d = (float*)(d_top_ids + (size_t)nq * k);
    DAB_CUDA(cudaFuncSetAttribute(cand_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tsmem));
    cand_topk_kernel<<<(nq + 3) / 4, 128, tsmem, st>>>(d_cand, (const float*)idx->s_out2.p, nq, c, k, d_top_ids, d_top_d);
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    // certify every query; the others go through the exact scan
    DAB_CUDA(cudaMemsetAsync(d_redo, 0, 4, st));
    launch_certify(idx->dtype, (nq + 3) / 4, st, (const uint8_t*)d_qraw, nq, dim, kp, cert_kind, (const float*)d_top_d, k, (const float*)d_worst,
                   splits, (const float*)idx->d_tc_coef + 2 * n, n_tiles, tiles_per_split, d_redo);
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    uint32_t n_redo = 0;
    DAB_CUDA(cudaMemcpyAsync(&n_redo, d_redo, 4, cudaMemcpyDeviceToHost, st));
    DAB_CUDA(cudaStreamSynchronize(st));
    if (n_redo) {
        uint8_t* d_rows = ids_base + o_rows;
        uint32_t* d_redo_ids = (uint32_t*)(ids_base + o_top);
        float* d_redo_d = (float*)(d_redo_ids + (size_t)n_redo * k);
        gather_rows_kernel<<<n_redo, 128, 0, st>>>(d_qraw, qrow, d_redo, d_rows);
        DAB_LAUNCHED();
        if ((rc = flat_knn_device(idx, d_rows, n_redo, k, d_redo_ids, d_redo_d))) return rc;
        scatter_topk_kernel<<<n_redo, 32, 0, st>>>(d_redo, k, d_redo_ids, d_redo_d, d_top_ids, d_top_d);
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
    }
    DAB_CUDA(cudaMemcpyAsync(out_ids, d_top_ids, (size_t)nq * k * 4, cudaMemcpyDeviceToHost, st));
    DAB_CUDA(cudaMemcpyAsync(out_dists, d_top_d, (size_t)nq * k * 4, cudaMemcpyDeviceToHost, st));
    DAB_CUDA(cudaStreamSynchronize(st));
    return DAB_OK;
}

}  // extern "C"
