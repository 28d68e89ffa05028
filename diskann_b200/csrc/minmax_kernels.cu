// minmax_kernels.cu — the MinMax quantizer (diskann-quantization/src/minmax): per-vector N-bit compression with the
// compensation coefficients in front of the codes, and the distances between two compressed vectors.
//
//   * MinMaxQuantizer::compress (quantizer.rs:153-228, get_range :117-151, Transform::Null) is scalar and sequential in the
//     reference: a min / max fold (for one bit: the means of the values below / not below the mean), then one pass that
//     rounds every value to its code and accumulates norm_squared, code_sum and the loss in index order.  Here one lane
//     owns one vector and runs exactly those chains; a warp takes 32 vectors at a time and moves them through a
//     [32][33] shared-memory tile so the global reads are coalesced (row-major in, column access conflict-free), and
//     the 32 finished rows leave through shared memory as one contiguous byte range.
//   * MinMax{IP, L2Squared, Cosine, CosineNormalized} over two Data rows (vectors.rs:206-455): an exact integer inner
//     product of the codes (bits/distances.rs; dp4a on masked fields, popc for one bit) and a five-term f32 epilogue
//     in the reference's association.  Eight lanes per pair, 4-byte loads of the dense codes.
// The quantizer runs on Transform::Null input, or behind a Hadamard transform (transform_kernels.cu writes the
// transformed rows into device memory and these kernels run on them unchanged, dim = the transform's output dim).
// Row layout = the reference's canonical-front Data<NBITS> (meta/vector.rs:377-392): MinMaxCompensation {dim u32, b, n, a,
// norm_squared} (vectors.rs:43-52, 20 bytes) then ceil(dim * NBITS / 8) bytes of codes, value i at bit i * NBITS.
// HBM-bound byte work: no tensor cores.
#include "dab_common.cuh"
#include "minmax.cuh"
#include "quant_device.cuh"
#include "transform.cuh"

#include <algorithm>

namespace dab {

// `walk(f)` calls f(i, v_i) for i = 0 .. dim-1 in index order on the lane's own vector, the warp moving 32 x 32 tiles
// through shared memory (all lanes must call it together).
template <typename F>
__device__ __forceinline__ void walk_rows(const MinMaxCompressParams& p, uint64_t v0, float (*tile)[33], int lane, F&& f) {
    for (uint32_t t0 = 0; t0 < p.dim; t0 += 32) {
        __syncwarp();
#pragma unroll 4
        for (int r = 0; r < 32; ++r) {
            const uint64_t v = v0 + r;
            tile[r][lane] = (v < p.n && t0 + lane < p.dim) ? __ldg(p.vectors + v * p.dim + t0 + lane) : 0.0f;
        }
        __syncwarp();
        const uint32_t m = min(32u, p.dim - t0);
        for (uint32_t j = 0; j < m; ++j) f(t0 + j, tile[lane][j]);
    }
}

__global__ void __launch_bounds__(128) minmax_compress_kernel(const MinMaxCompressParams p) {
    extern __shared__ __align__(16) uint8_t mm_smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    uint8_t* base = mm_smem + (size_t)wib * p.warp_smem;
    float (*tile)[33] = reinterpret_cast<float (*)[33]>(base);
    uint8_t* srows = base + 32 * 33 * 4;
    uint8_t* mine = srows + (size_t)lane * p.srow_stride;
    const uint32_t warps = gridDim.x * (blockDim.x >> 5);
    const float domain_max = (float)((1u << p.nbits) - 1u);
    const uint32_t code_bytes = p.row_bytes - kMmMeta;

    for (uint64_t v0 = ((uint64_t)blockIdx.x * (blockDim.x >> 5) + wib) * 32; v0 < p.n; v0 += (uint64_t)warps * 32) {
        // ---- get_range (quantizer.rs:117-151)
        float mn, mx;
        if (p.nbits == 1) {
            float sum = -0.0f;  // <f32 as Sum>::sum folds from -0.0
            walk_rows(p, v0, tile, lane, [&](uint32_t, float e) { sum = __fadd_rn(sum, e); });
            const float mean = __fdiv_rn(sum, (float)p.dim);
            float a = 0.0f, ac = 0.0f, b = 0.0f, bc = 0.0f;
            walk_rows(p, v0, tile, lane, [&](uint32_t, float e) {
                const float m = e < mean ? 1.0f : 0.0f;
                a = __fadd_rn(a, __fmul_rn(m, e));
                ac = __fadd_rn(ac, m);
                b = __fadd_rn(b, __fmul_rn(__fsub_rn(1.0f, m), e));
                bc = __fadd_rn(bc, __fsub_rn(1.0f, m));
            });
            mn = fminf(__fdiv_rn(a, ac), mean);  // f32::min / max: the other operand when one is NaN (fminf / fmaxf do the same)
            mx = fmaxf(__fdiv_rn(b, bc), mean);
        } else {
            mn = mx = __int_as_float(0x7FC00000);
            walk_rows(p, v0, tile, lane, [&](uint32_t, float e) {
                mn = fminf(mn, e);
                mx = fmaxf(mx, e);
            });
        }
        const float width = __fdiv_rn(__fsub_rn(mx, mn), 2.0f);
        const float mid = __fadd_rn(mn, width);
        const float lo = __fsub_rn(mid, __fmul_rn(width, p.grid_scale));
        const float hi = __fadd_rn(mid, __fmul_rn(width, p.grid_scale));
        const float inverse_scale = __fdiv_rn(fmaxf(__fsub_rn(hi, lo), 1e-8f), domain_max);

        // ---- codes + the three sequential sums (quantizer.rs:186-209); codes packed value i at bit i * nbits
        for (uint32_t w = 0; w < (code_bytes + 3) / 4; ++w) reinterpret_cast<uint32_t*>(mine + kMmMeta)[w] = 0;  // (stays inside the lane's stride)
        float norm_squared = 0.0f, code_sum = 0.0f, loss = 0.0f;
        bool nan = false;
        const int nbits = p.nbits;
        walk_rows(p, v0, tile, lane, [&](uint32_t i, float e) {
            nan |= e != e;
            const float t = __fdiv_rn(__fsub_rn(e, lo), inverse_scale);
            float code = t != t ? t : (t < 0.0f ? 0.0f : (t > domain_max ? domain_max : t));  // f32::clamp keeps NaN
            code = roundf(code);                                                              // half away from zero
            const float vr = __fadd_rn(__fmul_rn(code, inverse_scale), lo);
            norm_squared = __fadd_rn(norm_squared, __fmul_rn(vr, vr));
            code_sum = __fadd_rn(code_sum, code);
            const float d = __fsub_rn(vr, e);
            loss = __fadd_rn(loss, __fmul_rn(d, d));
            const uint32_t c = code != code ? 0u : (uint32_t)code;  // `as u8`: NaN -> 0
            const uint32_t bit = i * (uint32_t)nbits;
            mine[kMmMeta + (bit >> 3)] |= (uint8_t)(c << (bit & 7u));
        });
        {   // MinMaxCompensation {dim, b, n, a, norm_squared}
            uint32_t* mw = reinterpret_cast<uint32_t*>(mine);
            mw[0] = p.dim;
            mw[1] = __float_as_uint(lo);
            mw[2] = __float_as_uint(__fmul_rn(inverse_scale, code_sum));
            mw[3] = __float_as_uint(inverse_scale);
            mw[4] = __float_as_uint(norm_squared);
        }
        const uint64_t v = v0 + lane;
        if (v < p.n) {
            if (p.loss) p.loss[v] = loss;
            if (nan) atomicMin(p.first_nan, (unsigned long long)v);
        }
        __syncwarp();
        // ---- the 32 rows of the warp are one contiguous byte range of the output
        const uint64_t nrows = min((uint64_t)32, p.n - v0);
        for (uint32_t r = 0; r < nrows; ++r) {
            const uint8_t* src = srows + (size_t)r * p.srow_stride;
            uint8_t* dst = p.rows + (v0 + r) * p.row_bytes;
            for (uint32_t bb = lane; bb < p.row_bytes; bb += 32) dst[bb] = src[bb];
        }
        __syncwarp();
    }
}

struct MinMaxDistanceParams {
    int metric, nbits_x, nbits_y;
    uint32_t dim;
    const uint8_t* x;
    const uint8_t* y;
    uint32_t row_bytes_x, row_bytes_y;
    uint64_t n;
    float* out;
};

__device__ __forceinline__ uint32_t mm_code_at(const uint8_t* codes, uint32_t i, int nbits) {
    const uint32_t bit = i * (uint32_t)nbits;
    return ((uint32_t)__ldg(codes + (bit >> 3)) >> (bit & 7u)) & ((1u << nbits) - 1u);
}

// eight lanes per pair, four pairs per warp pass (rows are 36 - 150 bytes at 128 dimensions: a whole warp per pair would
// leave most lanes without a word to load)
__global__ void __launch_bounds__(256) minmax_distance_kernel(const MinMaxDistanceParams p) {
    const int lane = threadIdx.x & 31, team = lane >> 3, tl = lane & 7;
    const uint64_t warp = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
    const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const bool words = p.nbits_x == p.nbits_y && (p.row_bytes_x & 3u) == 0 && (p.row_bytes_y & 3u) == 0;
    for (uint64_t i0 = warp * 4; i0 < p.n; i0 += nwarps * 4) {
        const uint64_t i = i0 + team;
        const bool live = i < p.n;
        const uint8_t* xr = p.x + (live ? i : i0) * p.row_bytes_x;
        const uint8_t* yr = p.y + (live ? i : i0) * p.row_bytes_y;
        uint32_t ip = 0, unused = 0;
        if (words) {
            // same width on both sides: whole 32-bit words of the dense codes (padding bits are zero)
            const uint32_t* xw = reinterpret_cast<const uint32_t*>(xr + kMmMeta);
            const uint32_t* yw = reinterpret_cast<const uint32_t*>(yr + kMmMeta);
            const uint32_t nw = (p.row_bytes_x - kMmMeta) >> 2;
            for (uint32_t w = tl; w < nw; w += 8) {
                const uint32_t a = __ldg(xw + w), b = __ldg(yw + w);
                switch (p.nbits_x) {
                    case 8: sq_word<8>(a, b, true, unused, ip); break;
                    case 4: sq_word<4>(a, b, true, unused, ip); break;
                    case 2: sq_word<2>(a, b, true, unused, ip); break;
                    default: sq_word<1>(a, b, true, unused, ip); break;
                }
            }
        } else {
            for (uint32_t e = tl; e < p.dim; e += 8) ip += mm_code_at(xr + kMmMeta, e, p.nbits_x) * mm_code_at(yr + kMmMeta, e, p.nbits_y);
        }
        ip += __shfl_xor_sync(kFull, ip, 4);
        ip += __shfl_xor_sync(kFull, ip, 2);
        ip += __shfl_xor_sync(kFull, ip, 1);
        if (tl == 0 && live) {
            const uint32_t* xm = reinterpret_cast<const uint32_t*>(xr);  // rows are at least 4-byte aligned only when
            const uint32_t* ym = reinterpret_cast<const uint32_t*>(yr);  // row_bytes % 4 == 0: read the meta bytewise otherwise
            float xb, xn, xa, xq, yb, yn, ya, yq;
            uint32_t dx, dy;
            if (((p.row_bytes_x | p.row_bytes_y) & 3u) == 0) {
                dx = xm[0], xb = __uint_as_float(xm[1]), xn = __uint_as_float(xm[2]), xa = __uint_as_float(xm[3]), xq = __uint_as_float(xm[4]);
                dy = ym[0], yb = __uint_as_float(ym[1]), yn = __uint_as_float(ym[2]), ya = __uint_as_float(ym[3]), yq = __uint_as_float(ym[4]);
            } else {
                auto rd = [](const uint8_t* q) { return (uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | ((uint32_t)q[3] << 24); };
                dx = rd(xr), xb = __uint_as_float(rd(xr + 4)), xn = __uint_as_float(rd(xr + 8)), xa = __uint_as_float(rd(xr + 12)), xq = __uint_as_float(rd(xr + 16));
                dy = rd(yr), yb = __uint_as_float(rd(yr + 4)), yn = __uint_as_float(rd(yr + 8)), ya = __uint_as_float(rd(yr + 12)), yq = __uint_as_float(rd(yr + 16));
            }
            float r;
            if (dx != dy || dx != p.dim) {
                r = __int_as_float(0x7FC00000);  // UnequalLengths
            } else {
                r = minmax_finish(p.metric, ip, dx, xb, xn, xa, xq, yb, yn, ya, yq);
            }
            p.out[i] = r;
        }
    }
}

// ---------------------------------------------------------------- full-precision query x compressed rows
// MinMax{IP, L2Squared, Cosine, CosineNormalized}::evaluate(FullQueryRef, DataRef<NBITS>) (vectors.rs:272-305, 347-392,
// 417-476): raw = InnerProduct(&[f32], BitSlice<NBITS>) — the x86-64-v3 kernels of bits/distances.rs for 1 / 2 / 4 bits
// (:2295-2436, :2438-2595, :2603-2665: eight f32 lanes, FMA, one or two accumulators, zero-filled remainder loads,
// sum_tree), the scalar mul-then-add loop for 8 bits (:2668-2725) — then ip = raw * a + sum(q) * b and the metric's
// epilogue.  A team of eight GPU lanes is the eight SIMD lanes of the reference (every lane runs its own FMA chain, the
// tree is xor 4, 2, 1), four (query, row) pairs per warp; for 8 bits one lane per pair runs the sequential chain.
struct MinMaxQueryParams {
    int metric, nbits;
    uint32_t dim;
    const float* queries;  // [nq][dim]
    uint32_t nq;
    const uint8_t* rows;   // [n][row_bytes]
    uint32_t row_bytes;
    uint64_t n;
    float* meta;           // [nq][2]: sum, norm_squared (FullQueryMeta)
    float* out;            // [nq][n]
    unsigned long long* first_nan;
};

// CompressInto<&[f32], FullQueryMut> (quantizer.rs:393-417): sequential sums; NaN input is an error
__global__ void __launch_bounds__(128) minmax_query_meta_kernel(const MinMaxQueryParams p) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= p.nq) return;
    const float* v = p.queries + (size_t)q * p.dim;
    float ns = -0.0f, s = -0.0f;  // <f32 as Sum>::sum folds from -0.0
    bool nan = false;
    for (uint32_t i = 0; i < p.dim; ++i) {
        const float e = v[i];
        nan |= e != e;
        ns = __fadd_rn(ns, __fmul_rn(e, e));
        s = __fadd_rn(s, e);
    }
    p.meta[2 * q] = s;
    p.meta[2 * q + 1] = ns;
    if (nan) atomicMin(p.first_nan, (unsigned long long)q);
}

__device__ __forceinline__ uint32_t mm_load_bytes(const uint8_t* ptr, uint32_t nbytes) {
    uint32_t v = 0;
    for (uint32_t i = 0; i < nbytes; ++i) v |= (uint32_t)__ldg(ptr + i) << (8 * i);
    return v;
}

template <int NBITS>
__global__ void __launch_bounds__(256) minmax_query_distance_kernel(const MinMaxQueryParams p) {
    extern __shared__ float mq[];  // the query
    const uint32_t q = blockIdx.y;
    for (uint32_t e = threadIdx.x; e < p.dim; e += blockDim.x) mq[e] = __ldg(p.queries + (size_t)q * p.dim + e);
    __syncthreads();
    const float q_sum = p.meta[2 * q], q_ns = p.meta[2 * q + 1];
    const uint32_t len = p.dim;
    const int lane = threadIdx.x & 31;
    constexpr int LPP = NBITS == 8 ? 1 : 8;  // lanes per pair
    const int l = lane % LPP;
    const uint64_t pair0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / LPP;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x / LPP;
    const uint64_t rounds = (p.n + stride - 1) / stride;  // every lane makes the same number of passes (team shuffles)
    for (uint64_t it = 0; it < rounds; ++it) {
        const uint64_t r = pair0 + it * stride;
        const bool live = r < p.n;
        const uint8_t* row = p.rows + (live ? r : 0) * p.row_bytes;
        const uint8_t* codes = row + kMmMeta;
        float raw;
        if (NBITS == 8) {
            float s = 0.0f;
            for (uint32_t i = 0; i < len; ++i) s = __fadd_rn(s, __fmul_rn(mq[i], (float)__ldg(codes + i)));
            raw = s;
        } else {
            float s = 0.0f;
            const uint32_t tail = (len & 7u) == 0 ? 8u : (len & 7u);
            if (NBITS == 4) {
                const uint32_t blocks = len / 8;
                for (uint32_t b = 0; b < blocks; ++b) {
                    const uint32_t w = mm_load_bytes(codes + 4 * b, 4);
                    s = __fmaf_rn(mq[8 * b + l], (float)((w >> (4 * l)) & 15u), s);
                }
                const uint32_t rem = len & 7u;
                if (rem) {
                    const uint32_t w = mm_load_bytes(codes + 4 * blocks, (rem + 1) / 2);
                    s = __fmaf_rn((uint32_t)l < rem ? mq[8 * blocks + l] : 0.0f, (float)((w >> (4 * l)) & 15u), s);
                }
            } else if (NBITS == 2) {
                const uint32_t blocks = len / 16;
                if (blocks) {
                    float s0 = 0.0f, s1 = 0.0f;
                    for (uint32_t b = 0; b < blocks; ++b) {
                        const uint32_t w = mm_load_bytes(codes + 4 * b, 4);
                        s0 = __fmaf_rn(mq[16 * b + l], (float)((w >> (2 * l)) & 3u), s0);
                        s1 = __fmaf_rn(mq[16 * b + 8 + l], (float)((w >> (16 + 2 * l)) & 3u), s1);
                    }
                    s = __fadd_rn(s0, s1);
                }
                const uint32_t rem = len & 15u;
                if (rem) {
                    const uint32_t w = mm_load_bytes(codes + 4 * blocks, (rem + 3) / 4);
                    const float* px = mq + 16 * blocks;
                    if (rem <= 8) {
                        s = __fmaf_rn((uint32_t)l < tail ? px[l] : 0.0f, (float)((w >> (2 * l)) & 3u), s);
                    } else {
                        s = __fmaf_rn(px[l], (float)((w >> (2 * l)) & 3u), s);
                        s = __fmaf_rn((uint32_t)l < tail ? px[8 + l] : 0.0f, (float)((w >> (16 + 2 * l)) & 3u), s);
                    }
                }
            } else {
                const uint32_t blocks = len / 32;
                if (blocks) {
                    float s0 = 0.0f, s1 = 0.0f;
                    for (uint32_t b = 0; b < blocks; ++b) {
                        const uint32_t w = mm_load_bytes(codes + 4 * b, 4);
                        s0 = __fmaf_rn(mq[32 * b + l], (float)((w >> l) & 1u), s0);
                        s1 = __fmaf_rn(mq[32 * b + 8 + l], (float)((w >> (8 + l)) & 1u), s1);
                        s0 = __fmaf_rn(mq[32 * b + 16 + l], (float)((w >> (16 + l)) & 1u), s0);
                        s1 = __fmaf_rn(mq[32 * b + 24 + l], (float)((w >> (24 + l)) & 1u), s1);
                    }
                    s = __fadd_rn(s0, s1);
                }
                const uint32_t rem = len & 31u;
                if (rem) {
                    const uint32_t groups = (rem + 7) / 8;
                    const uint32_t w = mm_load_bytes(codes + 4 * blocks, groups);
                    const float* px = mq + 32 * blocks;
                    for (uint32_t j = 0; j < groups; ++j) {
                        const bool in = j + 1 < groups || (uint32_t)l < tail;
                        s = __fmaf_rn(in ? px[8 * j + l] : 0.0f, (float)((w >> (8 * j + l)) & 1u), s);
                    }
                }
            }
            // sum_tree (diskann-wide/src/traits.rs:583-595) over the team's eight lanes
            s = __fadd_rn(s, __shfl_xor_sync(kFull, s, 4));
            s = __fadd_rn(s, __shfl_xor_sync(kFull, s, 2));
            s = __fadd_rn(s, __shfl_xor_sync(kFull, s, 1));
            raw = s;
        }
        if (live && l == 0) {
            auto rd = [](const uint8_t* b) { return (uint32_t)__ldg(b) | ((uint32_t)__ldg(b + 1) << 8) | ((uint32_t)__ldg(b + 2) << 16) | ((uint32_t)__ldg(b + 3) << 24); };
            const uint32_t d = rd(row);
            const float yb = __uint_as_float(rd(row + 4)), ya = __uint_as_float(rd(row + 12)), yq = __uint_as_float(rd(row + 16));
            float res;
            if (d != p.dim) {
                res = __int_as_float(0x7FC00000);  // UnequalLengths
            } else {
                const float ip = __fadd_rn(__fmul_rn(raw, ya), __fmul_rn(q_sum, yb));
                if (p.metric == DAB_INNER_PRODUCT) res = -ip;
                else if (p.metric == DAB_L2) res = __fsub_rn(__fadd_rn(q_ns, yq), __fmul_rn(2.0f, ip));
                else if (p.metric == DAB_COSINE) res = __fsub_rn(1.0f, __fdiv_rn(ip, __fmul_rn(__fsqrt_rn(q_ns), __fsqrt_rn(yq))));
                else res = __fsub_rn(1.0f, ip);
            }
            p.out[(size_t)q * p.n + r] = res;
        }
    }
}

}  // namespace dab

using namespace dab;

static bool mm_bits_ok(int nbits) { return nbits == 1 || nbits == 2 || nbits == 4 || nbits == 8; }

namespace dab {

bool mm_compress_setup(float grid_scale, uint32_t dim, int nbits, uint64_t n, MinMaxCompressParams& p, int& warps, size_t& smem) {
    memset(&p, 0, sizeof(p));
    p.grid_scale = grid_scale;
    p.dim = dim;
    p.nbits = nbits;
    p.n = n;
    p.row_bytes = kMmMeta + (uint32_t)(((uint64_t)dim * nbits + 7) / 8);
    uint32_t words = (p.row_bytes + 3) / 4;
    if ((words & 1u) == 0) ++words;
    p.srow_stride = words * 4;
    p.warp_smem = 32 * 33 * 4 + 32 * p.srow_stride;
    warps = 4;
    while (warps > 1 && (size_t)warps * p.warp_smem > 200 * 1024) warps >>= 1;
    smem = (size_t)warps * p.warp_smem;
    return smem <= 200 * 1024;
}

cudaError_t mm_compress_launch(const MinMaxCompressParams& p, int warps, size_t smem, cudaStream_t stream) {
    cudaError_t e = cudaFuncSetAttribute(minmax_compress_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) {
        const uint64_t groups = (p.n + 31) / 32;
        const int grid = (int)std::min<uint64_t>((groups + warps - 1) / warps, 132ull * 8);
        minmax_compress_kernel<<<grid, warps * 32, smem, stream>>>(p);
        DAB_LAUNCHED();
        e = cudaGetLastError();
    }
    return e;
}

}  // namespace dab

// the FullQueryMeta kernel, then the distance kernel for p.nbits (p's pointers are device pointers)
static cudaError_t mm_query_launch(const MinMaxQueryParams& p) {
    minmax_query_meta_kernel<<<(p.nq + 127) / 128, 128>>>(p);
    DAB_LAUNCHED();
    const uint32_t lpp = p.nbits == 8 ? 1 : 8;
    const uint64_t pairs_per_cta = 256 / lpp;
    const dim3 grid((unsigned)std::min<uint64_t>((p.n + pairs_per_cta - 1) / pairs_per_cta, 132ull * 8), p.nq);
    const size_t smem = (size_t)p.dim * 4;
    switch (p.nbits) {
        case 8: minmax_query_distance_kernel<8><<<grid, 256, smem>>>(p); break;
        case 4: minmax_query_distance_kernel<4><<<grid, 256, smem>>>(p); break;
        case 2: minmax_query_distance_kernel<2><<<grid, 256, smem>>>(p); break;
        default: minmax_query_distance_kernel<1><<<grid, 256, smem>>>(p); break;
    }
    DAB_LAUNCHED();
    return cudaGetLastError();
}

extern "C" {

uint32_t dab_minmax_row_bytes(uint32_t dim, int nbits) { return mm_bits_ok(nbits) ? kMmMeta + (uint32_t)(((uint64_t)dim * nbits + 7) / 8) : 0; }

int dab_minmax_compress(int device, float grid_scale, uint32_t dim, int nbits, const float* vectors, uint64_t n, uint8_t* out_rows,
                        float* out_loss) {
    if (!mm_bits_ok(nbits)) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_minmax_compress: nbits must be 1, 2, 4 or 8");
    if (!(grid_scale > 0.0f)) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_minmax_compress: grid_scale must be positive (num::Positive)");
    if (n == 0) return DAB_OK;
    if (!vectors || !out_rows || dim == 0) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_minmax_compress: NULL argument");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(DAB_ERR_NO_DEVICE, "dab_minmax_compress: no CUDA device visible");
    DAB_CUDA(cudaSetDevice(device));
    MinMaxCompressParams p;
    int warps;
    size_t smem;
    if (!mm_compress_setup(grid_scale, dim, nbits, n, p, warps, smem))
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_minmax_compress: rows of %u bytes do not fit the staging buffers", p.row_bytes);
    float *d_vec = nullptr, *d_loss = nullptr;
    uint8_t* d_rows = nullptr;
    unsigned long long* d_nan = nullptr;
    cudaError_t e = cudaMalloc(&d_vec, n * dim * 4);
    if (e == cudaSuccess) e = cudaMalloc(&d_rows, n * p.row_bytes);
    if (e == cudaSuccess) e = cudaMalloc(&d_loss, n * 4);
    if (e == cudaSuccess) e = cudaMalloc(&d_nan, 8);
    if (e == cudaSuccess) e = cudaMemcpy(d_vec, vectors, n * dim * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemset(d_nan, 0xFF, 8);
    unsigned long long first_nan = ~0ull;
    if (e == cudaSuccess) {
        p.vectors = d_vec;
        p.rows = d_rows;
        p.loss = d_loss;
        p.first_nan = d_nan;
        e = mm_compress_launch(p, warps, smem);
    }
    if (e == cudaSuccess) e = cudaMemcpy(out_rows, d_rows, n * p.row_bytes, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && out_loss) e = cudaMemcpy(out_loss, d_loss, n * 4, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(&first_nan, d_nan, 8, cudaMemcpyDeviceToHost);
    int rc = DAB_OK;
    if (e != cudaSuccess) rc = fail(e == cudaErrorMemoryAllocation ? DAB_ERR_OUT_OF_MEMORY : DAB_ERR_CUDA, "dab_minmax_compress: %s", cudaGetErrorString(e));
    else if (first_nan != ~0ull)
        rc = fail(DAB_ERR_INVALID_ARGUMENT, "dab_minmax_compress: vector %llu contains NaN (InputContainsNaN); its row was written all the same", first_nan);
    cudaFree(d_vec);
    cudaFree(d_rows);
    cudaFree(d_loss);
    cudaFree(d_nan);
    return rc;
}

int dab_minmax_distances(int device, int metric, int nbits_x, int nbits_y, uint32_t dim, const uint8_t* x_rows, const uint8_t* y_rows,
                         uint64_t n, float* out) {
    if (!mm_bits_ok(nbits_x) || !mm_bits_ok(nbits_y)) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_minmax_distances: nbits must be 1, 2, 4 or 8");
    if (nbits_x != nbits_y && nbits_x != 8)
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_minmax_distances: the reference pairs N x N and 8 x N bit vectors (got %d x %d)", nbits_x, nbits_y);
    if (metric < DAB_COSINE || metric > DAB_COSINE_NORMALIZED) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_minmax_distances: unknown metric %d", metric);
    if (n == 0) return DAB_OK;
    if (!x_rows || !y_rows || !out || dim == 0) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_minmax_distances: NULL argument");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(DAB_ERR_NO_DEVICE, "dab_minmax_distances: no CUDA device visible");
    DAB_CUDA(cudaSetDevice(device));
    MinMaxDistanceParams p;
    memset(&p, 0, sizeof(p));
    p.metric = metric;
    p.nbits_x = nbits_x;
    p.nbits_y = nbits_y;
    p.dim = dim;
    p.row_bytes_x = dab_minmax_row_bytes(dim, nbits_x);
    p.row_bytes_y = dab_minmax_row_bytes(dim, nbits_y);
    p.n = n;
    uint8_t *dx = nullptr, *dy = nullptr;
    float* dout = nullptr;
    cudaError_t e = cudaMalloc(&dx, n * p.row_bytes_x);
    if (e == cudaSuccess) e = cudaMalloc(&dy, n * p.row_bytes_y);
    if (e == cudaSuccess) e = cudaMalloc(&dout, n * 4);
    if (e == cudaSuccess) e = cudaMemcpy(dx, x_rows, n * p.row_bytes_x, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dy, y_rows, n * p.row_bytes_y, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        p.x = dx;
        p.y = dy;
        p.out = dout;
        const int grid = (int)std::min<uint64_t>((n + 31) / 32, 132ull * 8);  // 8 warps x 4 pairs per CTA pass
        minmax_distance_kernel<<<grid, 256>>>(p);
        DAB_LAUNCHED();
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, dout, n * 4, cudaMemcpyDeviceToHost);
    int rc = DAB_OK;
    if (e != cudaSuccess) rc = fail(e == cudaErrorMemoryAllocation ? DAB_ERR_OUT_OF_MEMORY : DAB_ERR_CUDA, "dab_minmax_distances: %s", cudaGetErrorString(e));
    cudaFree(dx);
    cudaFree(dy);
    cudaFree(dout);
    return rc;
}

int dab_minmax_query_distances(int device, int metric, int nbits, uint32_t dim, const float* queries, uint32_t nq, const uint8_t* rows,
                               uint64_t n, float* out) {
    if (!mm_bits_ok(nbits)) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_minmax_query_distances: nbits must be 1, 2, 4 or 8");
    if (metric < DAB_COSINE || metric > DAB_COSINE_NORMALIZED) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_minmax_query_distances: unknown metric %d", metric);
    if (nq == 0 || n == 0) return DAB_OK;
    if (!queries || !rows || !out || dim == 0) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_minmax_query_distances: NULL argument");
    if ((size_t)dim * 4 > 48 * 1024) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_minmax_query_distances: dim %u too large", dim);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(DAB_ERR_NO_DEVICE, "dab_minmax_query_distances: no CUDA device visible");
    DAB_CUDA(cudaSetDevice(device));
    MinMaxQueryParams p;
    memset(&p, 0, sizeof(p));
    p.metric = metric;
    p.nbits = nbits;
    p.dim = dim;
    p.nq = nq;
    p.row_bytes = dab_minmax_row_bytes(dim, nbits);
    p.n = n;
    float *dq = nullptr, *dmeta = nullptr, *dout = nullptr;
    uint8_t* drows = nullptr;
    unsigned long long* d_nan = nullptr;
    cudaError_t e = cudaMalloc(&dq, (size_t)nq * dim * 4);
    if (e == cudaSuccess) e = cudaMalloc(&drows, n * p.row_bytes);
    if (e == cudaSuccess) e = cudaMalloc(&dmeta, (size_t)nq * 8);
    if (e == cudaSuccess) e = cudaMalloc(&dout, (size_t)nq * n * 4);
    if (e == cudaSuccess) e = cudaMalloc(&d_nan, 8);
    if (e == cudaSuccess) e = cudaMemcpy(dq, queries, (size_t)nq * dim * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(drows, rows, n * p.row_bytes, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemset(d_nan, 0xFF, 8);
    unsigned long long first_nan = ~0ull;
    if (e == cudaSuccess) {
        p.queries = dq;
        p.rows = drows;
        p.meta = dmeta;
        p.out = dout;
        p.first_nan = d_nan;
        e = mm_query_launch(p);
    }
    if (e == cudaSuccess) e = cudaMemcpy(&first_nan, d_nan, 8, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && first_nan == ~0ull) e = cudaMemcpy(out, dout, (size_t)nq * n * 4, cudaMemcpyDeviceToHost);
    int rc = DAB_OK;
    if (e != cudaSuccess) rc = fail(e == cudaErrorMemoryAllocation ? DAB_ERR_OUT_OF_MEMORY : DAB_ERR_CUDA, "dab_minmax_query_distances: %s", cudaGetErrorString(e));
    else if (first_nan != ~0ull) rc = fail(DAB_ERR_INVALID_ARGUMENT, "dab_minmax_query_distances: query %llu contains NaN (InputContainsNaN)", first_nan);
    cudaFree(dq);
    cudaFree(drows);
    cudaFree(dmeta);
    cudaFree(dout);
    cudaFree(d_nan);
    return rc;
}

// ---------------------------------------------------------------- behind a Hadamard transform (transform_kernels.cu)

int dab_minmax_compress_transformed(const dab_transform* t, int device, float grid_scale, int nbits, const float* vectors, uint64_t n,
                                    uint8_t* out_rows, float* out_loss) {
    static const char* who = "dab_minmax_compress_transformed";
    if (!t) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL transform", who);
    if (!mm_bits_ok(nbits)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: nbits must be 1, 2, 4 or 8", who);
    if (!(grid_scale > 0.0f)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: grid_scale must be positive (num::Positive)", who);
    if (n == 0) return DAB_OK;
    if ((!vectors && t->input_dim) || !out_rows) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL argument", who);
    const uint32_t dim = t->output_dim;
    MinMaxCompressParams p;
    int warps;
    size_t smem;
    if (!mm_compress_setup(grid_scale, dim, nbits, n, p, warps, smem))
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: rows of %u bytes do not fit the staging buffers", who, p.row_bytes);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(DAB_ERR_NO_DEVICE, "%s: no CUDA device visible", who);
    DAB_CUDA(cudaSetDevice(device));
    float *d_in = nullptr, *d_vec = nullptr, *d_loss = nullptr;
    uint8_t* d_rows = nullptr;
    unsigned long long* d_nan = nullptr;
    cudaError_t e = cudaMalloc(&d_in, std::max<uint64_t>(1, n * t->input_dim) * 4);
    if (e == cudaSuccess) e = cudaMalloc(&d_vec, n * dim * 4);
    if (e == cudaSuccess) e = cudaMalloc(&d_rows, n * p.row_bytes);
    if (e == cudaSuccess) e = cudaMalloc(&d_loss, n * 4);
    if (e == cudaSuccess) e = cudaMalloc(&d_nan, 8);
    if (e == cudaSuccess && t->input_dim) e = cudaMemcpy(d_in, vectors, n * t->input_dim * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemset(d_nan, 0xFF, 8);
    if (e == cudaSuccess) e = transform_rows(t, d_in, n, d_vec, nullptr);
    unsigned long long first_nan = ~0ull;
    if (e == cudaSuccess) {
        // quantizer.rs:171-228: the quantizer runs on the transformed vector, and so does its NaN check
        p.vectors = d_vec;
        p.rows = d_rows;
        p.loss = d_loss;
        p.first_nan = d_nan;
        e = mm_compress_launch(p, warps, smem);
    }
    if (e == cudaSuccess) e = cudaMemcpy(out_rows, d_rows, n * p.row_bytes, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && out_loss) e = cudaMemcpy(out_loss, d_loss, n * 4, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(&first_nan, d_nan, 8, cudaMemcpyDeviceToHost);
    int rc = DAB_OK;
    if (e != cudaSuccess) rc = fail(e == cudaErrorMemoryAllocation ? DAB_ERR_OUT_OF_MEMORY : DAB_ERR_CUDA, "%s: %s", who, cudaGetErrorString(e));
    else if (first_nan != ~0ull)
        rc = fail(DAB_ERR_INVALID_ARGUMENT, "%s: vector %llu contains NaN after the transform (InputContainsNaN); its row was written all the same", who,
                  first_nan);
    cudaFree(d_in);
    cudaFree(d_vec);
    cudaFree(d_rows);
    cudaFree(d_loss);
    cudaFree(d_nan);
    return rc;
}

int dab_minmax_query_distances_transformed(const dab_transform* t, int device, int metric, int nbits, const float* queries, uint32_t nq,
                                           const uint8_t* rows, uint64_t n, float* out) {
    static const char* who = "dab_minmax_query_distances_transformed";
    if (!t) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL transform", who);
    if (!mm_bits_ok(nbits)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: nbits must be 1, 2, 4 or 8", who);
    if (metric < DAB_COSINE || metric > DAB_COSINE_NORMALIZED) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: unknown metric %d", who, metric);
    if (nq == 0 || n == 0) return DAB_OK;
    if ((!queries && t->input_dim) || !rows || !out) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL argument", who);
    const uint32_t dim = t->output_dim;
    if ((size_t)dim * 4 > 48 * 1024) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: output dim %u too large", who, dim);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(DAB_ERR_NO_DEVICE, "%s: no CUDA device visible", who);
    DAB_CUDA(cudaSetDevice(device));
    MinMaxQueryParams p;
    memset(&p, 0, sizeof(p));
    p.metric = metric;
    p.nbits = nbits;
    p.dim = dim;
    p.nq = nq;
    p.row_bytes = dab_minmax_row_bytes(dim, nbits);
    p.n = n;
    float *dq_in = nullptr, *dq = nullptr, *dmeta = nullptr, *dout = nullptr;
    uint8_t* drows = nullptr;
    unsigned long long* d_nan = nullptr;  // [0]: NaN in an untransformed query, [1]: the meta kernel's flag (not read)
    cudaError_t e = cudaMalloc(&dq_in, std::max<uint64_t>(1, (uint64_t)nq * t->input_dim) * 4);
    if (e == cudaSuccess) e = cudaMalloc(&dq, (size_t)nq * dim * 4);
    if (e == cudaSuccess) e = cudaMalloc(&drows, n * p.row_bytes);
    if (e == cudaSuccess) e = cudaMalloc(&dmeta, (size_t)nq * 8);
    if (e == cudaSuccess) e = cudaMalloc(&dout, (size_t)nq * n * 4);
    if (e == cudaSuccess) e = cudaMalloc(&d_nan, 16);
    if (e == cudaSuccess && t->input_dim) e = cudaMemcpy(dq_in, queries, (size_t)nq * t->input_dim * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(drows, rows, n * p.row_bytes, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemset(d_nan, 0xFF, 16);
    // quantizer.rs:398-401: the NaN check is on the input; the transformed query may hold NaN (inf - inf) and is used as is
    if (e == cudaSuccess) e = transform_rows(t, dq_in, nq, dq, d_nan);
    unsigned long long first_nan = ~0ull;
    if (e == cudaSuccess) {
        p.queries = dq;
        p.rows = drows;
        p.meta = dmeta;
        p.out = dout;
        p.first_nan = d_nan + 1;
        e = mm_query_launch(p);
    }
    if (e == cudaSuccess) e = cudaMemcpy(&first_nan, d_nan, 8, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && first_nan == ~0ull) e = cudaMemcpy(out, dout, (size_t)nq * n * 4, cudaMemcpyDeviceToHost);
    int rc = DAB_OK;
    if (e != cudaSuccess) rc = fail(e == cudaErrorMemoryAllocation ? DAB_ERR_OUT_OF_MEMORY : DAB_ERR_CUDA, "%s: %s", who, cudaGetErrorString(e));
    else if (first_nan != ~0ull) rc = fail(DAB_ERR_INVALID_ARGUMENT, "%s: query %llu contains NaN (InputContainsNaN)", who, first_nan);
    cudaFree(dq_in);
    cudaFree(dq);
    cudaFree(drows);
    cudaFree(dmeta);
    cudaFree(dout);
    cudaFree(d_nan);
    return rc;
}

}  // extern "C"
