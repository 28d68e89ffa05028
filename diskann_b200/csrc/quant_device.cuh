// quant_device.cuh — thread-serial emulation of the reference's simd_op for short f32 chunks
// (PQ LUT entries, encode), the packed-code integer cores, the scalar quantizer and the SQ / MinMax
// epilogues, shared by quant_kernels.cu, sq_index.cu and search_kernel_pq.cu.
#pragma once

#include "distance_device.cuh"

namespace dab {

// ------------------------------------------------------------------ thread-serial simd_op
// One thread emulates simd_op (simd.rs:686-747) for f32 x f32 with NA accumulators of 8
// lanes and returns the *combined* 8-lane accumulator (what Resumable::combine_with receives,
// simd.rs:637-671).  Used where work items are tiny (PQ chunks of 2..16 dims).
template <int NA, int KIND /*L2 or IP*/>
__device__ __forceinline__ void thread_simd_combined(const float* __restrict__ x, const float* __restrict__ y,
                                                     int len, float (&c)[8]) {
    float s[NA][8];
#pragma unroll
    for (int a = 0; a < NA; ++a)
#pragma unroll
        for (int l = 0; l < 8; ++l) s[a][l] = 0.0f;
    const int full = len >> 3;
    const int groups = full / NA;
    for (int g = 0; g < groups; ++g) {
#pragma unroll
        for (int a = 0; a < NA; ++a) {
            const int base = (g * NA + a) * 8;
#pragma unroll
            for (int l = 0; l < 8; ++l) {
                float xv = x[base + l], yv = y[base + l];
                if (KIND == KIND_L2) {
                    float d = __fsub_rn(xv, yv);
                    s[a][l] = __fmaf_rn(d, d, s[a][l]);
                } else {
                    s[a][l] = __fmaf_rn(xv, yv, s[a][l]);
                }
            }
        }
    }
    const int ep = full - groups * NA;
#pragma unroll
    for (int a = 0; a < NA - 1; ++a) {
        if (a < ep) {
            const int base = (groups * NA + a) * 8;
#pragma unroll
            for (int l = 0; l < 8; ++l) {
                float xv = x[base + l], yv = y[base + l];
                if (KIND == KIND_L2) {
                    float d = __fsub_rn(xv, yv);
                    s[a][l] = __fmaf_rn(d, d, s[a][l]);
                } else {
                    s[a][l] = __fmaf_rn(xv, yv, s[a][l]);
                }
            }
        }
    }
#pragma unroll
    for (int l = 0; l < 8; ++l) {
        if (NA == 4)
            c[l] = __fadd_rn(__fadd_rn(s[0][l], s[1][l]), __fadd_rn(s[2 % NA][l], s[3 % NA][l]));
        else
            c[l] = __fadd_rn(s[0][l], s[1 % NA][l]);
    }
    const int rem = len & 7;
    if (rem) {
        const int base = full * 8;
#pragma unroll
        for (int l = 0; l < 8; ++l) {
            float xv = l < rem ? x[base + l] : 0.0f, yv = l < rem ? y[base + l] : 0.0f;
            if (KIND == KIND_L2) {
                float d = __fsub_rn(xv, yv);
                c[l] = __fmaf_rn(d, d, c[l]);
            } else {
                c[l] = __fmaf_rn(xv, yv, c[l]);
            }
        }
    }
}

__device__ __forceinline__ float thread_tree8(const float (&c)[8]) {
    float a0 = __fadd_rn(c[0], c[4]), a1 = __fadd_rn(c[1], c[5]), a2 = __fadd_rn(c[2], c[6]), a3 = __fadd_rn(c[3], c[7]);
    return __fadd_rn(__fadd_rn(a0, a2), __fadd_rn(a1, a3));
}

template <int KIND>
__device__ __forceinline__ float thread_simd_l2ip(const float* x, const float* y, int len) {
    float c[8];
    thread_simd_combined<4, KIND>(x, y, len, c);
    return thread_tree8(c);
}

// ------------------------------------------------------------------ packed N-bit integer cores (bits/distances.rs:397, 979)
// integer cores over one 32-bit word of dense NBITS codes (fields never straddle bytes for 1/2/4/8 bits)
template <int NBITS>
__device__ __forceinline__ void sq_word(uint32_t a, uint32_t b, bool want_ip, uint32_t& l2, uint32_t& ip) {
    if (NBITS == 1) {
        if (want_ip) ip += __popc(a & b);
        else l2 += __popc(a ^ b);
        return;
    }
    constexpr uint32_t kMask = NBITS == 8 ? 0xFFFFFFFFu : NBITS == 4 ? 0x0F0F0F0Fu : 0x03030303u;
#pragma unroll
    for (int sh = 0; sh < 8; sh += NBITS) {
        const uint32_t x = (a >> sh) & kMask, y = (b >> sh) & kMask;
        if (want_ip) {
            ip = __dp4a(x, y, ip);
        } else {
            const uint32_t d = __vabsdiffu4(x, y);
            l2 = __dp4a(d, d, l2);
        }
    }
}

// ------------------------------------------------------------------ scalar quantizer (scalar/quantizer.rs:190-239, 407-430)
// The code of one value: (v - shift) * inverse_scale (= maxv / scale), f32::clamp to [0, maxv] (keeps NaN), rounded half
// away from zero.  A NaN code packs as 0.
__device__ __forceinline__ float sq_code(float v, float shift, float inverse_scale, float maxv) {
    const float t = __fmul_rn(__fsub_rn(v, shift), inverse_scale);
    return roundf(t != t ? t : (t < 0.0f ? 0.0f : (t > maxv ? maxv : t)));
}

// The compensation of a vector from `dot`, the sequential FMA chain of its codes with the shift in dimension order
// (inverse_bit_scale = 1 / maxv).
__device__ __forceinline__ float sq_compensation(float scale, float inverse_bit_scale, float dot) {
    return __fmul_rn(__fmul_rn(scale, inverse_bit_scale), dot);
}

// Compensated{SquaredL2, IP, CosineNormalized} (scalar/vectors.rs:206-237, 310-376, 380-460) of two code vectors x and y
// from the exact integer cores of their codes; mul = bit_scale * scale^2 (AsFunctor, scalar/quantizer.rs:316-335).  Only
// InnerProduct reads the compensations.
__device__ __forceinline__ float sq_finish(int metric, uint32_t l2, uint32_t ip, float mul, float shift_square_norm, float comp_x,
                                           float comp_y) {
    if (metric == DAB_INNER_PRODUCT) return -__fadd_rn(__fmaf_rn(mul, (float)ip, shift_square_norm), __fadd_rn(comp_y, comp_x));
    const float l = __fmul_rn(mul, (float)l2);
    if (metric == DAB_L2) return l;
    return __fsub_rn(1.0f, __fsub_rn(1.0f, __fdiv_rn(l, 2.0f)));
}

// ------------------------------------------------------------------ MinMax epilogue (minmax/vectors.rs:206-228)
// The distance between two MinMax vectors x and y of `dim` codes from the exact inner product `ip` of their codes and
// their compensations {b, n, a, norm_squared}: term0 + term1_x + term1_y + term2 left to right, then the metric's finish.
__device__ __forceinline__ float minmax_finish(int metric, uint32_t ip, uint32_t dim, float xb, float xn, float xa, float xq, float yb,
                                               float yn, float ya, float yq) {
    const float term0 = __fmul_rn(__fmul_rn(xa, ya), (float)ip);
    const float term1_x = __fmul_rn(xn, yb);
    const float term1_y = __fmul_rn(yn, xb);
    const float term2 = __fmul_rn(__fmul_rn(xb, yb), (float)dim);
    const float v = __fadd_rn(__fadd_rn(__fadd_rn(term0, term1_x), term1_y), term2);
    if (metric == DAB_INNER_PRODUCT) return -v;
    if (metric == DAB_L2) return __fadd_rn(__fadd_rn(__fmul_rn(-2.0f, v), xq), yq);
    if (metric == DAB_COSINE) return __fsub_rn(1.0f, __fdiv_rn(v, __fmul_rn(__fsqrt_rn(xq), __fsqrt_rn(yq))));
    return __fsub_rn(1.0f, v);
}

// ------------------------------------------------------------------ PQ table entries from shared-memory pivots
__device__ __forceinline__ void prefetch_l2(const void* ptr) { asm volatile("prefetch.global.L2 [%0];" ::"l"(ptr)); }

// Table entry of (chunk, centre) computed from a query (qf) and a pivot table (spiv, rows pstride floats apart)
// in shared memory; CL = 4 / 8: every chunk has that length and starts 16-byte aligned, 0: lengths from `offsets`.
// The arithmetic is thread_simd_l2ip either way — the same bits whether the entry is stored in a table first or not
// (fixed_chunk_pq_table.rs:152-187; TableIP entries are -dot, implementations.rs:309-314).
template <int CL>
__device__ __forceinline__ float pqs_term(const float* qf, const float* spiv, uint32_t pstride, const uint32_t* __restrict__ offsets,
                                          uint32_t ch, uint32_t center, bool ip) {
    if constexpr (CL == 4 || CL == 8) {
        constexpr int N = CL;
        float x[N], y[N];
        const float4* xp = reinterpret_cast<const float4*>(qf + ch * N);
        const float4* yp = reinterpret_cast<const float4*>(spiv + (size_t)center * pstride + ch * N);
#pragma unroll
        for (int v = 0; v < N / 4; ++v) {
            const float4 a = xp[v], b = yp[v];
            x[4 * v] = a.x, x[4 * v + 1] = a.y, x[4 * v + 2] = a.z, x[4 * v + 3] = a.w;
            y[4 * v] = b.x, y[4 * v + 1] = b.y, y[4 * v + 2] = b.z, y[4 * v + 3] = b.w;
        }
        return ip ? -thread_simd_l2ip<KIND_IP>(x, y, N) : thread_simd_l2ip<KIND_L2>(x, y, N);
    } else {
        const uint32_t start = __ldg(offsets + ch), stop = __ldg(offsets + ch + 1);
        const float* xp = qf + start;
        const float* yp = spiv + (size_t)center * pstride + start;
        return ip ? -thread_simd_l2ip<KIND_IP>(xp, yp, (int)(stop - start)) : thread_simd_l2ip<KIND_L2>(xp, yp, (int)(stop - start));
    }
}

}  // namespace dab
