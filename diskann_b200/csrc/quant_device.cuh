// quant_device.cuh — thread-serial emulation of the reference's simd_op for short f32 chunks
// (PQ LUT entries, encode), the packed-code integer cores, the scalar quantizer and the SQ / MinMax
// epilogues, and the per-candidate distances of the quantized traversals, shared by quant_kernels.cu, sq_index.cu,
// minmax_kernels.cu, search_kernel_pq.cu, search_kernel_pqs.cu and the StoreSource of the paged, diverse, filtered and
// range traversals (search_source.cuh).
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

// ------------------------------------------------------------------ per-candidate distances of the quantized traversals
// What one lane computes for one candidate in the quantized accessor's expand_beam: search_kernel_pq.cu (one-shot and
// in-flight batches) and StoreSource (paged, diverse, filtered and range search) share these, so all return the same bits.

// the integer cores of one packed code row against the query's code words, 16 B at a time
template <int NBITS>
__device__ __forceinline__ void sq_row(const uint4* __restrict__ row, const uint4* qc, uint32_t vecs, bool want_ip, uint32_t& l2,
                                       uint32_t& ip) {
    for (uint32_t v = 0; v < vecs; ++v) {
        const uint4 a = __ldg(row + v);
        const uint4 b = qc[v];
        sq_word<NBITS>(a.x, b.x, want_ip, l2, ip);
        sq_word<NBITS>(a.y, b.y, want_ip, l2, ip);
        sq_word<NBITS>(a.z, b.z, want_ip, l2, ip);
        sq_word<NBITS>(a.w, b.w, want_ip, l2, ip);
    }
}

// MODE 1 (SQ) / MODE 2 (MinMax): the distance of packed code row `id` to the query's code words qc (16 B aligned; MinMax:
// its {b, n, a, norm_squared} follow the words), the query as x and the row as y.  P names the store as SearchParamsPq
// does (row_codes, row_meta, code_stride, code_nbits, code_metric, code_dim, sq_scale_squared, sq_shift_square_norm).
// Only SQ InnerProduct loads the row's compensation; MinMax loads the row's four.
template <int MODE, class P>
__device__ __forceinline__ float packed_code_distance(const P& p, const uint32_t* qc, float q_comp, uint32_t id) {
    const uint4* row = reinterpret_cast<const uint4*>(p.row_codes + (size_t)id * p.code_stride);
    const uint4* q4 = reinterpret_cast<const uint4*>(qc);
    const uint32_t vecs = p.code_stride >> 4;
    const bool want_ip = MODE == 2 || p.code_metric == DAB_INNER_PRODUCT;  // MinMax: every metric
    uint32_t l2 = 0, ip = 0;
    switch (p.code_nbits) {
        case 8: sq_row<8>(row, q4, vecs, want_ip, l2, ip); break;
        case 4: sq_row<4>(row, q4, vecs, want_ip, l2, ip); break;
        case 2: sq_row<2>(row, q4, vecs, want_ip, l2, ip); break;
        default: sq_row<1>(row, q4, vecs, want_ip, l2, ip); break;
    }
    if (MODE == 1) {
        const float ibs = __fdiv_rn(1.0f, (float)((1u << p.code_nbits) - 1u));
        const float mul = __fmul_rn(__fmul_rn(ibs, ibs), p.sq_scale_squared);
        return sq_finish(p.code_metric, l2, ip, mul, p.sq_shift_square_norm, q_comp, want_ip ? __ldg(p.row_meta + id) : 0.0f);
    } else {
        const float4 qm = *reinterpret_cast<const float4*>(qc + (p.code_stride >> 2));
        const float4 rm = __ldg(reinterpret_cast<const float4*>(p.row_meta) + id);
        return minmax_finish(p.code_metric, ip, p.code_dim, qm.x, qm.y, qm.z, qm.w, rm.x, rm.y, rm.z, rm.w);
    }
}

// PQ: P names the table as SearchParamsPq does (codes, n_chunks, n_centers, offsets, pivots, ip_table).
// DirectCosine (pq/distance/cosine.rs:16-70; direct_distance_impl, fixed_chunk_pq_table.rs:35-59): the Resumable V3
// cosine (Strategy2x4) accumulated chunk by chunk over the pivots the code of row `id` selects, 1 - cos.  qf: the f32 query.
template <class P>
__device__ __forceinline__ float pq_direct_cosine(const P& p, const float* qf, int dim, uint32_t id) {
    const uint8_t* code = p.codes + (size_t)id * p.n_chunks;
    float nx[8], ny[8], xy[8];
#pragma unroll
    for (int l = 0; l < 8; ++l) nx[l] = ny[l] = xy[l] = 0.0f;
    for (uint32_t ch = 0; ch < p.n_chunks; ++ch) {
        const uint32_t start = p.offsets[ch], stop = p.offsets[ch + 1];
        const float* xc = qf + start;
        const float* yc = p.pivots + (size_t)__ldg(code + ch) * dim + start;
        float a[8], b[8], d[8];
        thread_simd_combined<2, KIND_IP>(xc, xc, (int)(stop - start), a);
        thread_simd_combined<2, KIND_IP>(yc, yc, (int)(stop - start), b);
        thread_simd_combined<2, KIND_IP>(xc, yc, (int)(stop - start), d);
#pragma unroll
        for (int l = 0; l < 8; ++l) {
            nx[l] = __fadd_rn(nx[l], a[l]);
            ny[l] = __fadd_rn(ny[l], b[l]);
            xy[l] = __fadd_rn(xy[l], d[l]);
        }
    }
    return __fsub_rn(1.0f, cosine_finish(thread_tree8(nx), thread_tree8(ny), thread_tree8(xy)));
}

// TableL2 / TableIP: the ADC lookups of row `id` in the query's table (n_chunks x n_centers f32 in global memory, read
// through L2), summed in chunk order from 0.0 (pq_dist_lookup_single, fixed_chunk_pq_table.rs:82-98)
template <class P>
__device__ __forceinline__ float pq_table_distance(const P& p, const float* lut, uint32_t id) {
    const uint8_t* code = p.codes + (size_t)id * p.n_chunks;
    float accum = 0.0f;
    uint32_t ch = 0;
    if ((p.n_chunks & 15u) == 0) {
        for (; ch < p.n_chunks; ch += 16) {
            const uint4 w = __ldg(reinterpret_cast<const uint4*>(code + ch));
            const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
            float v[16];
#pragma unroll
            for (int k2 = 0; k2 < 16; ++k2) v[k2] = __ldcg(lut + (ch + k2) * p.n_centers + ((ws[k2 >> 2] >> ((k2 & 3) * 8)) & 0xFFu));
#pragma unroll
            for (int k2 = 0; k2 < 16; ++k2) accum = __fadd_rn(accum, v[k2]);
        }
    } else {
        for (; ch < p.n_chunks; ++ch) accum = __fadd_rn(accum, __ldcg(lut + ch * p.n_centers + __ldg(code + ch)));
    }
    return accum;
}

// entry t = chunk * n_centers + centre of the query's table (fixed_chunk_pq_table.rs:152-187): TableIP entries are -dot
template <class P>
__device__ __forceinline__ float pq_table_entry(const P& p, const float* qf, int dim, uint32_t t) {
    const uint32_t chunk = t / p.n_centers, center = t % p.n_centers;
    const uint32_t start = p.offsets[chunk], stop = p.offsets[chunk + 1];
    const float* piv = p.pivots + (size_t)center * dim + start;
    float v;
    if (p.ip_table) v = -thread_simd_l2ip<KIND_IP>(qf + start, piv, (int)(stop - start));
    else v = thread_simd_l2ip<KIND_L2>(qf + start, piv, (int)(stop - start));
    return v;
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
