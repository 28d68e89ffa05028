// distance_device.cuh — device-side distance arithmetic, bit-identical to the reference's
// x86-64-v3 SIMD schemas (diskann-vector/src/distance/simd.rs).
//
// How the order is reproduced.  The reference accumulates 8-wide vectors round-robin into NA
// accumulators (Strategy4x1/4x2: NA = 4, Strategy2x4: NA = 2; simd.rs:245-483): element e of a
// row lands in "slot" e mod 8*NA = (accumulator (e/8) mod NA, lane e mod 8) and every slot is
// a sequential FMA chain in increasing e.  Here a team of S = 8*NA GPU lanes owns one row and
// lane s owns slot s, so each lane runs exactly the CPU's chain with IEEE fmaf.  The
// accumulators are then combined with xor-shuffles in the reference's order
// ((s0+s1)+(s2+s3): xor 8 then xor 16), the masked remainder (len % 8, zero filled) is
// accumulated on the combined vector (simd.rs:733-744) and sum_tree
// (diskann-wide/src/traits.rs:583-595) is xor 4, 2, 1.  Float addition is commutative, so
// every lane ends with the same bits as the CPU's scalar result.
//
// Integer kernels are exact in i32 (simd.rs:1157-1225, 1913-2146, 2750-3035), so any order
// gives the reference's bits; they use dp4a and redux.sync.
//
// Compile with -fmad=false: all fused multiply-adds here are explicit __fmaf_rn.
#pragma once

#include <cuda_fp16.h>
#include <stdint.h>

#include <type_traits>

#include "dab_common.cuh"

namespace dab {

enum Kind { KIND_L2 = 0, KIND_IP = 1, KIND_COS = 2 };
enum Post { POST_ID = 0, POST_NEG = 1, POST_ONE_MINUS = 2 };

constexpr unsigned kFull = 0xFFFFFFFFu;

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f32(int8_t v) { return (float)v; }
__device__ __forceinline__ float to_f32(uint8_t v) { return (float)v; }

__device__ __forceinline__ float ldg_elem(const float* p) { return __ldg(p); }
__device__ __forceinline__ float ldg_elem(const __half* p) {
    return __half2float(__ushort_as_half(__ldg(reinterpret_cast<const unsigned short*>(p))));
}

// FullCosineAccumulator::sum, simd.rs:2328-2364
__device__ __forceinline__ float cosine_finish(float normx, float normy, float prod) {
    float denominator = __fmul_rn(__fsqrt_rn(normx), __fsqrt_rn(normy));
    if (normx < 1.17549435e-38f || normy < 1.17549435e-38f) return 0.0f;
    float v = __fdiv_rn(prod, denominator);
    return fmaxf(-1.0f, fminf(1.0f, v));
}

// implementations.rs:217-404
template <int POST>
__device__ __forceinline__ float post_op(float v) {
    if (POST == POST_NEG) return -v;
    if (POST == POST_ONE_MINUS) return __fsub_rn(1.0f, v);
    return v;
}

// sum_tree over the 8 CPU lanes held by GPU lanes differing in bits 0..2
__device__ __forceinline__ float tree8(float a) {
    a = __fadd_rn(a, __shfl_xor_sync(kFull, a, 4));
    a = __fadd_rn(a, __shfl_xor_sync(kFull, a, 2));
    a = __fadd_rn(a, __shfl_xor_sync(kFull, a, 1));
    return a;
}

template <int NA>
__device__ __forceinline__ float combine_acc(float a) {
    a = __fadd_rn(a, __shfl_xor_sync(kFull, a, 8));
    if (NA == 4) a = __fadd_rn(a, __shfl_xor_sync(kFull, a, 16));
    return a;
}

// U rows against one query, one team of S = 8*NA lanes per row, all 32 lanes of the warp
// must call this together.  `slot` = lane index inside the team.  q: query elements
// (shared or global memory), rows[u]: global rows.  Returns the mathematical value
// (pre post-op) of row u in out[u] on every lane of the team.
// EU: unroll factor of the element loop — EU * U independent row loads in flight per lane (the
// pure gather kernels need the memory-level parallelism; the search kernels keep registers).
template <int NA, int KIND, int U, int EU = 1, typename TQ, typename TD>
__device__ __forceinline__ void team_float_multi(const TQ* __restrict__ q,
                                                 const TD* const (&rows)[U], int dim, int slot,
                                                 float (&out)[U]) {
    constexpr int S = 8 * NA;
    const int full8 = dim & ~7;
    const int rem = dim & 7;
    if (KIND == KIND_COS) {
        float nx = 0.0f, ny[U], xy[U];
#pragma unroll
        for (int u = 0; u < U; ++u) ny[u] = xy[u] = 0.0f;
#pragma unroll(EU)
        for (int e = slot; e < full8; e += S) {
            float x = to_f32(q[e]);
            float y[U];
#pragma unroll
            for (int u = 0; u < U; ++u) y[u] = ldg_elem(rows[u] + e);
            nx = __fmaf_rn(x, x, nx);
#pragma unroll
            for (int u = 0; u < U; ++u) {
                ny[u] = __fmaf_rn(y[u], y[u], ny[u]);
                xy[u] = __fmaf_rn(x, y[u], xy[u]);
            }
        }
        nx = combine_acc<NA>(nx);
#pragma unroll
        for (int u = 0; u < U; ++u) {
            ny[u] = combine_acc<NA>(ny[u]);
            xy[u] = combine_acc<NA>(xy[u]);
        }
        if (rem) {
            const int l = slot & 7;
            float x = l < rem ? to_f32(q[full8 + l]) : 0.0f;
            nx = __fmaf_rn(x, x, nx);
#pragma unroll
            for (int u = 0; u < U; ++u) {
                float y = l < rem ? ldg_elem(rows[u] + full8 + l) : 0.0f;
                ny[u] = __fmaf_rn(y, y, ny[u]);
                xy[u] = __fmaf_rn(x, y, xy[u]);
            }
        }
        nx = tree8(nx);
#pragma unroll
        for (int u = 0; u < U; ++u) out[u] = cosine_finish(nx, tree8(ny[u]), tree8(xy[u]));
    } else {
        float acc[U];
#pragma unroll
        for (int u = 0; u < U; ++u) acc[u] = 0.0f;
#pragma unroll(EU)
        for (int e = slot; e < full8; e += S) {
            float x = to_f32(q[e]);
            float y[U];
#pragma unroll
            for (int u = 0; u < U; ++u) y[u] = ldg_elem(rows[u] + e);
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (KIND == KIND_L2) {
                    float c = __fsub_rn(x, y[u]);
                    acc[u] = __fmaf_rn(c, c, acc[u]);
                } else {
                    acc[u] = __fmaf_rn(x, y[u], acc[u]);
                }
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) acc[u] = combine_acc<NA>(acc[u]);
        if (rem) {
            const int l = slot & 7;
            float x = l < rem ? to_f32(q[full8 + l]) : 0.0f;
#pragma unroll
            for (int u = 0; u < U; ++u) {
                float y = l < rem ? ldg_elem(rows[u] + full8 + l) : 0.0f;
                if (KIND == KIND_L2) {
                    float c = __fsub_rn(x, y);
                    acc[u] = __fmaf_rn(c, c, acc[u]);
                } else {
                    acc[u] = __fmaf_rn(x, y, acc[u]);
                }
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) out[u] = tree8(acc[u]);
    }
}

// ---- integers: whole warp per row -----------------------------------------------------
template <bool SIGNED>
__device__ __forceinline__ int dp4(int a, int b, int c) {
    if (SIGNED) return __dp4a(a, b, c);
    return (int)__dp4a((unsigned)a, (unsigned)b, (unsigned)c);
}
template <bool SIGNED>
__device__ __forceinline__ int byte_at(const uint8_t* p, int i) {
    return SIGNED ? (int)((const int8_t*)p)[i] : (int)p[i];
}

// sum x*x over a byte vector by the whole warp (exact); p must be 4-byte aligned.
template <bool SIGNED>
__device__ __forceinline__ int warp_int_self(const uint8_t* p, int dim, int lane) {
    int acc = 0;
    const int nwords = dim >> 2;
    for (int w = lane; w < nwords; w += 32) {
        int x = reinterpret_cast<const int*>(p)[w];
        acc = dp4<SIGNED>(x, x, acc);
    }
    const int tail = dim & 3;
    if (lane < tail) {
        int x = byte_at<SIGNED>(p, (nwords << 2) + lane);
        acc += x * x;
    }
    return __reduce_add_sync(kFull, acc);
}

// U rows against one query by the whole warp.  q and rows 4-byte aligned.  qq = sum q*q.
template <bool SIGNED, int KIND, int U>
__device__ __forceinline__ void warp_int_multi(const uint8_t* __restrict__ q,
                                               const uint8_t* const (&rows)[U], int dim, int lane,
                                               int qq, float (&out)[U]) {
    int xy[U], yy[U];
#pragma unroll
    for (int u = 0; u < U; ++u) xy[u] = yy[u] = 0;
    const int nwords = dim >> 2;
    for (int w = lane; w < nwords; w += 32) {
        int x = reinterpret_cast<const int*>(q)[w];
        int y[U];
#pragma unroll
        for (int u = 0; u < U; ++u) y[u] = __ldg(reinterpret_cast<const int*>(rows[u]) + w);
#pragma unroll
        for (int u = 0; u < U; ++u) {
            xy[u] = dp4<SIGNED>(x, y[u], xy[u]);
            if (KIND != KIND_IP) yy[u] = dp4<SIGNED>(y[u], y[u], yy[u]);
        }
    }
    const int tail = dim & 3;
    if (lane < tail) {
        const int i = (nwords << 2) + lane;
        int x = byte_at<SIGNED>(q, i);
#pragma unroll
        for (int u = 0; u < U; ++u) {
            int y = byte_at<SIGNED>(rows[u], i);
            xy[u] += x * y;
            if (KIND != KIND_IP) yy[u] += y * y;
        }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
        int sxy = __reduce_add_sync(kFull, xy[u]);
        if (KIND == KIND_IP) {
            out[u] = (float)sxy;
        } else {
            int syy = __reduce_add_sync(kFull, yy[u]);
            if (KIND == KIND_L2) {
                // sum (x-y)^2 = sum x^2 + sum y^2 - 2 sum xy, exact in wrapping i32
                out[u] = (float)(int)((unsigned)qq + (unsigned)syy - 2u * (unsigned)sxy);
            } else {
                out[u] = cosine_finish((float)qq, (float)syy, (float)sxy);
            }
        }
    }
}

// ---- metric dispatch --------------------------------------------------------------------
// Which (kind, post-op) a metric means: implementations.rs:217-404; integer CosineNormalized
// is Cosine (distance_provider.rs:275-297).
struct MetricPlan {
    int kind;
    int post;
};
__host__ __device__ inline MetricPlan plan_for(int metric, bool is_int) {
    switch (metric) {
        case DAB_L2: return {KIND_L2, POST_ID};
        case DAB_INNER_PRODUCT: return {KIND_IP, POST_NEG};
        case DAB_COSINE: return {KIND_COS, POST_ONE_MINUS};
        default: return is_int ? MetricPlan{KIND_COS, POST_ONE_MINUS} : MetricPlan{KIND_IP, POST_ONE_MINUS};
    }
}

// ---- schema dispatch (host) --------------------------------------------------------------
// What a row of the index is compared with: a query (float queries are widened to f32,
// diskann-inmem/src/layers/full.rs:421-423) or another row of the index (data x data).
enum Operands { OPS_QUERY, OPS_ROW };

// The compile-time values of one distance schema, as the launchers' kernels take them.
template <typename TQ_, typename TD_, int NA_, int KIND_, int POST_>
struct Schema {
    using TQ = TQ_;  // the other operand: float, __half (f16 x f16), int8_t or uint8_t
    using TD = TD_;  // row elements: float, __half, int8_t or uint8_t
    static constexpr int NA = NA_, KIND = KIND_, POST = POST_;
    static constexpr bool IS_INT = std::is_same<TD, int8_t>::value || std::is_same<TD, uint8_t>::value;
    static constexpr bool SIGNED = std::is_same<TD, int8_t>::value;
};

// The row type of the kernels that take integer rows as uint8_t plus a SIGNED flag.
template <typename S>
using KernelRow = typename std::conditional<S::IS_INT, uint8_t, typename S::TD>::type;

// The reference's schema for TQ x TD under `metric`: (KIND, POST) from plan_for; NA = 2 for cosine over
// float operands and for f16 x f16 (Strategy2x4, simd.rs:424-483, 989, 1752, 2591), otherwise NA = 4
// (Strategy4x1 / 4x2; the integer kernels ignore it).  Only these schemas are ever instantiated.
template <typename TQ, typename TD, typename F>
int visit_plan(int metric, F&& f) {
    constexpr bool I = std::is_same<TD, int8_t>::value || std::is_same<TD, uint8_t>::value;
    constexpr int NA = std::is_same<TQ, __half>::value ? 2 : 4;
    const MetricPlan plan = plan_for(metric, I);
    if (plan.kind == KIND_L2) return f(Schema<TQ, TD, NA, KIND_L2, POST_ID>{});
    if (plan.kind == KIND_COS) return f(Schema<TQ, TD, I ? 4 : 2, KIND_COS, POST_ONE_MINUS>{});
    if constexpr (!I) {  // float CosineNormalized; for integers it is Cosine
        if (plan.post == POST_ONE_MINUS) return f(Schema<TQ, TD, NA, KIND_IP, POST_ONE_MINUS>{});
    }
    return f(Schema<TQ, TD, NA, KIND_IP, POST_NEG>{});
}

// Calls f(Schema<...>{}) once, with the schema of rows of `dtype` against operands O under `metric`,
// and returns what f returns.
template <Operands O, typename F>
int visit_schema(int dtype, int metric, F&& f) {
    switch (dtype) {
        case DAB_F32: return visit_plan<float, float>(metric, f);
        case DAB_F16: return visit_plan<typename std::conditional<O == OPS_QUERY, float, __half>::type, __half>(metric, f);
        case DAB_I8: return visit_plan<int8_t, int8_t>(metric, f);
        case DAB_U8: return visit_plan<uint8_t, uint8_t>(metric, f);
    }
    return fail(DAB_ERR_INVALID_ARGUMENT, "unsupported dtype %d", dtype);
}

}  // namespace dab
