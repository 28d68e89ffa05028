// transform_kernels.cu — the Hadamard transforms of diskann-quantization/src/algorithms/transforms on the device:
// PaddingHadamard::transform_into (padding_hadamard.rs:204-273) and DoubleHadamard::transform_into
// (double_hadamard.rs:238-287), bit-identical to the reference's x86-64-v3 path.
//
//   * hadamard_transform (hadamard.rs:22-137) dispatches to V3 (V4 retargets to V3), whose order is not the scalar
//     recursion: lengths below 64 run radix-2 butterflies at strides 1 .. len/2 (base case (l + r, l - r)); longer ones
//     split into 64-element blocks that each run micro_kernel_64 (:248-371) — eight 8-point transforms as FMA chains over
//     HADAMARD_8 from +0.0, inputs j = 0..7 in order, then the e / f combination at strides 8, 16, 32 — followed by
//     butterflies at strides 64 .. len/2.  Every element is then multiplied by 1 / sqrt(len) (a length-1 vector is left
//     untouched).  A butterfly level touches each pair once, so running the levels bottom-up gives the recursion's
//     values exactly.
//   * One warp owns one vector, staged in shared memory at its inner length: the input is read coalesced with the sign
//     xor and the zero padding applied on the way in, the stages are separated by __syncwarp, and the output (the whole
//     vector, or the rescaled subsample gather) leaves coalesced.  Element i is stored at sw(i): every 64 elements are
//     followed by 8 unused words, so the four 64-blocks a warp's micro-kernel pass reads start 8 banks apart.
// Explicit __fadd_rn / __fsub_rn / __fmaf_rn / __fmul_rn and no flush-to-zero: subnormals are kept, as on the CPU.
#include "transform.cuh"

#include <algorithm>
#include <new>

namespace dab {

struct TransformParams {
    uint32_t input_dim, inner_dim, output_dim;
    uint32_t split;         // length of each Hadamard transform
    int two_stages;         // DoubleHadamard: H on [0, split), xor signs1, H on [inner - split, inner)
    float scale;            // 1 / sqrt(split)
    float rescale;          // sqrt(inner / output_dim) when subsampling
    const uint32_t* signs0;     // [input_dim]
    const uint32_t* signs1;     // [inner_dim] (two stages only)
    const uint32_t* subsample;  // [output_dim] or NULL
    const float* src;           // [n][input_dim]
    float* dst;                 // [n][output_dim]
    uint64_t n;
    uint32_t warp_floats;       // shared-memory words per warp
    unsigned long long* first_nan;
};

// shared-memory position of element i of the staged vector
__device__ __forceinline__ uint32_t sw(uint32_t i) { return i + ((i >> 6) << 3); }

// radix-2 butterflies (l + r, l - r) at strides s_begin .. len/2 over elements [off, off + len)
__device__ __forceinline__ void butterflies(float* x, uint32_t off, uint32_t len, uint32_t s_begin, int lane) {
    for (uint32_t s = s_begin; s < len; s <<= 1) {
        for (uint32_t p = lane; p < len / 2; p += 32) {
            const uint32_t i = off + (((p & ~(s - 1)) << 1) | (p & (s - 1)));  // pair p: (i, i + s)
            const float l = x[sw(i)], r = x[sw(i + s)];
            x[sw(i)] = __fadd_rn(l, r);
            x[sw(i + s)] = __fsub_rn(l, r);
        }
        __syncwarp();
    }
}

// hadamard_transform over elements [off, off + len) (len a power of two), all lanes of the warp together
__device__ void hadamard_warp(float* x, uint32_t off, uint32_t len, float scale, int lane) {
    if (len == 1) return;
    if (len < 64) {
        butterflies(x, off, len, 1, lane);
    } else {
        // micro_kernel_64: lane item = (64-block, column l); it reads the block's 64 inputs and owns outputs 8 * b + l
        const uint32_t items = (len / 64) * 8;
        for (uint32_t base = 0; base < items; base += 32) {
            const uint32_t item = base + lane;
            float o[8];
            if (item < items) {
                const uint32_t blk = off + (item / 8) * 64;
                const uint32_t l = item & 7u;
                float d[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    float acc = 0.0f;
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc = __fmaf_rn(x[sw(blk + 8 * k + j)], (__popc(j & l) & 1) ? -1.0f : 1.0f, acc);  // HADAMARD_8[j][l]
                    d[k] = acc;
                }
                const float e0 = __fadd_rn(d[0], d[1]), e1 = __fsub_rn(d[0], d[1]);
                const float e2 = __fadd_rn(d[2], d[3]), e3 = __fsub_rn(d[2], d[3]);
                const float e4 = __fadd_rn(d[4], d[5]), e5 = __fsub_rn(d[4], d[5]);
                const float e6 = __fadd_rn(d[6], d[7]), e7 = __fsub_rn(d[6], d[7]);
                const float f0 = __fadd_rn(e0, e2), f1 = __fadd_rn(e1, e3), f2 = __fsub_rn(e0, e2), f3 = __fsub_rn(e1, e3);
                const float f4 = __fadd_rn(e4, e6), f5 = __fadd_rn(e5, e7), f6 = __fsub_rn(e4, e6), f7 = __fsub_rn(e5, e7);
                o[0] = __fadd_rn(f0, f4), o[1] = __fadd_rn(f1, f5), o[2] = __fadd_rn(f2, f6), o[3] = __fadd_rn(f3, f7);
                o[4] = __fsub_rn(f0, f4), o[5] = __fsub_rn(f1, f5), o[6] = __fsub_rn(f2, f6), o[7] = __fsub_rn(f3, f7);
            }
            __syncwarp();  // every lane has read its block before any lane overwrites it
            if (item < items) {
                const uint32_t blk = off + (item / 8) * 64;
                const uint32_t l = item & 7u;
#pragma unroll
                for (int b = 0; b < 8; ++b) x[sw(blk + 8 * b + l)] = o[b];
            }
            __syncwarp();
        }
        butterflies(x, off, len, 64, lane);
    }
    for (uint32_t i = off + lane; i < off + len; i += 32) x[sw(i)] = __fmul_rn(x[sw(i)], scale);
    __syncwarp();
}

__global__ void __launch_bounds__(256) hadamard_transform_kernel(const TransformParams p) {
    extern __shared__ float ht_smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    float* x = ht_smem + (size_t)wib * p.warp_floats;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t v = (uint64_t)blockIdx.x * (blockDim.x >> 5) + wib; v < p.n; v += warps) {
        // copy_and_flip_signs: xor the sign words, zero-pad to the inner length
        const float* src = p.src + v * p.input_dim;
        bool nan = false;
        for (uint32_t i = lane; i < p.inner_dim; i += 32) {
            float e = 0.0f;
            if (i < p.input_dim) {
                const float s = __ldg(src + i);
                nan |= s != s;
                e = __uint_as_float(__float_as_uint(s) ^ __ldg(p.signs0 + i));
            }
            x[sw(i)] = e;
        }
        if (p.first_nan && __any_sync(0xFFFFFFFFu, nan) && lane == 0) atomicMin(p.first_nan, (unsigned long long)v);
        __syncwarp();
        hadamard_warp(x, 0, p.split, p.scale, lane);
        if (p.two_stages) {
            for (uint32_t i = lane; i < p.inner_dim; i += 32) x[sw(i)] = __uint_as_float(__float_as_uint(x[sw(i)]) ^ __ldg(p.signs1 + i));
            __syncwarp();
            hadamard_warp(x, p.inner_dim - p.split, p.split, p.scale, lane);
        }
        float* dst = p.dst + v * p.output_dim;
        if (p.subsample) {
            for (uint32_t o = lane; o < p.output_dim; o += 32) dst[o] = __fmul_rn(x[sw(__ldg(p.subsample + o))], p.rescale);
        } else {
            for (uint32_t o = lane; o < p.output_dim; o += 32) dst[o] = x[sw(o)];
        }
        __syncwarp();
    }
}

std::vector<uint32_t> transform_tables(const dab_transform* t) {
    std::vector<uint32_t> tables(t->signs0);
    tables.insert(tables.end(), t->signs1.begin(), t->signs1.end());
    tables.insert(tables.end(), t->subsample.begin(), t->subsample.end());
    tables.push_back(0);  // never empty
    return tables;
}

cudaError_t transform_rows(const dab_transform* t, const float* d_src, uint64_t n, float* d_dst, unsigned long long* d_first_nan) {
    if (n == 0) return cudaSuccess;
    const std::vector<uint32_t> tables = transform_tables(t);
    uint32_t* d_tables = nullptr;
    cudaError_t e = cudaMalloc(&d_tables, tables.size() * 4);
    if (e == cudaSuccess) e = cudaMemcpy(d_tables, tables.data(), tables.size() * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = transform_launch(t, d_tables, d_src, n, d_dst, d_first_nan, 0);
    cudaFree(d_tables);  // synchronizes with the kernel
    return e;
}

cudaError_t transform_launch(const dab_transform* t, const uint32_t* d_tables, const float* d_src, uint64_t n, float* d_dst,
                             unsigned long long* d_first_nan, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    TransformParams p;
    memset(&p, 0, sizeof(p));
    p.input_dim = t->input_dim;
    p.inner_dim = t->inner_dim;
    p.output_dim = t->output_dim;
    p.two_stages = t->kind == DAB_TRANSFORM_DOUBLE_HADAMARD;
    uint32_t split = 1;
    while (split <= t->inner_dim / 2) split <<= 1;  // the largest power of two <= inner_dim
    p.split = split;
    p.scale = 1.0f / sqrtf((float)split);                                                        // hadamard.rs:132
    p.rescale = t->subsampled ? sqrtf((float)t->inner_dim / (float)t->output_dim) : 1.0f;        // padding_hadamard.rs:262
    p.signs0 = d_tables;
    p.signs1 = d_tables + t->signs0.size();
    p.subsample = t->subsampled ? d_tables + t->signs0.size() + t->signs1.size() : nullptr;
    p.src = d_src;
    p.dst = d_dst;
    p.n = n;
    p.warp_floats = t->inner_dim + t->inner_dim / 8 + 8;  // sw(inner_dim - 1) < this
    p.first_nan = d_first_nan;
    int warps = 8;
    while (warps > 1 && (size_t)warps * p.warp_floats * 4 > 96 * 1024) warps >>= 1;
    const size_t smem = (size_t)warps * p.warp_floats * 4;
    cudaError_t e = cudaFuncSetAttribute(hadamard_transform_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) {
        const int grid = (int)std::min<uint64_t>((n + warps - 1) / warps, 132ull * 16);
        hadamard_transform_kernel<<<grid, warps * 32, smem, stream>>>(p);
        DAB_LAUNCHED();
        e = cudaGetLastError();
    }
    return e;
}

}  // namespace dab

using namespace dab;

static bool strictly_increasing(const uint32_t* v, uint32_t n) {
    for (uint32_t i = 1; i < n; ++i)
        if (v[i] <= v[i - 1]) return false;
    return true;
}

static bool bools_ok(const uint8_t* v, uint32_t n) {
    for (uint32_t i = 0; i < n; ++i)
        if (v[i] > 1) return false;
    return true;
}

extern "C" {

int dab_transform_create(dab_transform** out, int kind, uint32_t input_dim, uint32_t inner_dim, const uint8_t* signs0,
                         const uint8_t* signs1, const uint32_t* subsample, uint32_t n_subsample) {
    static const char* who = "dab_transform_create";
    if (!out) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL output handle", who);
    *out = nullptr;
    if (kind != DAB_TRANSFORM_PADDING_HADAMARD && kind != DAB_TRANSFORM_DOUBLE_HADAMARD)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: unknown transform kind %d", who, kind);
    if ((input_dim && !signs0) || (!subsample && n_subsample))
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL argument", who);
    if (kind == DAB_TRANSFORM_PADDING_HADAMARD) {
        // PaddingHadamard::try_from_parts (padding_hadamard.rs:137-173), in its order
        if (signs1) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: PaddingHadamard has one sign vector (signs1 must be NULL)", who);
        if (!bools_ok(signs0, input_dim))
            return fail(DAB_ERR_INVALID_ARGUMENT, "%s: an invalid sign representation was discovered (InvalidSignRepresentation)", who);
        if (input_dim > inner_dim) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: `signs` length exceeds `padded_dim` (SignsTooLong)", who);
        if (inner_dim == 0 || (inner_dim & (inner_dim - 1)))
            return fail(DAB_ERR_INVALID_ARGUMENT, "%s: padded dim is not a power of two (DimNotPowerOfTwo)", who);
        if (subsample) {
            if (!strictly_increasing(subsample, n_subsample))
                return fail(DAB_ERR_INVALID_ARGUMENT, "%s: subsample indices is not monotonic (SubsampleNotMonotonic)", who);
            if (n_subsample == 0) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: subsample indices cannot be empty (SubsampleEmpty)", who);
            if (subsample[n_subsample - 1] >= inner_dim)
                return fail(DAB_ERR_INVALID_ARGUMENT, "%s: last subsample index exceeded `padded_dim` (LastSubsampleTooLarge)", who);
        }
    } else {
        // DoubleHadamard::try_from_parts (double_hadamard.rs:146-206), in its order
        if (input_dim == 0) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: first signs stage cannot be empty (Signs0Empty)", who);
        if (!signs1 && inner_dim) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL argument", who);
        if (inner_dim < input_dim)
            return fail(DAB_ERR_INVALID_ARGUMENT, "%s: second sign stage must be at least as large as the first stage (Signs1TooSmall)", who);
        if (!bools_ok(signs0, input_dim)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: first signs stage has invalid coding (Signs0Invalid)", who);
        if (!bools_ok(signs1, inner_dim))
            return fail(DAB_ERR_INVALID_ARGUMENT, "%s: invalid sign representation for second stage (Signs1Invalid)", who);
        if (subsample) {
            if (!strictly_increasing(subsample, n_subsample))
                return fail(DAB_ERR_INVALID_ARGUMENT, "%s: subsample indices is not monotonic (SubsampleNotMonotonic)", who);
            if (n_subsample == 0)
                return fail(DAB_ERR_INVALID_ARGUMENT, "%s: subsample length must equal `target_dim` (InvalidSubsampleLength)", who);
            if (subsample[n_subsample - 1] >= inner_dim)
                return fail(DAB_ERR_INVALID_ARGUMENT, "%s: last subsample index exceeded intermediate dim (LastSubsampleTooLarge)", who);
        }
    }
    if (inner_dim > kMaxTransformDim)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: inner dimension %u exceeds %u, the largest vector a warp stages in shared memory", who,
                    inner_dim, kMaxTransformDim);
    dab_transform* t = new (std::nothrow) dab_transform;
    if (!t) return fail(DAB_ERR_OUT_OF_MEMORY, "%s: out of host memory", who);
    t->kind = kind;
    t->input_dim = input_dim;
    t->inner_dim = inner_dim;
    t->subsampled = subsample != nullptr;
    t->output_dim = t->subsampled ? n_subsample : inner_dim;
    for (uint32_t i = 0; i < input_dim; ++i) t->signs0.push_back(signs0[i] ? 0x80000000u : 0u);
    if (kind == DAB_TRANSFORM_DOUBLE_HADAMARD)
        for (uint32_t i = 0; i < inner_dim; ++i) t->signs1.push_back(signs1[i] ? 0x80000000u : 0u);
    if (subsample) t->subsample.assign(subsample, subsample + n_subsample);
    *out = t;
    return DAB_OK;
}

void dab_transform_destroy(dab_transform* t) { delete t; }

uint32_t dab_transform_input_dim(const dab_transform* t) { return t ? t->input_dim : 0; }

uint32_t dab_transform_output_dim(const dab_transform* t) { return t ? t->output_dim : 0; }

int dab_transform_apply(const dab_transform* t, int device, const float* src, uint64_t n, float* dst) {
    if (!t) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_transform_apply: NULL transform");
    if (n == 0) return DAB_OK;
    if ((!src && t->input_dim) || !dst) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_transform_apply: NULL argument");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(DAB_ERR_NO_DEVICE, "dab_transform_apply: no CUDA device visible");
    DAB_CUDA(cudaSetDevice(device));
    float *d_src = nullptr, *d_dst = nullptr;
    cudaError_t e = cudaMalloc(&d_src, std::max<uint64_t>(1, n * t->input_dim) * 4);
    if (e == cudaSuccess) e = cudaMalloc(&d_dst, n * t->output_dim * 4);
    if (e == cudaSuccess && t->input_dim) e = cudaMemcpy(d_src, src, n * t->input_dim * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = transform_rows(t, d_src, n, d_dst, nullptr);
    if (e == cudaSuccess) e = cudaMemcpy(dst, d_dst, n * t->output_dim * 4, cudaMemcpyDeviceToHost);
    int rc = DAB_OK;
    if (e != cudaSuccess) rc = fail(e == cudaErrorMemoryAllocation ? DAB_ERR_OUT_OF_MEMORY : DAB_ERR_CUDA, "dab_transform_apply: %s", cudaGetErrorString(e));
    cudaFree(d_src);
    cudaFree(d_dst);
    return rc;
}

}  // extern "C"
