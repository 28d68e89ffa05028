// minmax_index.cu — the MinMax store of an index: MinMaxElement<NBITS> as the VectorRepr of an index
// (diskann-providers/src/common/minmax_repr.rs:167-336), the way diskann-garnet runs it as its traversal store
// (quantization.rs:229-362, provider.rs:1170-1358): one compressed row per point, behind an optional Hadamard transform,
// so that dab_search_batch_minmax (search_kernel_pq.cu, MODE 2) can traverse over them.
//
// Host-facing rows use the canonical-front layout of Data<NBITS> (meta/vector.rs:377-392): MinMaxCompensation {dim u32,
// b, n, a, norm_squared} (20 bytes) then ceil(dim * NBITS / 8) bytes of dense codes, value i at bit i * NBITS.  On the
// device the codes are 16 B-aligned rows, zero padded (the traversal reads whole uint4 words), and {b, n, a,
// norm_squared} a separate float4 array; dim is the store's, checked on upload.  Rows and queries are compressed by
// the same launches as the standalone entry points (hadamard_transform_kernel, minmax_compress_kernel); the kernels here
// only widen index rows to f32 and split / join canonical rows.
#include "dab_common.cuh"
#include "distance_device.cuh"
#include "minmax.cuh"
#include "search_pq.cuh"
#include "transform.cuh"

#include <algorithm>
#include <new>

namespace dab {

namespace {

// T::as_f32: rows of `dim` elements, src_stride bytes apart -> dense [n][dim] f32
template <typename T>
__global__ void __launch_bounds__(256) mm_widen_kernel(const uint8_t* __restrict__ src, size_t src_stride, uint64_t n, uint32_t dim,
                                                       float* __restrict__ dst) {
    const uint64_t total = n * dim;
    for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t r = t / dim;
        dst[t] = to_f32(reinterpret_cast<const T*>(src + r * src_stride)[t - r * dim]);
    }
}

__device__ __forceinline__ uint32_t load_u32(const uint8_t* b) {
    return (uint32_t)b[0] | ((uint32_t)b[1] << 8) | ((uint32_t)b[2] << 16) | ((uint32_t)b[3] << 24);
}

// canonical rows -> device layout (one thread per byte of the padded code row).  The bits past dim * nbits in the last
// code byte are cleared: the reference's BitSlice never reads them, the integer cores here read whole words.
// first_bad (may be NULL): atomicMin of every row whose stored dim is not `dim`.
__global__ void __launch_bounds__(256) mm_split_kernel(const uint8_t* __restrict__ rows, uint64_t n, uint32_t row_bytes, uint32_t stride,
                                                       uint32_t dim, int nbits, uint8_t* __restrict__ codes, float4* __restrict__ meta,
                                                       unsigned long long* first_bad) {
    const uint32_t code_bytes = row_bytes - kMmMeta;
    const uint32_t tail_bits = (uint32_t)(((uint64_t)dim * nbits) & 7u);
    const uint64_t total = n * stride;
    for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t r = t / stride;
        const uint32_t b = (uint32_t)(t - r * stride);
        const uint8_t* src = rows + r * row_bytes;
        uint32_t v = 0;
        if (b < code_bytes) {
            v = src[kMmMeta + b];
            if (b + 1 == code_bytes && tail_bits) v &= (1u << tail_bits) - 1u;
        }
        codes[t] = (uint8_t)v;
        if (b == 0) {
            if (first_bad && load_u32(src) != dim) atomicMin(first_bad, (unsigned long long)r);
            meta[r] = make_float4(__uint_as_float(load_u32(src + 4)), __uint_as_float(load_u32(src + 8)), __uint_as_float(load_u32(src + 12)),
                                  __uint_as_float(load_u32(src + 16)));
        }
    }
}

__global__ void __launch_bounds__(256) mm_join_kernel(const uint8_t* __restrict__ codes, const float4* __restrict__ meta, uint64_t n,
                                                      uint32_t row_bytes, uint32_t stride, uint32_t dim, uint8_t* __restrict__ rows) {
    const uint64_t total = n * row_bytes;
    for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t r = t / row_bytes;
        const uint32_t b = (uint32_t)(t - r * row_bytes);
        uint8_t v;
        if (b < kMmMeta) {
            const float4 m = meta[r];
            const uint32_t w = b < 4 ? dim : __float_as_uint(b < 8 ? m.x : b < 12 ? m.y : b < 16 ? m.z : m.w);
            v = (uint8_t)(w >> (8 * (b & 3u)));
        } else {
            v = codes[r * stride + (b - kMmMeta)];
        }
        rows[t] = v;
    }
}

int grid_for(const dab_index* idx, uint64_t work) { return (int)std::max<uint64_t>(1, std::min<uint64_t>((work + 255) / 256, (uint64_t)idx->sm_count * 16)); }

int require_minmax(const dab_index* idx, const char* who) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", who);
    if (!idx->d_mm_codes || !idx->mm_nbits) return fail(DAB_ERR_NOT_READY, "%s: dab_upload_minmax has not been called", who);
    return DAB_OK;
}

// as_f32 of n rows of the index dtype (src_stride bytes apart) into dst [n][dim]
int widen_launch(dab_index* idx, const void* src, size_t src_stride, uint64_t n, float* dst) {
    const int grid = grid_for(idx, n * idx->dim);
    const uint8_t* s = (const uint8_t*)src;
    switch (idx->dtype) {
        case DAB_F32: mm_widen_kernel<float><<<grid, 256, 0, idx->stream>>>(s, src_stride, n, idx->dim, dst); break;
        case DAB_F16: mm_widen_kernel<__half><<<grid, 256, 0, idx->stream>>>(s, src_stride, n, idx->dim, dst); break;
        case DAB_I8: mm_widen_kernel<int8_t><<<grid, 256, 0, idx->stream>>>(s, src_stride, n, idx->dim, dst); break;
        default: mm_widen_kernel<uint8_t><<<grid, 256, 0, idx->stream>>>(s, src_stride, n, idx->dim, dst); break;
    }
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    return DAB_OK;
}

// as_f32 -> transform -> compress_into for n rows (src_stride bytes apart) into canonical rows [n][mm_row_bytes] in
// `canon`; *first_nan (device) takes the first row whose transformed vector holds a NaN.  `work` holds the f32 rows:
// n * (dim + out_dim) floats.  Queued on the index's stream.
int compress_rows(dab_index* idx, const void* src, size_t src_stride, uint64_t n, float* work, uint8_t* canon, unsigned long long* first_nan) {
    int rc;
    if ((rc = widen_launch(idx, src, src_stride, n, work))) return rc;
    const float* vec = work;
    if (idx->mm_transform) {
        float* out = work + n * idx->dim;
        DAB_CUDA(transform_launch(idx->mm_transform, idx->d_mm_tables, work, n, out, nullptr, idx->stream));
        vec = out;
    }
    MinMaxCompressParams p;
    int warps;
    size_t smem;
    mm_compress_setup(idx->mm_grid_scale, idx->mm_dim, idx->mm_nbits, n, p, warps, smem);  // fits: checked by dab_upload_minmax
    p.vectors = vec;
    p.rows = canon;
    p.first_nan = first_nan;
    DAB_CUDA(mm_compress_launch(p, warps, smem, idx->stream));
    return DAB_OK;
}

// the staging buffer of `n` rows through compress_rows and the split: f32 rows, canonical rows, the NaN flag
struct Staging {
    float* work;
    uint8_t* canon;
    unsigned long long* flag;
};

size_t staging_canon_off(const dab_index* idx, uint64_t n) { return round_up(n * (idx->dim + (idx->mm_transform ? idx->mm_dim : 0)) * 4, 256); }
size_t staging_flag_off(const dab_index* idx, uint64_t n) { return staging_canon_off(idx, n) + round_up(n * idx->mm_row_bytes, 256); }
size_t staging_bytes(const dab_index* idx, uint64_t n) { return staging_flag_off(idx, n) + 256; }

Staging staging_layout(const dab_index* idx, uint64_t n, uint8_t* base) {
    return Staging{(float*)base, base + staging_canon_off(idx, n), (unsigned long long*)(base + staging_flag_off(idx, n))};
}

}  // namespace

void minmax_release(dab_index* idx) {
    cudaFree(idx->d_mm_codes);
    cudaFree(idx->d_mm_meta);
    cudaFree(idx->d_mm_tables);
    delete idx->mm_transform;
    idx->d_mm_codes = nullptr;
    idx->d_mm_meta = nullptr;
    idx->d_mm_tables = nullptr;
    idx->mm_transform = nullptr;
    idx->mm_nbits = 0;
    idx->mm_ready = false;
}

int minmax_stage_queries(dab_index* idx, const void* d_queries, uint32_t nq, const uint8_t** d_qcodes, const float4** d_qmeta) {
    int rc;
    const size_t codes_off = staging_bytes(idx, nq), meta_off = codes_off + round_up((size_t)nq * idx->mm_stride, 256);
    if ((rc = idx->s_stage.reserve(meta_off + (size_t)nq * 16))) return rc;
    uint8_t* base = (uint8_t*)idx->s_stage.p;
    const Staging s = staging_layout(idx, nq, base);
    uint8_t* qcodes = base + codes_off;
    float4* qmeta = (float4*)(base + meta_off);
    DAB_CUDA(cudaMemsetAsync(s.flag, 0xFF, 8, idx->stream));
    if ((rc = compress_rows(idx, d_queries, (size_t)idx->dim * elem_size(idx->dtype), nq, s.work, s.canon, s.flag))) return rc;
    mm_split_kernel<<<grid_for(idx, (uint64_t)nq * idx->mm_stride), 256, 0, idx->stream>>>(s.canon, nq, idx->mm_row_bytes, idx->mm_stride,
                                                                                           idx->mm_dim, idx->mm_nbits, qcodes, qmeta, nullptr);
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    unsigned long long first_nan = ~0ull;
    DAB_CUDA(cudaMemcpyAsync(&first_nan, s.flag, 8, cudaMemcpyDeviceToHost, idx->stream));
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    if (first_nan != ~0ull)
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_search_batch_minmax: query %llu contains NaN after the transform (InputContainsNaN)", first_nan);
    *d_qcodes = qcodes;
    *d_qmeta = qmeta;
    return DAB_OK;
}

}  // namespace dab

using namespace dab;

static bool mm_width_ok(int nbits) { return nbits == 1 || nbits == 2 || nbits == 4 || nbits == 8; }

extern "C" {

int dab_upload_minmax(dab_index* idx, int nbits, float grid_scale, const dab_transform* t, const uint8_t* rows) {
    static const char* who = "dab_upload_minmax";
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", who);
    if (!mm_width_ok(nbits)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: nbits must be 1, 2, 4 or 8", who);
    if (!(grid_scale > 0.0f)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: grid_scale must be positive (num::Positive)", who);
    if (t && t->input_dim != idx->dim)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: the transform takes vectors of %u values, the index has %u", who, t->input_dim, idx->dim);
    const uint32_t out_dim = t ? t->output_dim : idx->dim;
    MinMaxCompressParams probe;
    int warps;
    size_t smem;
    if (!mm_compress_setup(grid_scale, out_dim, nbits, 1, probe, warps, smem))
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: rows of %u bytes do not fit the compressor's staging buffers", who, probe.row_bytes);
    DAB_CUDA(cudaSetDevice(idx->device));
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    minmax_release(idx);
    const uint64_t total = idx->n_total();
    idx->mm_dim = out_dim;
    idx->mm_row_bytes = probe.row_bytes;
    idx->mm_stride = (uint32_t)round_up(probe.row_bytes - kMmMeta, 16);
    idx->mm_grid_scale = grid_scale;
    if (t) {
        idx->mm_transform = new (std::nothrow) dab_transform(*t);
        if (!idx->mm_transform) return fail(DAB_ERR_OUT_OF_MEMORY, "%s: out of host memory", who);
        const std::vector<uint32_t> tables = transform_tables(t);
        DAB_CUDA(cudaMalloc(&idx->d_mm_tables, tables.size() * 4));
        DAB_CUDA(cudaMemcpy(idx->d_mm_tables, tables.data(), tables.size() * 4, cudaMemcpyHostToDevice));
    }
    DAB_CUDA(cudaMalloc(&idx->d_mm_codes, total * idx->mm_stride));
    DAB_CUDA(cudaMalloc(&idx->d_mm_meta, total * sizeof(float4)));
    idx->mm_nbits = nbits;
    if (!rows) {
        DAB_CUDA(cudaMemset(idx->d_mm_codes, 0, total * idx->mm_stride));
        DAB_CUDA(cudaMemset(idx->d_mm_meta, 0, total * sizeof(float4)));
        return DAB_OK;
    }
    // staged in slabs so that a 100M-point store does not need a second full copy on the device
    const uint64_t in_stride = idx->mm_row_bytes;
    const uint64_t slab = std::max<uint64_t>(1, std::min<uint64_t>(total, (256ull << 20) / in_stride));
    const size_t flag_off = round_up(slab * in_stride, 256);
    int rc;
    if ((rc = idx->s_stage.reserve(flag_off + 8))) return rc;
    uint8_t* stage = (uint8_t*)idx->s_stage.p;
    unsigned long long* d_bad = (unsigned long long*)(stage + flag_off);
    for (uint64_t first = 0; first < total; first += slab) {
        const uint64_t cnt = std::min(slab, total - first);
        DAB_CUDA(cudaMemcpyAsync(stage, rows + first * in_stride, cnt * in_stride, cudaMemcpyHostToDevice, idx->stream));
        DAB_CUDA(cudaMemsetAsync(d_bad, 0xFF, 8, idx->stream));
        mm_split_kernel<<<grid_for(idx, cnt * idx->mm_stride), 256, 0, idx->stream>>>(stage, cnt, idx->mm_row_bytes, idx->mm_stride, out_dim, nbits,
                                                                                       idx->d_mm_codes + first * idx->mm_stride,
                                                                                       idx->d_mm_meta + first, d_bad);
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
        unsigned long long bad = ~0ull;
        DAB_CUDA(cudaMemcpyAsync(&bad, d_bad, 8, cudaMemcpyDeviceToHost, idx->stream));
        DAB_CUDA(cudaStreamSynchronize(idx->stream));
        if (bad != ~0ull) {
            uint32_t stored;
            memcpy(&stored, rows + (first + bad) * in_stride, 4);
            return fail(DAB_ERR_INVALID_ARGUMENT, "%s: row %llu stores dim %u, the store's rows have %u (UnequalLengths)", who,
                        (unsigned long long)(first + bad), stored, out_dim);
        }
    }
    idx->mm_ready = true;
    return DAB_OK;
}

int dab_minmax_encode_all(dab_index* idx) {
    static const char* who = "dab_minmax_encode_all";
    int rc;
    if ((rc = require_minmax(idx, who))) return rc;
    if (!idx->vectors_ready) return fail(DAB_ERR_NOT_READY, "%s: vectors not uploaded", who);
    DAB_CUDA(cudaSetDevice(idx->device));
    idx->mm_ready = false;
    const uint64_t total = idx->n_total();
    const uint64_t per_row = (uint64_t)(idx->dim + (idx->mm_transform ? idx->mm_dim : 0)) * 4 + idx->mm_row_bytes;
    const uint64_t slab = std::max<uint64_t>(1, std::min<uint64_t>(total, (256ull << 20) / per_row));
    if ((rc = idx->s_stage.reserve(staging_bytes(idx, slab)))) return rc;
    const Staging s = staging_layout(idx, slab, (uint8_t*)idx->s_stage.p);
    for (uint64_t first = 0; first < total; first += slab) {
        const uint64_t cnt = std::min(slab, total - first);
        DAB_CUDA(cudaMemsetAsync(s.flag, 0xFF, 8, idx->stream));
        if ((rc = compress_rows(idx, idx->d_vectors + first * idx->row_stride, idx->row_stride, cnt, s.work, s.canon, s.flag))) return rc;
        mm_split_kernel<<<grid_for(idx, cnt * idx->mm_stride), 256, 0, idx->stream>>>(s.canon, cnt, idx->mm_row_bytes, idx->mm_stride, idx->mm_dim,
                                                                                      idx->mm_nbits, idx->d_mm_codes + first * idx->mm_stride,
                                                                                      idx->d_mm_meta + first, nullptr);
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
        unsigned long long first_nan = ~0ull;
        DAB_CUDA(cudaMemcpyAsync(&first_nan, s.flag, 8, cudaMemcpyDeviceToHost, idx->stream));
        DAB_CUDA(cudaStreamSynchronize(idx->stream));
        if (first_nan != ~0ull)
            return fail(DAB_ERR_INVALID_ARGUMENT, "%s: row %llu contains NaN after the transform (InputContainsNaN)", who,
                        (unsigned long long)(first + first_nan));
    }
    idx->mm_ready = true;
    return DAB_OK;
}

int dab_minmax_download(dab_index* idx, uint8_t* rows) {
    static const char* who = "dab_minmax_download";
    int rc;
    if ((rc = require_minmax(idx, who))) return rc;
    if (!rows) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: rows is NULL", who);
    if (!idx->mm_ready) return fail(DAB_ERR_NOT_READY, "%s: no rows (dab_upload_minmax with rows, or dab_minmax_encode_all)", who);
    DAB_CUDA(cudaSetDevice(idx->device));
    const uint64_t total = idx->n_total();
    const uint64_t out_stride = idx->mm_row_bytes;
    const uint64_t slab = std::max<uint64_t>(1, std::min<uint64_t>(total, (256ull << 20) / out_stride));
    if ((rc = idx->s_stage.reserve(slab * out_stride))) return rc;
    for (uint64_t first = 0; first < total; first += slab) {
        const uint64_t cnt = std::min(slab, total - first);
        mm_join_kernel<<<grid_for(idx, cnt * out_stride), 256, 0, idx->stream>>>(idx->d_mm_codes + first * idx->mm_stride, idx->d_mm_meta + first, cnt,
                                                                                 idx->mm_row_bytes, idx->mm_stride, idx->mm_dim, (uint8_t*)idx->s_stage.p);
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
        DAB_CUDA(cudaMemcpyAsync(rows + first * out_stride, idx->s_stage.p, cnt * out_stride, cudaMemcpyDeviceToHost, idx->stream));
        DAB_CUDA(cudaStreamSynchronize(idx->stream));
    }
    return DAB_OK;
}

}  // extern "C"
