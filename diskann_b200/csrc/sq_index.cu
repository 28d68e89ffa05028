// sq_index.cu — the scalar-quantized store of an index (providers inmem/scalar.rs SQStore<NBITS>,
// :60-258): dense N-bit codes + one f32 compensation per point, resident beside the graph so that
// dab_search_batch_sq (search_kernel_pq.cu, MODE 1) can traverse over them.
//
// Host-facing rows use the reference's canonical-front layout (meta/vector.rs:478-507): 4 bytes of
// f32 compensation followed by ceil(dim * nbits / 8) bytes of Dense-packed codes (bits/slice.rs:
// 261-323, value i at bit i * nbits) — what SQStore::set_quant_vector (:193-212) takes and what
// get_vector returns.  On the device the codes are 16 B-aligned rows (zero padded, so the integer
// cores can run over whole words) and the compensations a separate array.  sq_stage_queries
// compresses a search batch's queries into the same device layout before the traversal starts.
#include "dab_common.cuh"
#include "quant_device.cuh"
#include "search_pq.cuh"

#include <algorithm>

namespace dab {

namespace {

// canonical rows -> device layout (one thread per byte of the padded code row)
__global__ void __launch_bounds__(256) sq_split_kernel(const uint8_t* __restrict__ rows, uint64_t n, uint32_t row_bytes,
                                                       uint32_t stride, uint8_t* __restrict__ codes, float* __restrict__ comp) {
    const uint64_t total = n * stride;
    for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t r = t / stride;
        const uint32_t b = (uint32_t)(t - r * stride);
        const uint8_t* src = rows + r * (4ull + row_bytes);
        codes[t] = b < row_bytes ? src[4 + b] : (uint8_t)0;
        if (b == 0) {
            uint32_t w = (uint32_t)src[0] | ((uint32_t)src[1] << 8) | ((uint32_t)src[2] << 16) | ((uint32_t)src[3] << 24);
            comp[r] = __uint_as_float(w);
        }
    }
}

__global__ void __launch_bounds__(256) sq_join_kernel(const uint8_t* __restrict__ codes, const float* __restrict__ comp, uint64_t n,
                                                      uint32_t row_bytes, uint32_t stride, uint8_t* __restrict__ rows) {
    const uint64_t out_stride = 4ull + row_bytes;
    const uint64_t total = n * out_stride;
    for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t r = t / out_stride;
        const uint32_t b = (uint32_t)(t - r * out_stride);
        rows[t] = b < 4 ? (uint8_t)(__float_as_uint(comp[r]) >> (8 * b)) : codes[r * stride + (b - 4)];
    }
}

// SQStore::set_vector (providers inmem/scalar.rs:150-175): as_f32, then ScalarQuantizer::compress
// (scalar/quantizer.rs:190-239) with the compensation callback (:407-430).  The compensation is a
// sequential FMA chain over the dimensions, so one thread owns one row and packs its words as it goes.
template <typename T>
__global__ void __launch_bounds__(128) sq_encode_rows_kernel(const uint8_t* __restrict__ vectors, size_t row_stride, uint64_t n,
                                                             uint32_t dim, const float* __restrict__ shift, float scale, int nbits,
                                                             uint32_t stride, uint8_t* __restrict__ codes, float* __restrict__ comp) {
    const float maxv = (float)((1u << nbits) - 1u);
    const float inverse_scale = __fdiv_rn(maxv, scale);
    const float inverse_bit_scale = __fdiv_rn(1.0f, maxv);
    const uint32_t per_word = 32u / (uint32_t)nbits;
    for (uint64_t v = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; v < n; v += (uint64_t)gridDim.x * blockDim.x) {
        const T* row = reinterpret_cast<const T*>(vectors + v * row_stride);
        uint32_t* out = reinterpret_cast<uint32_t*>(codes + v * stride);
        float dot = 0.0f;
        uint32_t acc = 0, filled = 0, word = 0;
        for (uint32_t i = 0; i < dim; ++i) {
            const float s = __ldg(shift + i);
            const float code = sq_code(to_f32(row[i]), s, inverse_scale, maxv);
            dot = __fmaf_rn(code, s, dot);
            acc |= (code != code ? 0u : (uint32_t)code) << (filled * (uint32_t)nbits);
            if (++filled == per_word) {
                out[word++] = acc;
                acc = 0;
                filled = 0;
            }
        }
        if (filled) out[word++] = acc;
        for (; word < (stride >> 2); ++word) out[word] = 0;
        comp[v] = sq_compensation(scale, inverse_bit_scale, dot);
    }
}

// SQStore::query_computer (:227-253): as_f32, for InnerProduct the rescale to the store's mean norm, then the same
// compression as the rows.  One warp per query in `work` (its f32 copy): the codes in parallel, the norm and the
// compensation chain on lane 0; meta.x takes the compensation.
template <typename T>
__global__ void __launch_bounds__(128) sq_stage_kernel(const T* __restrict__ queries, uint32_t nq, int dim, const float* __restrict__ shift,
                                                       float scale, float mean_norm, bool rescale, int nbits, uint32_t stride,
                                                       float* __restrict__ work, uint32_t* __restrict__ codes, float4* __restrict__ meta) {
    const int lane = threadIdx.x & 31;
    const uint32_t q = blockIdx.x * 4u + (threadIdx.x >> 5);
    if (q >= nq) return;
    float* qf = work + (size_t)q * dim;
    for (int e = lane; e < dim; e += 32) qf[e] = to_f32(queries[(size_t)q * dim + e]);
    __syncwarp();
    // rescale (scalar/quantizer.rs:300-310): InnerProduct::evaluate(x, x), sqrt, x *= to_norm / norm
    if (rescale) {
        float norm = 0.0f;
        if (lane == 0) norm = __fsqrt_rn(thread_simd_l2ip<KIND_IP>(qf, qf, dim));
        norm = __shfl_sync(kFull, norm, 0);
        if (norm != 0.0f) {
            const float sc = __fdiv_rn(mean_norm, norm);
            for (int e = lane; e < dim; e += 32) qf[e] = __fmul_rn(qf[e], sc);
        }
        __syncwarp();
    }
    // ScalarQuantizer::compress: codes in parallel ...
    const float maxv = (float)((1u << nbits) - 1u);
    const float inverse_scale = __fdiv_rn(maxv, scale);
    for (int e = lane; e < dim; e += 32) qf[e] = sq_code(qf[e], __ldg(shift + e), inverse_scale, maxv);
    __syncwarp();
    // ... the compensation is one sequential FMA chain over the dimensions
    if (lane == 0) {
        float dot = 0.0f;
        for (int e = 0; e < dim; ++e) dot = __fmaf_rn(qf[e], __ldg(shift + e), dot);
        meta[q] = make_float4(sq_compensation(scale, __fdiv_rn(1.0f, maxv), dot), 0.0f, 0.0f, 0.0f);
    }
    // dense packing, value i at bit i * nbits (bits/slice.rs:261-305); padding words are zero
    const uint32_t per_word = 32u / (uint32_t)nbits;
    for (uint32_t wd = lane; wd < (stride >> 2); wd += 32) {
        uint32_t acc = 0;
        for (uint32_t j = 0; j < per_word; ++j) {
            const uint32_t e = wd * per_word + j;
            if (e < (uint32_t)dim) {
                const float c = qf[e];
                acc |= (c != c ? 0u : (uint32_t)c) << (j * (uint32_t)nbits);
            }
        }
        codes[(size_t)q * (stride >> 2) + wd] = acc;
    }
}

int require_sq(const dab_index* idx, const char* who) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", who);
    if (!idx->d_sq_codes || !idx->sq_nbits) return fail(DAB_ERR_NOT_READY, "%s: dab_upload_sq has not been called", who);
    return DAB_OK;
}

}  // namespace

int sq_stage_queries(dab_index* idx, const void* d_queries, uint32_t nq, const uint8_t** d_qcodes, const float4** d_qmeta) {
    int rc;
    const size_t codes_off = round_up((size_t)nq * idx->dim * 4, 256), meta_off = codes_off + round_up((size_t)nq * idx->sq_stride, 256);
    if ((rc = idx->s_stage.reserve(meta_off + (size_t)nq * 16))) return rc;
    uint8_t* base = (uint8_t*)idx->s_stage.p;
    uint32_t* qcodes = (uint32_t*)(base + codes_off);
    float4* qmeta = (float4*)(base + meta_off);
    const bool rescale = idx->metric == DAB_INNER_PRODUCT && idx->sq_mean_norm != 0.0f;
    const int grid = (int)(((uint64_t)nq + 3) / 4);
    auto launch = [&](auto* queries) {
        sq_stage_kernel<<<grid, 128, 0, idx->stream>>>(queries, nq, (int)idx->dim, idx->d_sq_shift, idx->sq_scale, idx->sq_mean_norm, rescale,
                                                       idx->sq_nbits, idx->sq_stride, (float*)base, qcodes, qmeta);
    };
    switch (idx->dtype) {
        case DAB_F32: launch((const float*)d_queries); break;
        case DAB_F16: launch((const __half*)d_queries); break;
        case DAB_I8: launch((const int8_t*)d_queries); break;
        default: launch((const uint8_t*)d_queries); break;
    }
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    *d_qcodes = (const uint8_t*)qcodes;
    *d_qmeta = qmeta;
    return DAB_OK;
}

}  // namespace dab

using namespace dab;

extern "C" {

int dab_upload_sq(dab_index* idx, int nbits, const float* shift, float scale, float shift_square_norm, float mean_norm,
                  const uint8_t* rows) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_upload_sq: idx is NULL");
    if (nbits != 1 && nbits != 2 && nbits != 4 && nbits != 8) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_upload_sq: nbits must be 1, 2, 4 or 8");
    if (!shift) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_upload_sq: shift is NULL");
    if (!(scale > 0.0f)) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_upload_sq: scale must be positive");  // ScalarQuantizer::new
    DAB_CUDA(cudaSetDevice(idx->device));
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    cudaFree(idx->d_sq_shift);
    cudaFree(idx->d_sq_codes);
    cudaFree(idx->d_sq_comp);
    idx->d_sq_shift = nullptr;
    idx->d_sq_codes = nullptr;
    idx->d_sq_comp = nullptr;
    idx->sq_codes_ready = false;
    idx->sq_nbits = 0;
    const uint64_t total = idx->n_total();
    const uint32_t row_bytes = (uint32_t)(((uint64_t)idx->dim * nbits + 7) / 8);
    const uint32_t stride = (uint32_t)round_up(row_bytes, 16);
    DAB_CUDA(cudaMalloc(&idx->d_sq_shift, (size_t)idx->dim * 4));
    DAB_CUDA(cudaMalloc(&idx->d_sq_codes, total * stride));
    DAB_CUDA(cudaMalloc(&idx->d_sq_comp, total * 4));
    DAB_CUDA(cudaMemcpy(idx->d_sq_shift, shift, (size_t)idx->dim * 4, cudaMemcpyHostToDevice));
    idx->sq_nbits = nbits;
    idx->sq_scale = scale;
    idx->sq_shift_square_norm = shift_square_norm;
    idx->sq_mean_norm = mean_norm;
    idx->sq_row_bytes = row_bytes;
    idx->sq_stride = stride;
    if (rows) {
        // staged in slabs so that a 100M-point store does not need a second full copy on the device
        const uint64_t in_stride = 4ull + row_bytes;
        const uint64_t slab = std::max<uint64_t>(1, std::min<uint64_t>(total, (256ull << 20) / in_stride));
        int rc;
        if ((rc = idx->s_queries.reserve(slab * in_stride))) return rc;
        for (uint64_t first = 0; first < total; first += slab) {
            const uint64_t cnt = std::min(slab, total - first);
            DAB_CUDA(cudaMemcpyAsync(idx->s_queries.p, rows + first * in_stride, cnt * in_stride, cudaMemcpyHostToDevice, idx->stream));
            const int grid = (int)std::min<uint64_t>((cnt * stride + 255) / 256, (uint64_t)idx->sm_count * 16);
            sq_split_kernel<<<grid, 256, 0, idx->stream>>>((const uint8_t*)idx->s_queries.p, cnt, row_bytes, stride,
                                                           idx->d_sq_codes + first * stride, idx->d_sq_comp + first);
            DAB_LAUNCHED();
            DAB_CUDA(cudaGetLastError());
            DAB_CUDA(cudaStreamSynchronize(idx->stream));
        }
        idx->sq_codes_ready = true;
    } else {
        DAB_CUDA(cudaMemset(idx->d_sq_codes, 0, total * stride));
        DAB_CUDA(cudaMemset(idx->d_sq_comp, 0, total * 4));
    }
    return DAB_OK;
}

int dab_sq_encode_all(dab_index* idx) {
    int rc;
    if ((rc = require_sq(idx, "dab_sq_encode_all"))) return rc;
    if (!idx->vectors_ready) return fail(DAB_ERR_NOT_READY, "dab_sq_encode_all: vectors not uploaded");
    DAB_CUDA(cudaSetDevice(idx->device));
    const uint64_t total = idx->n_total();
    const int grid = (int)std::min<uint64_t>((total + 127) / 128, (uint64_t)idx->sm_count * 16);
#define DAB_SQ_ENCODE(T)                                                                                                       \
    sq_encode_rows_kernel<T><<<grid, 128, 0, idx->stream>>>(idx->d_vectors, idx->row_stride, total, idx->dim, idx->d_sq_shift, \
                                                            idx->sq_scale, idx->sq_nbits, idx->sq_stride, idx->d_sq_codes, idx->d_sq_comp)
    switch (idx->dtype) {
        case DAB_F32: DAB_SQ_ENCODE(float); break;
        case DAB_F16: DAB_SQ_ENCODE(__half); break;
        case DAB_I8: DAB_SQ_ENCODE(int8_t); break;
        default: DAB_SQ_ENCODE(uint8_t); break;
    }
#undef DAB_SQ_ENCODE
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    idx->sq_codes_ready = true;
    return DAB_OK;
}

int dab_sq_download(dab_index* idx, uint8_t* rows) {
    int rc;
    if ((rc = require_sq(idx, "dab_sq_download"))) return rc;
    if (!rows) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_sq_download: rows is NULL");
    if (!idx->sq_codes_ready) return fail(DAB_ERR_NOT_READY, "dab_sq_download: no rows (dab_upload_sq with rows, or dab_sq_encode_all)");
    DAB_CUDA(cudaSetDevice(idx->device));
    const uint64_t total = idx->n_total();
    const uint64_t out_stride = 4ull + idx->sq_row_bytes;
    const uint64_t slab = std::max<uint64_t>(1, std::min<uint64_t>(total, (256ull << 20) / out_stride));
    if ((rc = idx->s_queries.reserve(slab * out_stride))) return rc;
    for (uint64_t first = 0; first < total; first += slab) {
        const uint64_t cnt = std::min(slab, total - first);
        const int grid = (int)std::min<uint64_t>((cnt * out_stride + 255) / 256, (uint64_t)idx->sm_count * 16);
        sq_join_kernel<<<grid, 256, 0, idx->stream>>>(idx->d_sq_codes + first * idx->sq_stride, idx->d_sq_comp + first, cnt,
                                                      idx->sq_row_bytes, idx->sq_stride, (uint8_t*)idx->s_queries.p);
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
        DAB_CUDA(cudaMemcpyAsync(rows + first * out_stride, idx->s_queries.p, cnt * out_stride, cudaMemcpyDeviceToHost, idx->stream));
        DAB_CUDA(cudaStreamSynchronize(idx->stream));
    }
    return DAB_OK;
}

}  // extern "C"
