// sq_index.cu — the scalar-quantized store of an index (providers inmem/scalar.rs SQStore<NBITS>,
// :60-258): dense N-bit codes + one f32 compensation per point, resident beside the graph so that
// dab_search_batch_sq (search_kernel_pq.cu, MODE 1) can traverse over them.
//
// Host-facing rows use the reference's canonical-front layout (meta/vector.rs:478-507): 4 bytes of
// f32 compensation followed by ceil(dim * nbits / 8) bytes of Dense-packed codes (bits/slice.rs:
// 261-323, value i at bit i * nbits) — what SQStore::set_quant_vector (:193-212) takes and what
// get_vector returns: a CodeStore with one f32 of header (code_store.cu holds the rows).
// sq_stage_queries compresses a search batch's queries into the same device layout before the
// traversal starts.
#include "dab_common.cuh"
#include "quant_device.cuh"
#include "search_pq.cuh"

#include <algorithm>

namespace dab {

namespace {

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

}  // namespace

int sq_encode_rows(const dab_index* idx, cudaStream_t stream, const uint8_t* src, size_t src_stride, uint64_t n, uint8_t* codes, float* comp) {
    const int grid = (int)std::min<uint64_t>((n + 127) / 128, (uint64_t)idx->sm_count * 16);
    const CodeStore& s = idx->sq;
#define DAB_SQ_ENCODE(T) \
    sq_encode_rows_kernel<T><<<grid, 128, 0, stream>>>(src, src_stride, n, idx->dim, idx->d_sq_shift, idx->sq_scale, s.nbits, s.stride, codes, comp)
    switch (idx->dtype) {
        case DAB_F32: DAB_SQ_ENCODE(float); break;
        case DAB_F16: DAB_SQ_ENCODE(__half); break;
        case DAB_I8: DAB_SQ_ENCODE(int8_t); break;
        default: DAB_SQ_ENCODE(uint8_t); break;
    }
#undef DAB_SQ_ENCODE
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    return DAB_OK;
}

size_t sq_stage_bytes(const dab_index* idx, uint32_t nq) { return stage_query_bytes(idx->sq, nq, (size_t)nq * idx->dim * 4); }

int sq_stage_queries(const dab_index* idx, cudaStream_t stream, Scratch& stage, const void* d_queries, uint32_t nq, const uint8_t** d_qcodes,
                     const float4** d_qmeta) {
    int rc;
    uint8_t* qcodes;
    float4* qmeta;
    if ((rc = stage_query_buffers(idx->sq, stage, nq, (size_t)nq * idx->dim * 4, &qcodes, &qmeta))) return rc;  // work: the f32 queries
    const bool rescale = idx->metric == DAB_INNER_PRODUCT && idx->sq_mean_norm != 0.0f;
    const int grid = (int)(((uint64_t)nq + 3) / 4);
    auto launch = [&](auto* queries) {
        sq_stage_kernel<<<grid, 128, 0, stream>>>(queries, nq, (int)idx->dim, idx->d_sq_shift, idx->sq_scale, idx->sq_mean_norm, rescale,
                                                  idx->sq.nbits, idx->sq.stride, (float*)stage.p, (uint32_t*)qcodes, qmeta);
    };
    switch (idx->dtype) {
        case DAB_F32: launch((const float*)d_queries); break;
        case DAB_F16: launch((const __half*)d_queries); break;
        case DAB_I8: launch((const int8_t*)d_queries); break;
        default: launch((const uint8_t*)d_queries); break;
    }
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    *d_qcodes = qcodes;
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
    int rc;
    if ((rc = retire_quantized_stores(idx))) return rc;  // batches in flight read the store
    ++idx->store_writes[STORE_SQ];
    store_release(idx->sq);
    cudaFree(idx->d_sq_shift);
    idx->d_sq_shift = nullptr;
    DAB_CUDA(cudaMalloc(&idx->d_sq_shift, (size_t)idx->dim * 4));
    DAB_CUDA(cudaMemcpyAsync(idx->d_sq_shift, shift, (size_t)idx->dim * 4, cudaMemcpyHostToDevice, idx->stream));  // see store_alloc
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    idx->sq_scale = scale;
    idx->sq_shift_square_norm = shift_square_norm;
    idx->sq_mean_norm = mean_norm;
    if ((rc = store_alloc(idx, idx->sq, nbits, idx->dim, false, 1))) return rc;  // the header: one f32 compensation
    return rows ? store_upload(idx, idx->sq, rows, "dab_upload_sq") : DAB_OK;
}

int dab_sq_encode_all(dab_index* idx) {
    int rc;
    if ((rc = store_require(idx, &dab_index::sq, "dab_upload_sq", "dab_sq_encode_all"))) return rc;
    if (!idx->vectors_ready) return fail(DAB_ERR_NOT_READY, "dab_sq_encode_all: vectors not uploaded");
    DAB_CUDA(cudaSetDevice(idx->device));
    ++idx->store_writes[STORE_SQ];
    if ((rc = sq_encode_rows(idx, idx->stream, idx->d_vectors, idx->row_stride, idx->n_total(), idx->sq.d_codes, idx->sq.d_meta))) return rc;
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    idx->sq.ready = true;
    return DAB_OK;
}

int dab_sq_download(dab_index* idx, uint8_t* rows) {
    int rc;
    if ((rc = store_require(idx, &dab_index::sq, "dab_upload_sq", "dab_sq_download"))) return rc;
    if (!rows) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_sq_download: rows is NULL");
    if (!idx->sq.ready) return fail(DAB_ERR_NOT_READY, "dab_sq_download: no rows (dab_upload_sq with rows, or dab_sq_encode_all)");
    DAB_CUDA(cudaSetDevice(idx->device));
    return store_download(idx, idx->sq, rows);
}

}  // extern "C"
