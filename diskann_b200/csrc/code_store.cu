// code_store.cu — the packed-code stores of an index (CodeStore, dab_common.cuh: the SQ store of sq_index.cu and the
// MinMax store of minmax_index.cu): allocation, the split of canonical-front rows into the device layout and the join
// back, the slabbed host upload and download, and the as_f32 widening of index rows that the encoders start from.
#include "dab_common.cuh"
#include "distance_device.cuh"

#include <algorithm>

namespace dab {

namespace {

// T::as_f32: rows of `dim` elements, src_stride bytes apart -> dense [n][dim] f32
template <typename T>
__global__ void __launch_bounds__(256) widen_kernel(const uint8_t* __restrict__ src, size_t src_stride, uint64_t n, uint32_t dim,
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
// first_bad (may be NULL): atomicMin of every row whose dim word is not s.dim.
__global__ void __launch_bounds__(256) split_kernel(const CodeStore s, const uint8_t* __restrict__ rows, uint64_t n, uint8_t* __restrict__ codes,
                                                    float* __restrict__ meta, unsigned long long* first_bad) {
    const uint32_t head = s.header_bytes(), code_bytes = s.row_bytes - head;
    const uint32_t tail_bits = (uint32_t)(((uint64_t)s.dim * s.nbits) & 7u);
    const uint64_t total = n * s.stride;
    for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t r = t / s.stride;
        const uint32_t b = (uint32_t)(t - r * s.stride);
        const uint8_t* src = rows + r * s.row_bytes;
        uint32_t v = 0;
        if (b < code_bytes) {
            v = src[head + b];
            if (b + 1 == code_bytes && tail_bits) v &= (1u << tail_bits) - 1u;
        }
        codes[t] = (uint8_t)v;
        if (b == 0) {
            if (s.dim_word) {
                if (first_bad && load_u32(src) != s.dim) atomicMin(first_bad, (unsigned long long)r);
                src += 4;
            }
            for (uint32_t j = 0; j < s.meta_words; ++j) meta[r * s.meta_words + j] = __uint_as_float(load_u32(src + 4 * j));
        }
    }
}

__global__ void __launch_bounds__(256) join_kernel(const CodeStore s, const uint8_t* __restrict__ codes, const float* __restrict__ meta, uint64_t n,
                                                   uint8_t* __restrict__ rows) {
    const uint32_t head = s.header_bytes(), lead = s.dim_word ? 4u : 0u;
    const uint64_t total = n * s.row_bytes;
    for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t r = t / s.row_bytes;
        const uint32_t b = (uint32_t)(t - r * s.row_bytes);
        uint8_t v;
        if (b < head) {
            const uint32_t w = b < lead ? s.dim : __float_as_uint(meta[r * s.meta_words + (b - lead) / 4]);
            v = (uint8_t)(w >> (8 * (b & 3u)));
        } else {
            v = codes[r * s.stride + (b - head)];
        }
        rows[t] = v;
    }
}

// rows per slab of the host copies: a 100M-point store does not need a second full copy on the device
uint64_t slab_rows(const dab_index* idx, uint64_t row_bytes) {
    return std::max<uint64_t>(1, std::min<uint64_t>(idx->n_total(), (256ull << 20) / row_bytes));
}

}  // namespace

int grid_for(const dab_index* idx, uint64_t work) { return (int)std::max<uint64_t>(1, std::min<uint64_t>((work + 255) / 256, (uint64_t)idx->sm_count * 16)); }

void store_release(CodeStore& s) {
    cudaFree(s.d_codes);
    cudaFree(s.d_meta);
    s = CodeStore{};
}

int store_alloc(dab_index* idx, CodeStore& s, int nbits, uint32_t dim, bool dim_word, uint32_t meta_words) {
    store_release(s);
    const uint64_t total = idx->n_total();
    const uint32_t code_bytes = (uint32_t)(((uint64_t)dim * nbits + 7) / 8);
    s.dim = dim;
    s.dim_word = dim_word;
    s.meta_words = meta_words;
    s.row_bytes = s.header_bytes() + code_bytes;
    s.stride = (uint32_t)round_up(code_bytes, 16);
    DAB_CUDA(cudaMalloc(&s.d_codes, total * s.stride));
    DAB_CUDA(cudaMalloc(&s.d_meta, total * meta_words * 4));
    // on the index's stream, which does not wait for the legacy default stream: a cudaMemset there could still be
    // clearing the arrays while an encode on idx->stream writes them.  The uploads of an index's parameters (PQ table,
    // SQ shift, MinMax transform tables) likewise copy on idx->stream.
    DAB_CUDA(cudaMemsetAsync(s.d_codes, 0, total * s.stride, idx->stream));
    DAB_CUDA(cudaMemsetAsync(s.d_meta, 0, total * meta_words * 4, idx->stream));
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    s.nbits = nbits;  // set up only once both arrays exist
    return DAB_OK;
}

int store_require(const dab_index* idx, CodeStore dab_index::*store, const char* upload, const char* who) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", who);
    const CodeStore& s = idx->*store;
    if (!s.d_codes || !s.nbits) return fail(DAB_ERR_NOT_READY, "%s: %s has not been called", who, upload);
    return DAB_OK;
}

int store_split(const dab_index* idx, cudaStream_t stream, const CodeStore& s, const uint8_t* rows, uint64_t n, uint8_t* codes, float* meta,
                unsigned long long* first_bad) {
    split_kernel<<<grid_for(idx, n * s.stride), 256, 0, stream>>>(s, rows, n, codes, meta, first_bad);
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    return DAB_OK;
}

int store_upload(dab_index* idx, CodeStore& s, const uint8_t* rows, const char* who) {
    const uint64_t total = idx->n_total(), slab = slab_rows(idx, s.row_bytes);
    const size_t flag_off = round_up(slab * s.row_bytes, 256);
    int rc;
    if ((rc = idx->s_stage.reserve(flag_off + 8))) return rc;
    uint8_t* stage = (uint8_t*)idx->s_stage.p;
    unsigned long long* d_bad = (unsigned long long*)(stage + flag_off);
    for (uint64_t first = 0; first < total; first += slab) {
        const uint64_t cnt = std::min(slab, total - first);
        DAB_CUDA(cudaMemcpyAsync(stage, rows + first * s.row_bytes, cnt * s.row_bytes, cudaMemcpyHostToDevice, idx->stream));
        DAB_CUDA(cudaMemsetAsync(d_bad, 0xFF, 8, idx->stream));
        if ((rc = store_split(idx, idx->stream, s, stage, cnt, s.d_codes + first * s.stride, s.d_meta + first * s.meta_words, d_bad))) return rc;
        unsigned long long bad = ~0ull;
        DAB_CUDA(cudaMemcpyAsync(&bad, d_bad, 8, cudaMemcpyDeviceToHost, idx->stream));
        DAB_CUDA(cudaStreamSynchronize(idx->stream));
        if (bad != ~0ull) {
            uint32_t stored;
            memcpy(&stored, rows + (first + bad) * s.row_bytes, 4);
            return fail(DAB_ERR_INVALID_ARGUMENT, "%s: row %llu stores dim %u, the store's rows have %u (UnequalLengths)", who,
                        (unsigned long long)(first + bad), stored, s.dim);
        }
    }
    s.ready = true;
    return DAB_OK;
}

int store_download(dab_index* idx, const CodeStore& s, uint8_t* rows) {
    const uint64_t total = idx->n_total(), slab = slab_rows(idx, s.row_bytes);
    int rc;
    if ((rc = idx->s_stage.reserve(slab * s.row_bytes))) return rc;
    for (uint64_t first = 0; first < total; first += slab) {
        const uint64_t cnt = std::min(slab, total - first);
        join_kernel<<<grid_for(idx, cnt * s.row_bytes), 256, 0, idx->stream>>>(s, s.d_codes + first * s.stride, s.d_meta + first * s.meta_words, cnt,
                                                                                (uint8_t*)idx->s_stage.p);
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
        DAB_CUDA(cudaMemcpyAsync(rows + first * s.row_bytes, idx->s_stage.p, cnt * s.row_bytes, cudaMemcpyDeviceToHost, idx->stream));
        DAB_CUDA(cudaStreamSynchronize(idx->stream));
    }
    return DAB_OK;
}

size_t stage_query_bytes(const CodeStore& s, uint32_t nq, size_t work) {
    return round_up(work, 256) + round_up((size_t)nq * s.stride, 256) + (size_t)nq * 16;
}

int stage_query_buffers(const CodeStore& s, Scratch& stage, uint32_t nq, size_t work, uint8_t** codes, float4** meta) {
    const size_t codes_off = round_up(work, 256), meta_off = codes_off + round_up((size_t)nq * s.stride, 256);
    int rc;
    if ((rc = stage.reserve(stage_query_bytes(s, nq, work)))) return rc;
    uint8_t* base = (uint8_t*)stage.p;
    *codes = base + codes_off;
    *meta = (float4*)(base + meta_off);
    return DAB_OK;
}

int widen_rows(const dab_index* idx, cudaStream_t stream, const void* src, size_t src_stride, uint64_t n, float* dst) {
    const int grid = grid_for(idx, n * idx->dim);
    const uint8_t* s = (const uint8_t*)src;
    switch (idx->dtype) {
        case DAB_F32: widen_kernel<float><<<grid, 256, 0, stream>>>(s, src_stride, n, idx->dim, dst); break;
        case DAB_F16: widen_kernel<__half><<<grid, 256, 0, stream>>>(s, src_stride, n, idx->dim, dst); break;
        case DAB_I8: widen_kernel<int8_t><<<grid, 256, 0, stream>>>(s, src_stride, n, idx->dim, dst); break;
        default: widen_kernel<uint8_t><<<grid, 256, 0, stream>>>(s, src_stride, n, idx->dim, dst); break;
    }
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    return DAB_OK;
}

}  // namespace dab
