// pq_train.cu — PQ codebook training on the device: per chunk k-means++ seeding followed by Lloyd
// iterations, then encoding of every stored row.
//
// Restates the training the reference benchmark runs before a quantized build
// (diskann-providers/src/index/diskann_async.rs:61-89 train_pq -> model/pq/pq_construction.rs:163-243
// -> diskann-quantization/src/product/train.rs) with the arithmetic in the reference's order, so the
// result is bit-identical to a sequential CPU run of the same algorithm for the same random draws:
//   * square norms: algorithms/kmeans/common.rs (8-lane accumulators, zero-filled remainder, sum_tree);
//   * k-means++: plusplus.rs:238-320, 381-498 — d = (norm_i + norm_c) + (-2 * dot) with dot an FMA
//     chain over the dimensions, running minimum with `<`; the minima enter an f64 rolling sum
//     block by block (16 rows, pairs (j, j + 8)); the winner is the first row whose f64 prefix sum
//     reaches the threshold (and d > 0, not yet picked).  Both f64 sums are SEQUENTIAL in the
//     reference; one thread per chunk runs them over shared-memory staged data so that no
//     re-association can change a pick;
//   * Lloyd: lloyds.rs:27-330 (assignment: n_c - s - s + n_i, first minimum in centre order),
//     lloyds.rs:345-366 (centroid = f64 sum in DATA ORDER / max(count, 1)): one warp per
//     (chunk, centre) walks the assignment array in order, lane = dimension.
// The random draws come from SplitMix64(seed + chunk) (Rust's StdRng is not restated).
// This is setup work (once per index), not the search hot path: plain CUDA cores, no tensor cores —
// a chunk is 4-dimensional for the headline configuration (32 chunks of a 128-d vector).
#include "dab_common.cuh"
#include "distance_device.cuh"

#include <algorithm>
#include <vector>

namespace dab {

namespace {

__device__ __forceinline__ float tree8_local(const float (&v)[8]) {
    return __fadd_rn(__fadd_rn(__fadd_rn(v[0], v[4]), __fadd_rn(v[2], v[6])), __fadd_rn(__fadd_rn(v[1], v[5]), __fadd_rn(v[3], v[7])));
}

// common.rs square_norm, one thread
__device__ float square_norm_ref(const float* __restrict__ x, int len) {
    float s[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    int i = 0;
    if (i + 32 <= len) {
        float a[4][8];
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int l = 0; l < 8; ++l) a[k][l] = 0.0f;
        while (i + 32 <= len) {
#pragma unroll
            for (int k = 0; k < 4; ++k)
#pragma unroll
                for (int l = 0; l < 8; ++l) a[k][l] = __fmaf_rn(x[i + 8 * k + l], x[i + 8 * k + l], a[k][l]);
            i += 32;
        }
#pragma unroll
        for (int l = 0; l < 8; ++l) s[l] = __fadd_rn(__fadd_rn(a[0][l], a[1][l]), __fadd_rn(a[2][l], a[3][l]));
    }
    while (i + 8 <= len) {
#pragma unroll
        for (int l = 0; l < 8; ++l) s[l] = __fmaf_rn(x[i + l], x[i + l], s[l]);
        i += 8;
    }
    const int rem = len - i;
    if (rem) {
#pragma unroll
        for (int l = 0; l < 8; ++l) {
            const float v = l < rem ? x[i + l] : 0.0f;
            s[l] = __fmaf_rn(v, v, s[l]);
        }
    }
    return tree8_local(s);
}

__device__ __forceinline__ float dot_chain(const float* __restrict__ a, const float* __restrict__ b, int len) {
    float s = 0.0f;
    for (int d = 0; d < len; ++d) s = __fmaf_rn(a[d], b[d], s);
    return s;
}

struct TrainParams {
    const float* data;   // [n][dim]
    uint64_t n;
    uint32_t dim, n_chunks, n_centers;
    const uint32_t* offsets;
    float* pivots;       // [n_centers][dim]
    float* norms;        // [n_chunks][n]
    float* mins;         // [n_chunks][n]
    double* block_sums;  // [n_chunks][nblk16]
    uint64_t nblk16;
    uint8_t* picked;     // [n_chunks][n]
    uint64_t* rng;       // [n_chunks] SplitMix64 state
    float* prev_norm;    // [n_chunks]
    uint32_t* selected;  // [n_chunks] centres seeded so far
    uint32_t* assign;    // [n_chunks][n]
    float* cnorm;        // [n_chunks][n_centers]
};

__global__ void norms_kernel(const TrainParams p) {
    const uint32_t ch = blockIdx.y;
    const int lo = (int)p.offsets[ch], len = (int)(p.offsets[ch + 1] - p.offsets[ch]);
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < p.n; i += (uint64_t)gridDim.x * blockDim.x)
        p.norms[(size_t)ch * p.n + i] = square_norm_ref(p.data + i * p.dim + lo, len);
}

__device__ __forceinline__ uint64_t splitmix_next(uint64_t& s) {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// first centre of every chunk: uniform row; also resets the per-chunk state
__global__ void pp_init_kernel(const TrainParams p, uint64_t seed) {
    const uint32_t ch = blockIdx.x;
    const int lo = (int)p.offsets[ch], len = (int)(p.offsets[ch + 1] - p.offsets[ch]);
    __shared__ uint64_t first;
    if (threadIdx.x == 0) {
        uint64_t s = seed + ch;
        const uint64_t r = splitmix_next(s);
        first = (uint64_t)__umul64hi(r, p.n);
        p.rng[ch] = s;
        p.prev_norm[ch] = p.norms[(size_t)ch * p.n + first];
        p.selected[ch] = 1;
        p.picked[(size_t)ch * p.n + first] = 1;
    }
    __syncthreads();
    for (uint32_t t = threadIdx.x; t < p.n_centers * (uint32_t)len; t += blockDim.x) {
        const uint32_t c = t / len, d = t % len;
        p.pivots[(size_t)c * p.dim + lo + d] = c == 0 ? p.data[first * p.dim + lo + d] : 0.0f;
    }
}

// update_distances against centre cur-1; one thread per block of 16 rows
__global__ void pp_update_kernel(const TrainParams p, uint32_t cur) {
    const uint32_t ch = blockIdx.y;
    if (p.selected[ch] != cur) return;  // this chunk stopped seeding (insufficient diversity)
    const int lo = (int)p.offsets[ch], len = (int)(p.offsets[ch + 1] - p.offsets[ch]);
    const float* last = p.pivots + (size_t)(cur - 1) * p.dim + lo;
    const float pn = p.prev_norm[ch];
    float* mins = p.mins + (size_t)ch * p.n;
    const float* norms = p.norms + (size_t)ch * p.n;
    for (uint64_t b = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; b < p.nblk16; b += (uint64_t)gridDim.x * blockDim.x) {
        float cur_d[16];
#pragma unroll
        for (int l = 0; l < 16; ++l) {
            const uint64_t i = b * 16 + l;
            if (i < p.n) {
                const float inter = __fmul_rn(dot_chain(p.data + i * p.dim + lo, last, len), -2.0f);
                const float d = __fadd_rn(__fadd_rn(norms[i], pn), inter);
                float m = cur == 1 ? __int_as_float(0x7F800000) : mins[i];
                if (d < m) m = d;
                mins[i] = m;
                cur_d[l] = m;
            } else {
                cur_d[l] = 0.0f;
            }
        }
        double blk = 0.0;
#pragma unroll
        for (int j = 0; j < 8; ++j) blk = __dadd_rn(blk, __dadd_rn((double)cur_d[j], (double)cur_d[8 + j]));
        p.block_sums[(size_t)ch * p.nblk16 + b] = blk;
    }
}

// one CTA per chunk: sequential f64 total, threshold, sequential f64 prefix scan, copy the winner
__global__ void __launch_bounds__(256) pp_select_kernel(const TrainParams p, uint32_t cur) {
    constexpr int kStage = 4096;
    __shared__ double sd[kStage];
    __shared__ double s_total;
    __shared__ long long s_win;
    __shared__ double s_roll;
    const uint32_t ch = blockIdx.x;
    if (p.selected[ch] != cur) return;
    const int lo = (int)p.offsets[ch], len = (int)(p.offsets[ch + 1] - p.offsets[ch]);
    const double* bs = p.block_sums + (size_t)ch * p.nblk16;
    if (threadIdx.x == 0) s_total = 0.0;
    for (uint64_t b0 = 0; b0 < p.nblk16; b0 += kStage) {
        const int m = (int)min((uint64_t)kStage, p.nblk16 - b0);
        __syncthreads();
        for (int t = threadIdx.x; t < m; t += blockDim.x) sd[t] = bs[b0 + t];
        __syncthreads();
        if (threadIdx.x == 0) {
            double s = s_total;
            for (int t = 0; t < m; ++t) s = __dadd_rn(s, sd[t]);
            s_total = s;
        }
    }
    __syncthreads();
    const double total = s_total;
    if (!(total > 0.0) || isinf(total)) return;  // Uniform::new(0, s) empty / non-finite: seeding stops here
    double threshold = 0.0;
    if (threadIdx.x == 0) {
        uint64_t s = p.rng[ch];
        threshold = __dmul_rn((double)(splitmix_next(s) >> 11) * (1.0 / 9007199254740992.0), total);
        p.rng[ch] = s;
        s_win = -1;
        s_roll = 0.0;
    }
    const float* mins = p.mins + (size_t)ch * p.n;
    const uint8_t* picked = p.picked + (size_t)ch * p.n;
    float* sf = reinterpret_cast<float*>(sd);
    uint8_t* sp = reinterpret_cast<uint8_t*>(sf + kStage);
    for (uint64_t i0 = 0; i0 < p.n; i0 += kStage) {
        const int m = (int)min((uint64_t)kStage, p.n - i0);
        __syncthreads();
        if (s_win >= 0) break;
        for (int t = threadIdx.x; t < m; t += blockDim.x) {
            sf[t] = mins[i0 + t];
            sp[t] = picked[i0 + t];
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            double r = s_roll;
            for (int t = 0; t < m; ++t) {
                r = __dadd_rn(r, (double)sf[t]);
                if (r >= threshold && sf[t] > 0.0f && !sp[t]) {
                    s_win = (long long)(i0 + t);
                    break;
                }
            }
            s_roll = r;
        }
    }
    __syncthreads();
    const long long win = s_win;
    if (win < 0) return;
    for (int d = threadIdx.x; d < len; d += blockDim.x) p.pivots[(size_t)cur * p.dim + lo + d] = p.data[(uint64_t)win * p.dim + lo + d];
    if (threadIdx.x == 0) {
        p.picked[(size_t)ch * p.n + win] = 1;
        p.prev_norm[ch] = p.norms[(size_t)ch * p.n + win];
        p.selected[ch] = cur + 1;
    }
}

__global__ void center_norms_kernel(const TrainParams p) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= p.n_chunks * p.n_centers) return;
    const uint32_t ch = t / p.n_centers, c = t % p.n_centers;
    const int lo = (int)p.offsets[ch], len = (int)(p.offsets[ch + 1] - p.offsets[ch]);
    p.cnorm[t] = square_norm_ref(p.pivots + (size_t)c * p.dim + lo, len);
}

// distances_in_place: centres of the chunk staged in shared memory, one thread per row
__global__ void __launch_bounds__(256) lloyd_assign_kernel(const TrainParams p) {
    extern __shared__ float sc[];  // [n_centers][len] + [n_centers] norms
    const uint32_t ch = blockIdx.y;
    const int lo = (int)p.offsets[ch], len = (int)(p.offsets[ch + 1] - p.offsets[ch]);
    float* scn = sc + (size_t)p.n_centers * len;
    for (uint32_t t = threadIdx.x; t < p.n_centers * (uint32_t)len; t += blockDim.x) sc[t] = p.pivots[(size_t)(t / len) * p.dim + lo + t % len];
    for (uint32_t t = threadIdx.x; t < p.n_centers; t += blockDim.x) scn[t] = p.cnorm[ch * p.n_centers + t];
    __syncthreads();
    const float* norms = p.norms + (size_t)ch * p.n;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < p.n; i += (uint64_t)gridDim.x * blockDim.x) {
        const float* x = p.data + i * p.dim + lo;
        const float ni = norms[i];
        float best = __int_as_float(0x7F800000);
        uint32_t arg = 0xFFFFFFFFu;
        for (uint32_t c = 0; c < p.n_centers; ++c) {
            const float s = dot_chain(sc + (size_t)c * len, x, len);
            const float d = __fadd_rn(__fsub_rn(__fsub_rn(scn[c], s), s), ni);
            if (d < best) {
                best = d;
                arg = c;
            }
        }
        p.assign[(size_t)ch * p.n + i] = arg;
    }
}

// update_centroids: one warp per (chunk, centre), lane = dimension (chunks wider than 32
// dimensions loop), f64 sums in data order
__global__ void __launch_bounds__(256) lloyd_update_kernel(const TrainParams p) {
    const int lane = threadIdx.x & 31;
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= p.n_chunks * p.n_centers) return;
    const uint32_t ch = w / p.n_centers, c = w % p.n_centers;
    const int lo = (int)p.offsets[ch], len = (int)(p.offsets[ch + 1] - p.offsets[ch]);
    const uint32_t* assign = p.assign + (size_t)ch * p.n;
    for (int d0 = 0; d0 < len; d0 += 32) {
        const int d = d0 + lane;
        double sum = 0.0;
        uint32_t count = 0;
        for (uint64_t i0 = 0; i0 < p.n; i0 += 32) {
            const uint64_t i = i0 + lane;
            unsigned m = __ballot_sync(kFull, i < p.n && assign[i] == c);
            count += __popc(m);
            while (m) {
                const int src = __ffs(m) - 1;
                m &= m - 1;
                if (d < len) sum = __dadd_rn(sum, (double)p.data[(i0 + src) * p.dim + lo + d]);
            }
        }
        if (d < len) p.pivots[(size_t)c * p.dim + lo + d] = (float)__ddiv_rn(sum, (double)max(count, 1u));
    }
}

struct DevMem {
    void* p = nullptr;
    ~DevMem() { cudaFree(p); }
    cudaError_t alloc(size_t n) { return cudaMalloc(&p, n ? n : 1); }
};

}  // namespace

}  // namespace dab

using namespace dab;

extern "C" {

int dab_pq_train(dab_index* idx, const float* train, uint64_t n, uint32_t n_chunks, uint32_t n_centers, uint32_t lloyds_reps,
                 uint64_t seed) {
    if (!idx || !train) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_pq_train: NULL argument");
    if (n_centers == 0 || n_centers > 256) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_pq_train: n_centers must be in [1, 256]");
    if (n_chunks == 0 || n_chunks > idx->dim) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_pq_train: n_chunks must be in [1, dim]");
    if (n < n_centers) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_pq_train: %llu training rows for %u centres", (unsigned long long)n, n_centers);
    DAB_CUDA(cudaSetDevice(idx->device));
    cudaStream_t st = idx->stream;
    const uint32_t dim = idx->dim;
    DAB_CUDA(cudaStreamSynchronize(st));
    int rc;
    if ((rc = retire_quantized_stores(idx))) return rc;  // batches in flight read the table and the codes
    ++idx->store_writes[STORE_PQ];
    // ChunkOffsets::partition (diskann-quantization/src/views.rs:226-243): the first dim % n_chunks chunks get one extra
    std::vector<uint32_t> off(n_chunks + 1, 0);
    uint32_t max_len = 0;
    for (uint32_t c = 0; c < n_chunks; ++c) {
        off[c + 1] = off[c] + dim / n_chunks + (c < dim % n_chunks ? 1 : 0);
        max_len = std::max(max_len, off[c + 1] - off[c]);
    }
    cudaFree(idx->d_pivots);
    cudaFree(idx->d_offsets);
    cudaFree(idx->d_codes);
    idx->d_pivots = nullptr;
    idx->d_offsets = nullptr;
    idx->d_codes = nullptr;
    idx->pq_chunks = idx->pq_centers = 0;
    DAB_CUDA(cudaMalloc(&idx->d_pivots, (size_t)n_centers * dim * 4));
    DAB_CUDA(cudaMalloc(&idx->d_offsets, (size_t)(n_chunks + 1) * 4));
    DAB_CUDA(cudaMalloc(&idx->d_codes, idx->n_total() * (size_t)n_chunks));
    DAB_CUDA(cudaMemsetAsync(idx->d_codes, 0, idx->n_total() * (size_t)n_chunks, st));
    DAB_CUDA(cudaMemcpyAsync(idx->d_offsets, off.data(), (size_t)(n_chunks + 1) * 4, cudaMemcpyHostToDevice, st));

    TrainParams p;
    memset(&p, 0, sizeof(p));
    p.n = n;
    p.dim = dim;
    p.n_chunks = n_chunks;
    p.n_centers = n_centers;
    p.offsets = idx->d_offsets;
    p.pivots = idx->d_pivots;
    p.nblk16 = (n + 15) / 16;
    DevMem data, norms, mins, bsum, picked, rng, prev, sel, assign, cnorm;
    const size_t cn = (size_t)n_chunks * n;
    cudaError_t e = data.alloc(n * (size_t)dim * 4);
    if (e == cudaSuccess) e = norms.alloc(cn * 4);
    if (e == cudaSuccess) e = mins.alloc(cn * 4);
    if (e == cudaSuccess) e = bsum.alloc((size_t)n_chunks * p.nblk16 * 8);
    if (e == cudaSuccess) e = picked.alloc(cn);
    if (e == cudaSuccess) e = rng.alloc((size_t)n_chunks * 8);
    if (e == cudaSuccess) e = prev.alloc((size_t)n_chunks * 4);
    if (e == cudaSuccess) e = sel.alloc((size_t)n_chunks * 4);
    if (e == cudaSuccess) e = assign.alloc(cn * 4);
    if (e == cudaSuccess) e = cnorm.alloc((size_t)n_chunks * n_centers * 4);
    if (e != cudaSuccess) return fail(DAB_ERR_OUT_OF_MEMORY, "dab_pq_train: device allocation failed: %s", cudaGetErrorString(e));
    p.data = (const float*)data.p;
    p.norms = (float*)norms.p;
    p.mins = (float*)mins.p;
    p.block_sums = (double*)bsum.p;
    p.picked = (uint8_t*)picked.p;
    p.rng = (uint64_t*)rng.p;
    p.prev_norm = (float*)prev.p;
    p.selected = (uint32_t*)sel.p;
    p.assign = (uint32_t*)assign.p;
    p.cnorm = (float*)cnorm.p;
    DAB_CUDA(cudaMemcpyAsync(data.p, train, n * (size_t)dim * 4, cudaMemcpyHostToDevice, st));
    DAB_CUDA(cudaMemsetAsync(picked.p, 0, cn, st));
    const int gx = (int)std::min<uint64_t>((n + 255) / 256, (uint64_t)idx->sm_count * 4);
    norms_kernel<<<dim3(gx, n_chunks), 256, 0, st>>>(p);
    DAB_LAUNCHED();
    pp_init_kernel<<<n_chunks, 256, 0, st>>>(p, seed);
    DAB_LAUNCHED();
    const int gb = (int)std::min<uint64_t>((p.nblk16 + 127) / 128, (uint64_t)idx->sm_count * 8);
    for (uint32_t cur = 1; cur < n_centers; ++cur) {
        pp_update_kernel<<<dim3(gb, n_chunks), 128, 0, st>>>(p, cur);
        pp_select_kernel<<<n_chunks, 256, 0, st>>>(p, cur);
        DAB_LAUNCHED();
        DAB_LAUNCHED();
    }
    const size_t smem = ((size_t)n_centers * max_len + n_centers) * 4;
    if (smem > 200 * 1024) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_pq_train: chunk of %u dimensions too wide for the assignment kernel", max_len);
    DAB_CUDA(cudaFuncSetAttribute(lloyd_assign_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const uint32_t nwarps = n_chunks * n_centers;
    for (uint32_t rep = 0; rep < lloyds_reps; ++rep) {
        center_norms_kernel<<<(nwarps + 255) / 256, 256, 0, st>>>(p);
        lloyd_assign_kernel<<<dim3(gx, n_chunks), 256, smem, st>>>(p);
        lloyd_update_kernel<<<(nwarps * 32 + 255) / 256, 256, 0, st>>>(p);
        DAB_LAUNCHED();
        DAB_LAUNCHED();
        DAB_LAUNCHED();
    }
    DAB_CUDA(cudaGetLastError());
    std::vector<uint32_t> h_sel(n_chunks);
    DAB_CUDA(cudaMemcpyAsync(h_sel.data(), sel.p, (size_t)n_chunks * 4, cudaMemcpyDeviceToHost, st));
    DAB_CUDA(cudaStreamSynchronize(st));
    idx->pq_chunks = n_chunks;
    idx->pq_centers = n_centers;
    idx->pq_uniform_len = dim % n_chunks == 0 ? dim / n_chunks : 0;
    idx->pq_codes_ready = false;
    for (uint32_t c = 0; c < n_chunks; ++c)
        if (h_sel[c] != n_centers)
            return fail(DAB_ERR_INVALID_ARGUMENT, "dab_pq_train: chunk %u could only be seeded with %u of %u distinct centres (insufficient diversity)",
                        c, h_sel[c], n_centers);
    return DAB_OK;
}

// Encodes every stored row (converted to f32: T: Into<f32>) with the resident table
// (BasicTable::compress_into for each vector, product/tables/basic.rs:161-194).
int dab_pq_encode_all(dab_index* idx) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_pq_encode_all: idx is NULL");
    if (!idx->d_pivots || !idx->pq_chunks) return fail(DAB_ERR_NOT_READY, "dab_pq_encode_all: no PQ table (dab_upload_pq / dab_pq_train)");
    if (!idx->vectors_ready) return fail(DAB_ERR_NOT_READY, "dab_pq_encode_all: vectors not uploaded");
    DAB_CUDA(cudaSetDevice(idx->device));
    ++idx->store_writes[STORE_PQ];
    const uint64_t total = idx->n_total();
    const uint64_t batch = std::max<uint64_t>(1, std::min<uint64_t>(total, (256ull << 20) / ((size_t)idx->dim * 4)));
    int rc;
    if ((rc = idx->s_queries.reserve(batch * idx->dim * 4))) return rc;
    float* d_f32 = (float*)idx->s_queries.p;
    for (uint64_t first = 0; first < total; first += batch) {
        const uint64_t cnt = std::min(batch, total - first);
        if ((rc = widen_rows(idx, idx->stream, idx->d_vectors + first * idx->row_stride, idx->row_stride, cnt, d_f32))) return rc;
        if ((rc = pq_encode_device(idx, d_f32, cnt, idx->d_codes + first * idx->pq_chunks, 0))) return rc;
    }
    idx->pq_codes_ready = true;
    return DAB_OK;
}

int dab_pq_download(dab_index* idx, float* pivots, uint64_t* offsets, uint8_t* codes) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_pq_download: idx is NULL");
    if (!idx->d_pivots || !idx->pq_chunks) return fail(DAB_ERR_NOT_READY, "dab_pq_download: no PQ table");
    DAB_CUDA(cudaSetDevice(idx->device));
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    if (pivots) DAB_CUDA(cudaMemcpy(pivots, idx->d_pivots, (size_t)idx->pq_centers * idx->dim * 4, cudaMemcpyDeviceToHost));
    if (offsets) {
        std::vector<uint32_t> off(idx->pq_chunks + 1);
        DAB_CUDA(cudaMemcpy(off.data(), idx->d_offsets, off.size() * 4, cudaMemcpyDeviceToHost));
        for (size_t c = 0; c < off.size(); ++c) offsets[c] = off[c];
    }
    if (codes) DAB_CUDA(cudaMemcpy(codes, idx->d_codes, idx->n_total() * (size_t)idx->pq_chunks, cudaMemcpyDeviceToHost));
    return DAB_OK;
}

}  // extern "C"
