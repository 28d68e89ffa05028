// graph_stats.cu — read-only checks of a device graph: DiskANNIndex::count_reachable_nodes (index.rs:2161-2189) and
// get_degree_stats (index.rs:2191-2240).  Neither writes the adjacency, so both may run while batches are in flight.
//
//   * count_reachable: a level-synchronous BFS.  The visited set is a bitmap of n_total bits (128 KB at 1M ids: it stays
//     in L2); one warp per row of the current level reads the list with coalesced loads, as the other adjacency kernels
//     do, claims each id with atomicOr and appends the winners to the next level through one warp-aggregated atomicAdd.
//     The levels are consecutive segments of one queue of n_total ids, since each id is claimed once.  The reference's
//     VecDeque / HashSet loop expands exactly the ids a BFS claims, so the count is the queue's final length; the host
//     reads one 4-byte level size per level.  An id >= n_total reached from an expanded list is what
//     the reference's get_neighbors fails on: the kernel keeps the smallest such id (atomicMin), so the error names it
//     deterministically.
//   * degree_stats: one pass over the list-length words (read as min(len, max_degree), as the traversals read them) with
//     warp reductions and one atomic per warp per statistic.
#include "dab_common.cuh"

#include <algorithm>
#include <vector>

namespace dab {

constexpr int kStatsThreads = 256;  // grid_for sizes grids in blocks of 256 threads

// Claims `id` for the lanes with `want`: the lanes whose atomicOr set the bit append it to next[*next_n ..] through one
// atomicAdd per warp.  Every lane of the warp calls.
__device__ __forceinline__ void bfs_claim(uint32_t id, bool want, uint32_t* __restrict__ visited, uint32_t* __restrict__ next,
                                          uint32_t* __restrict__ next_n, int lane) {
    bool won = false;
    if (want) {
        const uint32_t bit = 1u << (id & 31);
        uint32_t* w = visited + (id >> 5);
        won = !(*(volatile uint32_t*)w & bit) && !(atomicOr(w, bit) & bit);  // a plain read first: most ids are seen
    }
    const unsigned m = __ballot_sync(0xFFFFFFFFu, won);
    if (!m) return;
    const int leader = __ffs(m) - 1;
    uint32_t base = 0;
    if (lane == leader) base = atomicAdd(next_n, (uint32_t)__popc(m));
    base = __shfl_sync(0xFFFFFFFFu, base, leader);
    if (won) next[base + __popc(m & ((1u << lane) - 1u))] = id;
}

// The first frontier: the n start ids (all < n_total), each once.  ids NULL: [first, first + n).
__global__ void __launch_bounds__(kStatsThreads) bfs_seed_kernel(const uint32_t* __restrict__ ids, uint32_t first, uint32_t n,
                                                                 uint32_t* __restrict__ visited, uint32_t* __restrict__ next,
                                                                 uint32_t* __restrict__ next_n) {
    const int lane = threadIdx.x & 31;
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t i0 = blockIdx.x * blockDim.x; i0 < n; i0 += stride) {  // whole warps iterate together
        const uint32_t i = i0 + threadIdx.x;
        const uint32_t id = i < n ? (ids ? ids[i] : first + i) : kNoId;
        bfs_claim(id, i < n, visited, next, next_n, lane);
    }
}

// One warp per frontier row: every listed id < n_total is claimed; the smallest id >= n_total goes to *stray
__global__ void __launch_bounds__(kStatsThreads) bfs_expand_kernel(const uint32_t* __restrict__ adj, uint32_t adj_stride,
                                                                   uint32_t max_degree, uint64_t n_total,
                                                                   const uint32_t* __restrict__ frontier, uint32_t n_frontier,
                                                                   uint32_t* __restrict__ visited, uint32_t* __restrict__ next,
                                                                   uint32_t* __restrict__ next_n, uint32_t* __restrict__ stray) {
    const int lane = threadIdx.x & 31;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    uint32_t low_stray = kNoId;
    for (uint32_t f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; f < n_frontier; f += nwarps) {
        const uint32_t* row = adj + (size_t)frontier[f] * adj_stride;
        const uint32_t deg = min(row[0], max_degree);
        for (uint32_t c = 0; c < deg; c += 32) {
            const uint32_t j = c + lane;
            const uint32_t id = j < deg ? row[1 + j] : kNoId;
            const bool in_range = j < deg && id < n_total;
            if (j < deg && !in_range) low_stray = min(low_stray, id);
            bfs_claim(id, in_range, visited, next, next_n, lane);
        }
    }
    if (low_stray != kNoId) atomicMin(stray, low_stray);
}

// [0] max, [1] min, [2..3] total (u64), [4..5] lists shorter than two (u64)
__global__ void __launch_bounds__(kStatsThreads) degree_stats_kernel(const uint32_t* __restrict__ adj, uint32_t adj_stride,
                                                                     uint32_t max_degree, const uint32_t* __restrict__ ids,
                                                                     uint64_t n, uint32_t* __restrict__ out) {
    uint32_t mx = 0, mn = 0xFFFFFFFFu;
    unsigned long long total = 0, short_lists = 0;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t id = ids ? ids[i] : i;
        const uint32_t deg = min(adj[id * adj_stride], max_degree);
        mx = max(mx, deg);
        mn = min(mn, deg);
        total += deg;
        short_lists += deg < 2;
    }
    for (int o = 16; o > 0; o >>= 1) {
        mx = max(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, o));
        mn = min(mn, __shfl_xor_sync(0xFFFFFFFFu, mn, o));
        total += __shfl_xor_sync(0xFFFFFFFFu, total, o);
        short_lists += __shfl_xor_sync(0xFFFFFFFFu, short_lists, o);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMax(out, mx);
        atomicMin(out + 1, mn);
        atomicAdd(reinterpret_cast<unsigned long long*>(out + 2), total);
        atomicAdd(reinterpret_cast<unsigned long long*>(out + 4), short_lists);
    }
}

// "<who>: id %u out of range" for the first of the n ids >= n_total
static int check_ids(const dab_index* idx, const uint32_t* ids, uint64_t n, const char* who) {
    for (uint64_t i = 0; i < n; ++i)
        if (ids[i] >= idx->n_total())
            return fail(DAB_ERR_INVALID_ARGUMENT, "%s: id %u out of range (%llu ids)", who, ids[i], (unsigned long long)idx->n_total());
    return DAB_OK;
}

}  // namespace dab

using namespace dab;

extern "C" {

int dab_count_reachable(dab_index* idx, const uint32_t* start_ids, uint32_t n, uint64_t* out_count) {
    static const char* who = "dab_count_reachable";
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", who);
    if (!out_count) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: out_count is NULL", who);
    if (!start_ids && n) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: start_ids is NULL with n > 0", who);
    int rc;
    if (start_ids && (rc = check_ids(idx, start_ids, n, who))) return rc;
    if (!idx->graph_ready) return fail(DAB_ERR_NOT_READY, "%s: the graph must be uploaded first", who);
    *out_count = 0;
    const uint64_t n_total = idx->n_total();
    const uint32_t n_seed = start_ids ? n : idx->n_start;
    if (n_seed == 0) return DAB_OK;
    DAB_CUDA(cudaSetDevice(idx->device));
    cudaStream_t st = idx->stream;
    const size_t words = idx->deleted_words();
    // the visited bitmap; the queue of claimed ids, each level a segment of it (an id is claimed once, so n_total slots
    // hold every level); [0] the size of the level being written, [1] the smallest stray id
    DevBuf b_visited, b_queue, b_seed, b_counters;
    if ((rc = b_visited.alloc(words * 4, who)) || (rc = b_queue.alloc(n_total * 4, who)) || (rc = b_counters.alloc(8, who)))
        return rc;
    uint32_t* visited = (uint32_t*)b_visited.p;
    uint32_t* queue = (uint32_t*)b_queue.p;
    uint32_t* next_n = (uint32_t*)b_counters.p;
    uint32_t* stray = next_n + 1;
    const uint32_t* d_seed = nullptr;
    if (start_ids) {
        if ((rc = b_seed.alloc((size_t)n * 4, who))) return rc;
        DAB_CUDA(cudaMemcpyAsync(b_seed.p, start_ids, (size_t)n * 4, cudaMemcpyHostToDevice, st));
        d_seed = (const uint32_t*)b_seed.p;
    }
    DAB_CUDA(cudaMemsetAsync(visited, 0, words * 4, st));
    DAB_CUDA(cudaMemsetAsync(next_n, 0, 4, st));
    DAB_CUDA(cudaMemsetAsync(stray, 0xFF, 4, st));
    bfs_seed_kernel<<<grid_for(idx, n_seed), kStatsThreads, 0, st>>>(d_seed, (uint32_t)idx->n_points, n_seed, visited, queue, next_n);
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    uint64_t end = 0;  // the ids the levels before the one being written claimed
    for (;;) {
        uint32_t size = 0;
        DAB_CUDA(cudaMemcpyAsync(&size, next_n, 4, cudaMemcpyDeviceToHost, st));
        DAB_CUDA(cudaStreamSynchronize(st));
        if (size == 0) break;
        const uint64_t begin = end;  // the level to expand: queue[begin, end)
        end += size;
        DAB_CUDA(cudaMemsetAsync(next_n, 0, 4, st));
        bfs_expand_kernel<<<grid_for(idx, (uint64_t)size * 32), kStatsThreads, 0, st>>>(
            idx->d_adj, idx->adj_stride, idx->max_degree, n_total, queue + begin, size, visited, queue + end, next_n, stray);
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
    }
    uint32_t low_stray = kNoId;
    DAB_CUDA(cudaMemcpyAsync(&low_stray, stray, 4, cudaMemcpyDeviceToHost, st));
    DAB_CUDA(cudaStreamSynchronize(st));
    if (low_stray != kNoId)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: the traversal reached id %u, which is out of range (%llu ids)", who, low_stray,
                    (unsigned long long)n_total);
    *out_count = end;  // every claimed id
    return DAB_OK;
}

int dab_degree_stats(dab_index* idx, const uint32_t* ids, uint64_t n, uint32_t* out_max, float* out_avg, uint32_t* out_min,
                     uint64_t* out_less_than_two) {
    static const char* who = "dab_degree_stats";
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", who);
    if (!out_max || !out_avg || !out_min || !out_less_than_two) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL output", who);
    if (!ids && n) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: ids is NULL with n > 0", who);
    int rc;
    if (ids && (rc = check_ids(idx, ids, n, who))) return rc;
    if (!idx->graph_ready) return fail(DAB_ERR_NOT_READY, "%s: the graph must be uploaded first", who);
    *out_max = 0, *out_avg = 0.0f, *out_min = 0, *out_less_than_two = 0;
    const uint64_t count = ids ? n : idx->n_total();
    if (count == 0) return DAB_OK;  // the reference's guard against the division
    DAB_CUDA(cudaSetDevice(idx->device));
    cudaStream_t st = idx->stream;
    DevBuf b_ids, b_out;
    if ((rc = b_out.alloc(24, who))) return rc;
    if (ids) {
        if ((rc = b_ids.alloc(n * 4, who))) return rc;
        DAB_CUDA(cudaMemcpyAsync(b_ids.p, ids, n * 4, cudaMemcpyHostToDevice, st));
    }
    uint32_t h[6] = {0, 0xFFFFFFFFu, 0, 0, 0, 0};
    DAB_CUDA(cudaMemcpyAsync(b_out.p, h, 24, cudaMemcpyHostToDevice, st));
    degree_stats_kernel<<<grid_for(idx, count), kStatsThreads, 0, st>>>(idx->d_adj, idx->adj_stride, idx->max_degree,
                                                                      (const uint32_t*)b_ids.p, count, (uint32_t*)b_out.p);
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    DAB_CUDA(cudaMemcpyAsync(h, b_out.p, 24, cudaMemcpyDeviceToHost, st));
    DAB_CUDA(cudaStreamSynchronize(st));
    uint64_t total, short_lists;
    memcpy(&total, h + 2, 8);
    memcpy(&short_lists, h + 4, 8);
    *out_max = h[0];
    *out_min = h[1];
    *out_avg = (float)total / (float)count;  // Rust's `as f32`: each conversion rounds to nearest
    *out_less_than_two = short_lists;
    return DAB_OK;
}

}  // extern "C"
