// delete_kernels.cu — the deletion table of an index and what the searches do with it.
//
// Restates the providers' TableDeleteProviderAsync (diskann-providers/src/model/graph/provider/async_/
// table_delete_provider.rs; Delete for DefaultProvider, inmem/provider.rs:596-655): one bit per id.  The table lives on
// the host, where every call reads and checks it, and is copied to the device after every change; the device copy is
// allocated by the first dab_delete and read only by the searches' post-processing.  While no id is deleted every
// search launches exactly what it launches without a table.
//
// The searches' post-processing, Pipeline<FilterStartPoints, RemoveDeletedIdsAndCopy> (async_/postprocess.rs:35-61),
// takes the first k entries of the final candidate list that are neither start points nor deleted.  The traversal does
// not change (deleted nodes are still expanded and counted), so the traversal kernels write their whole non-start list
// and drop_deleted_kernel below filters it.  Consolidation, which repairs the graph around deleted points, is
// dab_consolidate in build_kernels.cu.
#include "dab_common.cuh"
#include "search_host.cuh"

#include <algorithm>
#include <vector>

namespace dab {

// One warp per query: the first k live entries of a list of `cap`, list order kept
__global__ void __launch_bounds__(128) drop_deleted_kernel(const uint32_t* __restrict__ ids, const float* __restrict__ dists, uint32_t cap,
                                                           uint32_t nq, uint32_t k, const uint32_t* __restrict__ deleted, uint64_t n_points,
                                                           uint32_t* __restrict__ out_ids, float* __restrict__ out_dists,
                                                           uint32_t* __restrict__ out_counts) {
    const int lane = threadIdx.x & 31;
    for (uint32_t q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < nq; q += (gridDim.x * blockDim.x) >> 5) {
        uint32_t count = 0;
        for (uint32_t b = 0; b < cap && count < k; b += 32) {
            const uint32_t i = b + lane;
            const uint32_t id = i < cap ? ids[(size_t)q * cap + i] : kNoId;
            // padding (UINT32_MAX) and start points are >= n_points
            const bool keep = id < n_points && !(__ldg(deleted + (id >> 5)) >> (id & 31) & 1u);
            const unsigned m = __ballot_sync(0xFFFFFFFFu, keep);
            const uint32_t pos = count + __popc(m & ((1u << lane) - 1u));
            if (keep && pos < k) {
                out_ids[(size_t)q * k + pos] = id;
                out_dists[(size_t)q * k + pos] = dists[(size_t)q * cap + i];
            }
            count += __popc(m);
        }
        count = min(count, k);
        for (uint32_t i = count + lane; i < k; i += 32) {
            out_ids[(size_t)q * k + i] = kNoId;
            out_dists[(size_t)q * k + i] = __int_as_float(0x7F800000);
        }
        if (lane == 0 && out_counts) out_counts[q] = count;
    }
}

int queue_drop_deleted(const dab_index* idx, cudaStream_t stream, const uint32_t* deleted, const uint32_t* ids, const float* dists,
                       uint32_t cap, uint32_t nq, uint32_t k, const SearchOut& out, uint64_t bound) {
    if (nq == 0) return DAB_OK;
    const int grid = (int)std::min<uint64_t>(((uint64_t)nq + 3) / 4, (uint64_t)idx->sm_count * 16);
    drop_deleted_kernel<<<grid, 128, 0, stream>>>(ids, dists, cap, nq, k, deleted, bound, out.ids, out.dists, out.counts);
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    return DAB_OK;
}

const uint32_t* deleted_filter(const dab_index* idx) { return idx->n_deleted ? idx->d_deleted : nullptr; }

void deleted_release(dab_index* idx) {
    cudaFree(idx->d_deleted);
    delete[] idx->h_deleted;
    idx->d_deleted = nullptr;
    idx->h_deleted = nullptr;
    idx->n_deleted = 0;
}

int deleted_alloc(dab_index* idx) {
    if (idx->h_deleted) return DAB_OK;
    const size_t bytes = idx->deleted_words() * 4;
    DAB_CUDA(cudaMalloc(&idx->d_deleted, bytes));
    DAB_CUDA(cudaMemsetAsync(idx->d_deleted, 0, bytes, idx->stream));
    idx->h_deleted = new uint32_t[idx->deleted_words()]();
    return DAB_OK;
}

// the host table -> the device copy
static int deleted_push(dab_index* idx) {
    DAB_CUDA(cudaMemcpyAsync(idx->d_deleted, idx->h_deleted, idx->deleted_words() * 4, cudaMemcpyHostToDevice, idx->stream));
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    return DAB_OK;
}

static bool is_deleted(const dab_index* idx, uint64_t id);

int deleted_mark(dab_index* idx, const uint32_t* ids, uint64_t n) {
    int rc;
    if ((rc = deleted_alloc(idx))) return rc;
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t id = ids[i];
        if (!is_deleted(idx, id)) {
            idx->h_deleted[id >> 5] |= 1u << (id & 31);
            ++idx->n_deleted;
        }
    }
    return deleted_push(idx);
}

int deleted_assign(dab_index* idx, const uint32_t* words, uint64_t n_deleted) {
    if (n_deleted == 0 && !idx->h_deleted) return DAB_OK;
    int rc;
    if ((rc = deleted_alloc(idx))) return rc;
    if (n_deleted)
        memcpy(idx->h_deleted, words, idx->deleted_words() * 4);
    else
        memset(idx->h_deleted, 0, idx->deleted_words() * 4);
    idx->n_deleted = n_deleted;
    return deleted_push(idx);
}

static bool is_deleted(const dab_index* idx, uint64_t id) {
    return idx->h_deleted && id < idx->n_points && (idx->h_deleted[id >> 5] >> (id & 31) & 1u);
}

int refuse_in_flight(const dab_index* idx, const char* api) {
    for (int i = 0; i < DAB_MAX_SLOTS; ++i) {
        const SearchSlot* s = (const SearchSlot*)idx->slots[i];
        if (s && s->job) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: slot %d holds a batch in flight (call dab_wait first)", api, i);
    }
    return DAB_OK;
}

__global__ void clear_rows_kernel(uint32_t* __restrict__ adj, uint32_t adj_stride, const uint32_t* __restrict__ ids, uint64_t n) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        adj[(size_t)ids[i] * adj_stride] = 0;
}

int clear_rows(const dab_index* idx, const uint32_t* d_ids, uint64_t n) {
    const int grid = (int)std::min<uint64_t>((n + 255) / 256, (uint64_t)idx->sm_count * 8);
    clear_rows_kernel<<<grid, 256, 0, idx->stream>>>(idx->d_adj, idx->adj_stride, d_ids, n);
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    return DAB_OK;
}

// DiskANNIndex::drop_deleted_neighbors (index.rs:1756-1816) for every node, one warp per node.  A node's new list depends
// only on its own list, the table and, with only_orphans, the lengths of its deleted neighbours' lists, and no deleted
// node's list is written: one pass in any order equals the sequential loop.  `list`: per warp, max_degree words of
// shared memory holding the list as read.
__global__ void __launch_bounds__(128) drop_deleted_neighbors_kernel(uint32_t* __restrict__ adj, uint32_t adj_stride, uint32_t max_degree,
                                                                     uint64_t n_total, const uint32_t* __restrict__ deleted,
                                                                     uint32_t degree, int only_orphans, uint32_t* __restrict__ rewritten) {
    extern __shared__ uint32_t drop_smem[];
    const int lane = threadIdx.x & 31;
    uint32_t* list = drop_smem + (threadIdx.x >> 5) * max_degree;
    auto dead = [&](uint32_t id) { return id >= n_total || (deleted && (__ldg(deleted + (id >> 5)) >> (id & 31) & 1u)); };
    for (uint64_t v = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5; v < n_total; v += ((uint64_t)gridDim.x * blockDim.x) >> 5) {
        if (dead((uint32_t)v)) continue;  // ConsolidateKind::Deleted
        uint32_t* row = adj + v * adj_stride;
        const uint32_t deg = min(row[0], max_degree);
        bool any_dead = false;
        for (uint32_t j = lane; j < deg; j += 32) {
            list[j] = row[1 + j];
            any_dead |= dead(list[j]);
        }
        any_dead = __any_sync(0xFFFFFFFFu, any_dead);
        if (!any_dead && deg <= degree) continue;  // nothing deleted, and no prune needed
        __syncwarp();
        // the pool: live neighbours in list order, then (only_orphans) the deleted ones whose list is not empty
        uint32_t n = 0;
        for (int pass = 0; pass < (only_orphans ? 2 : 1); ++pass) {
            for (uint32_t c0 = 0; c0 < deg; c0 += 32) {
                const uint32_t j = c0 + lane;
                const uint32_t id = j < deg ? list[j] : kNoId;
                bool keep = j < deg && !dead(id);
                if (pass == 1) keep = j < deg && dead(id) && id < n_total && adj[(size_t)id * adj_stride] != 0;
                const unsigned m = __ballot_sync(0xFFFFFFFFu, keep);
                if (keep) row[1 + n + __popc(m & ((1u << lane) - 1u))] = id;
                n += __popc(m);
            }
        }
        __syncwarp();
        if (lane == 0) {
            row[0] = n;
            atomicAdd(rewritten, 1u);
        }
    }
}

}  // namespace dab

using namespace dab;

extern "C" {

int dab_delete(dab_index* idx, const uint32_t* ids, uint64_t n) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_delete: idx is NULL");
    if (n && !ids) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_delete: NULL argument");
    int rc;
    if ((rc = refuse_in_flight(idx, "dab_delete"))) return rc;
    for (uint64_t i = 0; i < n; ++i)
        if (ids[i] >= idx->n_points)
            return fail(DAB_ERR_INVALID_ARGUMENT, "dab_delete: id %u is not a data point (n_points %llu; start points cannot be deleted)",
                        ids[i], (unsigned long long)idx->n_points);
    if (n == 0) return DAB_OK;
    DAB_CUDA(cudaSetDevice(idx->device));
    if ((rc = deleted_alloc(idx))) return rc;
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t id = ids[i];
        if (!is_deleted(idx, id)) {
            idx->h_deleted[id >> 5] |= 1u << (id & 31);
            ++idx->n_deleted;
        }
    }
    return deleted_push(idx);
}

int dab_release(dab_index* idx, const uint32_t* ids, uint64_t n) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_release: idx is NULL");
    if (n && !ids) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_release: NULL argument");
    int rc;
    if ((rc = refuse_in_flight(idx, "dab_release"))) return rc;
    for (uint64_t i = 0; i < n; ++i)
        if (!is_deleted(idx, ids[i])) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_release: id %u is not deleted", ids[i]);
    if (n == 0) return DAB_OK;
    DAB_CUDA(cudaSetDevice(idx->device));
    if ((rc = idx->s_ids.reserve(n * 4))) return rc;
    DAB_CUDA(cudaMemcpyAsync(idx->s_ids.p, ids, n * 4, cudaMemcpyHostToDevice, idx->stream));
    const int grid = (int)std::min<uint64_t>((n + 255) / 256, (uint64_t)idx->sm_count * 8);
    clear_rows_kernel<<<grid, 256, 0, idx->stream>>>(idx->d_adj, idx->adj_stride, (const uint32_t*)idx->s_ids.p, n);
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t id = ids[i];
        if (is_deleted(idx, id)) {
            idx->h_deleted[id >> 5] &= ~(1u << (id & 31));
            --idx->n_deleted;
        }
    }
    ++idx->generation;  // adjacency rows were written
    return deleted_push(idx);
}

int dab_drop_deleted_neighbors(dab_index* idx, uint32_t pruned_degree, int only_orphans, uint64_t* out_rewritten) {
    static const char* who = "dab_drop_deleted_neighbors";
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", who);
    int rc;
    if ((rc = refuse_in_flight(idx, who))) return rc;
    if (!idx->graph_ready) return fail(DAB_ERR_NOT_READY, "%s: the graph must be uploaded first", who);
    if (pruned_degree == 0 || pruned_degree > idx->max_degree)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: pruned_degree must be in [1, max_degree]", who);
    DAB_CUDA(cudaSetDevice(idx->device));
    if ((rc = idx->s_counters.reserve(4))) return rc;
    uint32_t* d_rewritten = (uint32_t*)idx->s_counters.p;
    DAB_CUDA(cudaMemsetAsync(d_rewritten, 0, 4, idx->stream));
    const size_t smem = (size_t)4 * idx->max_degree * 4;
    const int grid = (int)std::min<uint64_t>((idx->n_total() + 3) / 4, (uint64_t)idx->sm_count * 16);
    DAB_CUDA(cudaFuncSetAttribute(drop_deleted_neighbors_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    drop_deleted_neighbors_kernel<<<grid, 128, smem, idx->stream>>>(idx->d_adj, idx->adj_stride, idx->max_degree, idx->n_total(),
                                                                   deleted_filter(idx), pruned_degree, only_orphans ? 1 : 0, d_rewritten);
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    uint32_t rewritten = 0;
    DAB_CUDA(cudaMemcpyAsync(&rewritten, d_rewritten, 4, cudaMemcpyDeviceToHost, idx->stream));
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    if (rewritten) ++idx->generation;  // adjacency rows were written: open paged sessions fail their next page
    if (out_rewritten) *out_rewritten = rewritten;
    return DAB_OK;
}

int dab_delete_status(dab_index* idx, const uint32_t* ids, uint64_t n, uint8_t* out_deleted) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_delete_status: idx is NULL");
    if (n && (!ids || !out_deleted)) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_delete_status: NULL argument");
    for (uint64_t i = 0; i < n; ++i)
        if (ids[i] >= idx->n_total())
            return fail(DAB_ERR_INVALID_ARGUMENT, "dab_delete_status: id %u out of range (%llu ids)", ids[i], (unsigned long long)idx->n_total());
    for (uint64_t i = 0; i < n; ++i) out_deleted[i] = is_deleted(idx, ids[i]) ? 1 : 0;
    return DAB_OK;
}

}  // extern "C"
