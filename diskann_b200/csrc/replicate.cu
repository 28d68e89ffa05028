// replicate.cu — index replication across GPUs: one NCCL broadcast of the HBM-resident snapshot
// (vectors, adjacency, PQ table + codes) at load, no collective on the search path
// (SURVEY.md §8e; BASELINE.json north_star "one NCCL broadcast of the index at load").
//
// Two forms, both inside the C ABI so that a Rust host needs no torch:
//   * one process per GPU: dab_comm_unique_id (rank 0) -> the host ships the 128 bytes to the other
//     ranks by any means -> dab_comm_init(idx, id, n_ranks, rank) -> dab_broadcast_index(idx, root);
//   * one process driving several GPUs: dab_broadcast(per_gpu, n_gpus) (ncclCommInitAll + grouped
//     broadcasts), the form SURVEY.md §8b sketches.
// NCCL is resolved with dlopen("libnccl.so.2") at first use: the library keeps linking only the
// static CUDA runtime, and a host that never replicates needs no NCCL at all.
#include "dab_common.cuh"

#include <dlfcn.h>

#include <mutex>
#include <vector>

namespace dab {

namespace {

typedef struct ncclComm* ncclComm_t;
struct ncclUniqueId {
    char internal[128];
};
enum { kNcclSuccess = 0, kNcclUint8 = 1 };

struct Nccl {
    void* handle = nullptr;
    int (*GetUniqueId)(ncclUniqueId*) = nullptr;
    int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    int (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
    int (*CommDestroy)(ncclComm_t) = nullptr;
    int (*Broadcast)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool ok = false;
};

Nccl& nccl() {
    static Nccl n;
    static std::once_flag once;
    std::call_once(once, [] {
        for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
            n.handle = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
            if (n.handle) break;
        }
        if (!n.handle) return;
#define DAB_SYM(field, sym) *(void**)(&n.field) = dlsym(n.handle, sym)
        DAB_SYM(GetUniqueId, "ncclGetUniqueId");
        DAB_SYM(CommInitRank, "ncclCommInitRank");
        DAB_SYM(CommInitAll, "ncclCommInitAll");
        DAB_SYM(CommDestroy, "ncclCommDestroy");
        DAB_SYM(Broadcast, "ncclBroadcast");
        DAB_SYM(GroupStart, "ncclGroupStart");
        DAB_SYM(GroupEnd, "ncclGroupEnd");
        DAB_SYM(GetErrorString, "ncclGetErrorString");
#undef DAB_SYM
        n.ok = n.GetUniqueId && n.CommInitRank && n.CommInitAll && n.CommDestroy && n.Broadcast && n.GroupStart && n.GroupEnd;
    });
    return n;
}

int need_nccl(const char* who) {
    if (!nccl().ok) return fail(DAB_ERR_NOT_READY, "%s: NCCL (libnccl.so.2) could not be loaded: %s", who, dlerror() ? dlerror() : "symbols missing");
    return DAB_OK;
}

#define DAB_NCCL(expr)                                                                                     \
    do {                                                                                                   \
        const int _r = (expr);                                                                             \
        if (_r != kNcclSuccess)                                                                            \
            return fail(DAB_ERR_CUDA, "%s failed: %s", #expr, nccl().GetErrorString ? nccl().GetErrorString(_r) : "NCCL error"); \
    } while (0)

// what a replica must agree on with the root before any buffer is overwritten
struct IndexMeta {
    uint64_t n_points, row_stride;
    uint32_t dtype, metric, dim, n_start, max_degree, adj_stride, vectors_ready, graph_ready, pq_chunks, pq_centers, pq_codes_ready, pq_uniform_len;
    uint64_t n_deleted;  // the deletion table travels with the graph: replicas would otherwise return deleted ids
};

IndexMeta meta_of(const dab_index* idx) {
    IndexMeta m;
    memset(&m, 0, sizeof(m));
    m.n_points = idx->n_points;
    m.row_stride = idx->row_stride;
    m.dtype = (uint32_t)idx->dtype;
    m.metric = (uint32_t)idx->metric;
    m.dim = idx->dim;
    m.n_start = idx->n_start;
    m.max_degree = idx->max_degree;
    m.adj_stride = idx->adj_stride;
    m.vectors_ready = idx->vectors_ready;
    m.graph_ready = idx->graph_ready;
    m.pq_chunks = idx->pq_chunks;
    m.pq_centers = idx->pq_centers;
    m.pq_codes_ready = idx->pq_codes_ready;
    m.pq_uniform_len = idx->pq_uniform_len;
    m.n_deleted = idx->n_deleted;
    return m;
}

// broadcast every resident buffer of `idx` from `root` over `comm` (all ranks call this)
int broadcast_buffers(dab_index* idx, ncclComm_t comm, int root, bool is_root, IndexMeta* d_meta) {
    Nccl& n = nccl();
    cudaStream_t st = idx->stream;
    IndexMeta mine = meta_of(idx), got;
    DAB_CUDA(cudaMemcpyAsync(d_meta, &mine, sizeof(mine), cudaMemcpyHostToDevice, st));
    DAB_NCCL(n.Broadcast(d_meta, d_meta, sizeof(IndexMeta), kNcclUint8, root, comm, st));
    DAB_CUDA(cudaMemcpyAsync(&got, d_meta, sizeof(got), cudaMemcpyDeviceToHost, st));
    DAB_CUDA(cudaStreamSynchronize(st));
    if (got.n_points != mine.n_points || got.row_stride != mine.row_stride || got.dtype != mine.dtype || got.metric != mine.metric ||
        got.dim != mine.dim || got.n_start != mine.n_start || got.max_degree != mine.max_degree || got.adj_stride != mine.adj_stride)
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_broadcast: this replica was created with a different shape than the root "
                    "(n_points %llu vs %llu, dim %u vs %u, dtype %u vs %u, max_degree %u vs %u)", (unsigned long long)mine.n_points,
                    (unsigned long long)got.n_points, mine.dim, got.dim, mine.dtype, got.dtype, mine.max_degree, got.max_degree);
    const uint64_t total = idx->n_total();
    if (got.vectors_ready) DAB_NCCL(n.Broadcast(idx->d_vectors, idx->d_vectors, total * idx->row_stride, kNcclUint8, root, comm, st));
    if (got.graph_ready) DAB_NCCL(n.Broadcast(idx->d_adj, idx->d_adj, total * (size_t)idx->adj_stride * 4, kNcclUint8, root, comm, st));
    if (got.pq_chunks) {
        ++idx->store_writes[STORE_PQ];
        if (!is_root) {
            DAB_CUDA(cudaStreamSynchronize(st));
            int rc;
            if ((rc = retire_quantized_stores(idx))) return rc;  // batches in flight read the table and the codes
            cudaFree(idx->d_pivots);
            cudaFree(idx->d_offsets);
            cudaFree(idx->d_codes);
            idx->d_pivots = nullptr;
            idx->d_offsets = nullptr;
            idx->d_codes = nullptr;
            DAB_CUDA(cudaMalloc(&idx->d_pivots, (size_t)got.pq_centers * idx->dim * 4));
            DAB_CUDA(cudaMalloc(&idx->d_offsets, (size_t)(got.pq_chunks + 1) * 4));
            DAB_CUDA(cudaMalloc(&idx->d_codes, total * (size_t)got.pq_chunks));
        }
        DAB_NCCL(n.Broadcast(idx->d_pivots, idx->d_pivots, (size_t)got.pq_centers * idx->dim * 4, kNcclUint8, root, comm, st));
        DAB_NCCL(n.Broadcast(idx->d_offsets, idx->d_offsets, (size_t)(got.pq_chunks + 1) * 4, kNcclUint8, root, comm, st));
        DAB_NCCL(n.Broadcast(idx->d_codes, idx->d_codes, total * (size_t)got.pq_chunks, kNcclUint8, root, comm, st));
    }
    int rc;
    if (got.n_deleted) {
        // the root's table into every rank's device copy, then into its host copy
        if ((rc = deleted_alloc(idx))) return rc;
        DAB_NCCL(n.Broadcast(idx->d_deleted, idx->d_deleted, idx->deleted_words() * 4, kNcclUint8, root, comm, st));
        std::vector<uint32_t> words(idx->deleted_words());
        DAB_CUDA(cudaMemcpyAsync(words.data(), idx->d_deleted, idx->deleted_words() * 4, cudaMemcpyDeviceToHost, st));
        DAB_CUDA(cudaStreamSynchronize(st));
        if ((rc = deleted_assign(idx, words.data(), got.n_deleted))) return rc;
    } else if ((rc = deleted_assign(idx, nullptr, 0))) {
        return rc;
    }
    DAB_CUDA(cudaStreamSynchronize(st));
    ++idx->generation;
    idx->vectors_ready = got.vectors_ready != 0;
    if (got.vectors_ready && !is_root) ++idx->vectors_version;
    idx->graph_ready = got.graph_ready != 0;
    idx->pq_chunks = got.pq_chunks;
    idx->pq_centers = got.pq_centers;
    idx->pq_uniform_len = got.pq_uniform_len;
    idx->pq_codes_ready = got.pq_codes_ready != 0;
    return DAB_OK;
}

}  // namespace

void comm_release(dab_index* idx) {
    if (idx->nccl_comm && nccl().ok) nccl().CommDestroy((ncclComm_t)idx->nccl_comm);
    idx->nccl_comm = nullptr;
}

}  // namespace dab

using namespace dab;

extern "C" {

int dab_comm_unique_id(char* out_id128) {
    if (!out_id128) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_comm_unique_id: NULL argument");
    int rc = need_nccl("dab_comm_unique_id");
    if (rc) return rc;
    ncclUniqueId id;
    DAB_NCCL(nccl().GetUniqueId(&id));
    memcpy(out_id128, id.internal, 128);
    return DAB_OK;
}

int dab_comm_init(dab_index* idx, const char* id128, int n_ranks, int rank) {
    if (!idx || !id128) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_comm_init: NULL argument");
    if (n_ranks < 1 || rank < 0 || rank >= n_ranks) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_comm_init: rank %d of %d", rank, n_ranks);
    int rc = need_nccl("dab_comm_init");
    if (rc) return rc;
    DAB_CUDA(cudaSetDevice(idx->device));
    comm_release(idx);
    ncclUniqueId id;
    memcpy(id.internal, id128, 128);
    ncclComm_t comm = nullptr;
    DAB_NCCL(nccl().CommInitRank(&comm, n_ranks, id, rank));
    idx->nccl_comm = comm;
    idx->nccl_rank = rank;
    idx->nccl_ranks = n_ranks;
    return DAB_OK;
}

int dab_broadcast_index(dab_index* idx, int root) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_broadcast_index: idx is NULL");
    if (!idx->nccl_comm) return fail(DAB_ERR_NOT_READY, "dab_broadcast_index: dab_comm_init has not been called");
    if (root < 0 || root >= idx->nccl_ranks) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_broadcast_index: root %d of %d ranks", root, idx->nccl_ranks);
    DAB_CUDA(cudaSetDevice(idx->device));
    int rc;
    if ((rc = idx->s_counters.reserve(sizeof(IndexMeta) + 64))) return rc;
    return broadcast_buffers(idx, (ncclComm_t)idx->nccl_comm, root, idx->nccl_rank == root, (IndexMeta*)idx->s_counters.p);
}

int dab_comm_destroy(dab_index* idx) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_comm_destroy: idx is NULL");
    comm_release(idx);
    return DAB_OK;
}

// Single-process form (SURVEY.md §8b): per_gpu[0] is the root; every handle lives on its own device.
int dab_broadcast(dab_index* const* per_gpu, int n_gpus) {
    if (!per_gpu || n_gpus < 1) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_broadcast: NULL argument");
    if (n_gpus == 1) return DAB_OK;
    int rc = need_nccl("dab_broadcast");
    if (rc) return rc;
    std::vector<int> devs(n_gpus);
    for (int i = 0; i < n_gpus; ++i) {
        if (!per_gpu[i]) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_broadcast: handle %d is NULL", i);
        devs[i] = per_gpu[i]->device;
        for (int j = 0; j < i; ++j)
            if (devs[j] == devs[i]) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_broadcast: handles %d and %d share device %d", j, i, devs[i]);
    }
    std::vector<ncclComm_t> comms(n_gpus, nullptr);
    DAB_NCCL(nccl().CommInitAll(comms.data(), n_gpus, devs.data()));
    Nccl& n = nccl();
    const dab_index* root = per_gpu[0];
    const IndexMeta want = meta_of(root);
    int status = DAB_OK;
    for (int i = 1; i < n_gpus && status == DAB_OK; ++i) {
        const IndexMeta m = meta_of(per_gpu[i]);
        if (m.n_points != want.n_points || m.row_stride != want.row_stride || m.dtype != want.dtype || m.metric != want.metric ||
            m.dim != want.dim || m.n_start != want.n_start || m.max_degree != want.max_degree)
            status = fail(DAB_ERR_INVALID_ARGUMENT, "dab_broadcast: handle %d was created with a different shape than handle 0", i);
        else if (want.pq_chunks) {
            dab_index* r = per_gpu[i];
            ++r->store_writes[STORE_PQ];
            cudaSetDevice(r->device);
            cudaFree(r->d_pivots);
            cudaFree(r->d_offsets);
            cudaFree(r->d_codes);
            r->d_pivots = nullptr, r->d_offsets = nullptr, r->d_codes = nullptr;
            if (cudaMalloc(&r->d_pivots, (size_t)want.pq_centers * r->dim * 4) != cudaSuccess ||
                cudaMalloc(&r->d_offsets, (size_t)(want.pq_chunks + 1) * 4) != cudaSuccess ||
                cudaMalloc(&r->d_codes, r->n_total() * (size_t)want.pq_chunks) != cudaSuccess)
                status = fail(DAB_ERR_OUT_OF_MEMORY, "dab_broadcast: PQ buffers on device %d", r->device);
        }
    }
    const uint64_t total = root->n_total();
    auto bcast = [&](size_t bytes, auto field) -> int {
        if (n.GroupStart() != kNcclSuccess) return 1;
        int bad = 0;
        for (int i = 0; i < n_gpus; ++i) {
            cudaSetDevice(per_gpu[i]->device);
            void* buf = (void*)field(per_gpu[i]);
            bad |= n.Broadcast(buf, buf, bytes, kNcclUint8, 0, comms[i], per_gpu[i]->stream) != kNcclSuccess;
        }
        if (n.GroupEnd() != kNcclSuccess) return 1;
        return bad;
    };
    if (status == DAB_OK && want.vectors_ready && bcast(total * root->row_stride, [](dab_index* x) { return x->d_vectors; }))
        status = fail(DAB_ERR_CUDA, "dab_broadcast: ncclBroadcast(vectors) failed");
    if (status == DAB_OK && want.graph_ready && bcast(total * (size_t)root->adj_stride * 4, [](dab_index* x) { return x->d_adj; }))
        status = fail(DAB_ERR_CUDA, "dab_broadcast: ncclBroadcast(adjacency) failed");
    if (status == DAB_OK && want.pq_chunks) {
        if (bcast((size_t)want.pq_centers * root->dim * 4, [](dab_index* x) { return x->d_pivots; }) ||
            bcast((size_t)(want.pq_chunks + 1) * 4, [](dab_index* x) { return x->d_offsets; }) ||
            bcast(total * (size_t)want.pq_chunks, [](dab_index* x) { return x->d_codes; }))
            status = fail(DAB_ERR_CUDA, "dab_broadcast: ncclBroadcast(PQ) failed");
    }
    for (int i = 1; i < n_gpus && status == DAB_OK; ++i) {
        cudaSetDevice(per_gpu[i]->device);
        status = deleted_assign(per_gpu[i], root->h_deleted, root->n_deleted);
    }
    for (int i = 0; i < n_gpus; ++i) {
        cudaSetDevice(per_gpu[i]->device);
        cudaStreamSynchronize(per_gpu[i]->stream);
        if (status == DAB_OK && i) {
            per_gpu[i]->vectors_ready = want.vectors_ready != 0;
            ++per_gpu[i]->vectors_version;
            ++per_gpu[i]->generation;
            per_gpu[i]->graph_ready = want.graph_ready != 0;
            per_gpu[i]->pq_chunks = want.pq_chunks;
            per_gpu[i]->pq_centers = want.pq_centers;
            per_gpu[i]->pq_uniform_len = want.pq_uniform_len;
            per_gpu[i]->pq_codes_ready = want.pq_codes_ready != 0;
        }
        n.CommDestroy(comms[i]);
    }
    return status;
}

}  // extern "C"
