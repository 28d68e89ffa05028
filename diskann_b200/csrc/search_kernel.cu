// search_kernel.cu — the host side of batched graph search: the visited-table policy, the overflow re-runs and the
// host-buffer calls every search shares (search_host.cuh), the full-precision dispatcher, the slots of batches in flight
// (which the quantized *_async calls of search_kernel_pq.cu share) and the C entry points (dab_search_batch[_device][_async],
// dab_wait).
//
// A batch runs on search_kernel_v3 (visited set in shared memory) where its short lists make that the faster kernel,
// and on search_kernel_v2 (global visited tables) otherwise; queries whose visited set outgrows its table are re-run
// on v2 with larger tables, so membership stays exact.  Both kernels restate DiskANNIndex::search_internal
// (index.rs:1933-2000) bit for bit.
#include "dab_common.cuh"
#include "search_host.cuh"
#include "search_v2.cuh"
#include "search_v3.cuh"

#include <algorithm>

namespace dab {

int check_search_args(const dab_index* idx, uint32_t k, uint32_t l_search, uint32_t beam, bool need_vectors) {
    if (!idx->graph_ready || (need_vectors && !idx->vectors_ready))
        return fail(DAB_ERR_NOT_READY, need_vectors ? "search: vectors and graph must be uploaded first" : "search: graph must be uploaded first");
    if (k == 0 || l_search == 0 || beam == 0) return fail(DAB_ERR_INVALID_ARGUMENT, "search: k, l_search and beam_width must be > 0");
    if (beam > 64) return fail(DAB_ERR_INVALID_ARGUMENT, "search: beam_width %u > 64", beam);
    return DAB_OK;
}

// ---- visited tables in global memory (search_kernel_v2, search_kernel_pq, search_kernel_pqs) -----------------------
// Every warp owns a table of `slots` ids in 32-byte buckets of 8.  A query whose visited set passes 7/8 of its table
// stops and is listed in the pass's overflow list; it is re-run on a larger table, so membership is exact at any size.
uint64_t table_slots(const dab_index* idx, const VisitedHint& hint, uint32_t l_search, uint32_t beam, QuantStore mode) {
    if (idx->tune.test_visited_log2) return 1ull << idx->tune.test_visited_log2;  // tests force the overflow re-runs
    // the reference's estimate (scratch.rs:186-192: 1.1 * max_degree * 1.3 * L), never more than the index
    double est = 1.1 * idx->max_degree * 1.3 * (double)l_search;
    if (hint.visited > 0 && l_search <= hint.l && beam <= hint.beam && mode == hint.mode) {
        // the estimate is ~10x what a search touches: 1.15x the largest visited set seen at this (or a larger) L and
        // beam (visited sets grow monotonically with both) at 87.5 % load
        const double seen = ((double)hint.visited * 1.15 + idx->max_degree) / 0.875 + 8.0;
        est = std::min(est, seen);
    }
    est = std::min(est, (double)idx->n_total() * 1.34);
    return std::max<uint64_t>(256, (uint64_t)est + 1);
}

void learn_visited(VisitedHint& hint, uint32_t l_search, uint32_t beam, QuantStore mode, uint32_t visited) {
    if (l_search != hint.l || beam != hint.beam || mode != hint.mode) hint = VisitedHint{l_search, beam, 0, mode};
    hint.visited = std::max(hint.visited, visited);
}

int check_quant_store(const dab_index* idx, QuantStore store, const char* who, bool upload_first) {
    if (store == STORE_PQ) {
        if (upload_first && !idx->d_pivots) return fail(DAB_ERR_NOT_READY, "%s: dab_upload_pq has not been called", who);
        if (!idx->d_pivots || !idx->d_codes || !idx->pq_codes_ready)
            return fail(DAB_ERR_NOT_READY, "%s: no PQ codes (dab_upload_pq with codes, or dab_pq_encode_all)", who);
        return DAB_OK;
    }
    const bool sq = store == STORE_SQ;
    const CodeStore& cs = sq ? idx->sq : idx->mm;
    int rc;
    if (upload_first && (rc = store_require(idx, sq ? &dab_index::sq : &dab_index::mm, sq ? "dab_upload_sq" : "dab_upload_minmax", who))) return rc;
    if (!cs.d_codes || !cs.ready)
        return fail(DAB_ERR_NOT_READY, sq ? "%s: no scalar-quantized rows (dab_upload_sq with rows, or dab_sq_encode_all)"
                                          : "%s: no MinMax rows (dab_upload_minmax with rows, or dab_minmax_encode_all)", who);
    // SQStore::distance_computer (providers inmem/scalar.rs:214-226): UnsupportedDistanceMetric
    if (sq && idx->metric == DAB_COSINE)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: the scalar-quantized store supports L2, InnerProduct and CosineNormalized", who);
    return DAB_OK;
}

int grow_visited_tables(const dab_index* idx, int& pass, uint64_t& slots) {
    if (++pass >= 6) return fail(DAB_ERR_VISITED_OVERFLOW, "search: visited set still overflowing after 6 passes");
    slots *= 4;
    // a visited set holds at most n_total + max_degree ids: 2 * n_total + 2048 slots take it below the 7/8 limit
    if (slots > 4 * idx->n_total() + 4096) slots = 2 * idx->n_total() + 2048;
    return DAB_OK;
}

int take_overflow_list(cudaStream_t stream, const uint32_t* d_overflow, uint32_t n_over, Scratch& retry) {
    // the pass that wrote the list is complete, so `retry` (its own work list, or empty) can be overwritten
    int rc;
    if ((rc = retry.reserve((size_t)n_over * 4))) return rc;
    DAB_CUDA(cudaMemcpyAsync(retry.p, d_overflow, (size_t)n_over * 4, cudaMemcpyDeviceToDevice, stream));
    DAB_CUDA(cudaStreamSynchronize(stream));
    return DAB_OK;
}

// ---- one batch of searches as a resumable job ------------------------------------------------
// A batch is launched (`launch`: kernel + read-back of the four counters into pinned memory, nothing
// waits) and later completed (`finish`: waits, learns the visited-set size, re-runs the few queries
// whose visited set outgrew its table).  The synchronous entry points run launch + finish on the
// handle's stream; dab_search_batch_async / dab_wait keep several batches in flight on slot-owned
// streams so the tail of one batch (workers running out of queries) is filled by the next batch's
// CTAs and the host<->device copies of neighbouring batches overlap the kernel.
struct SearchJob : SlotJob {
    dab_index* idx = nullptr;
    cudaStream_t stream = nullptr;
    Scratch* tables = nullptr;
    Scratch* counters = nullptr;
    Scratch* lists = nullptr;        // the whole lists, while deleted ids are filtered
    uint32_t* h_counters = nullptr;  // pinned, 4 words
    bool full_grid = false;          // batches in flight: launch every resident worker (the next batch fills what this one leaves)

    uint32_t nq = 0, l_search = 0, beam = 0;
    bool recording = false;
    // some id is deleted: the traversal writes every non-start entry of a list (k = L + #start) to `lists`, and each
    // pass is followed by the filter into `filtered`, the caller's buffers
    const uint32_t* deleted = nullptr;
    SearchOut filtered{};
    uint32_t k_out = 0;
    SearchParamsV2 p2;
    SearchParamsV3 p3;
    V2Launch v2;
    V3Launch v3;
    uint64_t slots = 0;
    int stage = 1;  // 0: search_kernel_v3 pass in flight, 1: global-table pass in flight
    int pass = 0;
    Scratch retry_list;
    uint32_t *d_counters = nullptr, *d_overflow = nullptr;

    int prepare(const void* d_queries, const uint32_t* d_query_rows, uint32_t nq_, uint32_t k, uint32_t l_search_, uint32_t beam_,
                uint32_t* d_ids, float* d_dists, uint32_t* d_counts, uint32_t* d_cmps, uint32_t* d_hops, uint32_t* rec_ids,
                float* rec_dists, uint32_t* rec_counts, uint32_t rec_cap);
    int launch() override;
    int finish() override;
    ~SearchJob() override { retry_list.release(); }
};

int SearchJob::prepare(const void* d_queries, const uint32_t* d_query_rows, uint32_t nq_, uint32_t k, uint32_t l_search_,
                       uint32_t beam_, uint32_t* d_ids, float* d_dists, uint32_t* d_counts, uint32_t* d_cmps, uint32_t* d_hops,
                       uint32_t* rec_ids, float* rec_dists, uint32_t* rec_counts, uint32_t rec_cap) {
    nq = nq_, l_search = l_search_, beam = beam_;
    recording = rec_ids != nullptr;

    int rc;
    // the build's insert searches ignore deletions, as the reference's insert does
    deleted = recording ? nullptr : deleted_filter(idx);
    if (deleted) {
        const size_t cap = (size_t)l_search + idx->n_start;
        if ((rc = lists->reserve((size_t)nq * cap * 8))) return rc;
        filtered = SearchOut{d_ids, d_dists, d_counts, d_cmps, d_hops};
        k_out = k;
        k = (uint32_t)cap;
        d_ids = (uint32_t*)lists->p;
        d_dists = (float*)(d_ids + (size_t)nq * cap);
    }
    memset(&p2, 0, sizeof(p2));
    if ((rc = v2_prepare(idx, l_search, beam, full_grid, p2, v2))) return rc;
    p2.vectors = idx->d_vectors;
    p2.row_stride = idx->row_stride;
    p2.adj = idx->d_adj;
    p2.adj_stride = idx->adj_stride;
    p2.n_points = idx->n_points;
    p2.n_start = idx->n_start;
    p2.dim = idx->dim;
    p2.max_degree = idx->max_degree;
    p2.queries = d_queries;
    p2.query_rows = d_query_rows;
    p2.k = k;
    p2.cap = l_search + idx->n_start;  // scratch.rs:195-208
    p2.beam = beam;
    p2.out_ids = d_ids;
    p2.out_dists = d_dists;
    p2.out_counts = d_counts;
    p2.out_cmps = d_cmps;
    p2.out_hops = d_hops;
    p2.rec_ids = rec_ids;
    p2.rec_dists = rec_dists;
    p2.rec_counts = rec_counts;
    p2.rec_cap = rec_cap;

    slots = table_slots(idx, idx->hint, l_search, beam, STORE_PQ);
    if ((rc = counters->reserve(16 + (size_t)nq * 4))) return rc;
    d_counters = (uint32_t*)counters->p;
    d_overflow = d_counters + 4;
    p2.counters = d_counters;
    p2.overflow_list = d_overflow;
    p2.n_work = nq;
    p2.query_list = nullptr;

    // first pass with the visited sets in shared memory (search_kernel_v3) where it is the faster
    // kernel; queries that outgrow their table are re-run on global tables
    stage = 1;
    pass = 0;
    const uint32_t need = idx->tune.test_visited_log2 ? (1u << idx->tune.test_visited_log2) / 2 : 0;  // tests: tables that overflow
    const bool skip = idx->v3_overflow_l == l_search && idx->v3_overflow_beam == beam && idx->v3_overflow_frac > 0.25f;
    memset(&p3, 0, sizeof(p3));
    if (!skip && v3_prepare(idx, l_search, beam, need, p3, v3) == 0) {
        stage = 0;
        p3.vectors = p2.vectors, p3.row_stride = p2.row_stride, p3.adj = p2.adj, p3.adj_stride = p2.adj_stride;
        p3.n_points = p2.n_points, p3.n_start = p2.n_start, p3.dim = p2.dim, p3.max_degree = p2.max_degree;
        p3.queries = p2.queries, p3.query_rows = p2.query_rows, p3.query_list = nullptr, p3.n_work = nq;
        p3.k = p2.k, p3.cap = p2.cap, p3.beam = p2.beam;
        p3.out_ids = p2.out_ids, p3.out_dists = p2.out_dists, p3.out_counts = p2.out_counts;
        p3.out_cmps = p2.out_cmps, p3.out_hops = p2.out_hops;
        p3.rec_ids = p2.rec_ids, p3.rec_dists = p2.rec_dists, p3.rec_counts = p2.rec_counts, p3.rec_cap = p2.rec_cap;
        p3.counters = d_counters, p3.overflow_list = d_overflow;
    }
    return DAB_OK;
}

// launch the pass of the current stage and queue the read-back of its counters
int SearchJob::launch() {
    DAB_CUDA(cudaMemsetAsync(d_counters, 0, 16, stream));
    if (stage == 0) {
        v3.kern<<<balanced_grid(nq, v3.grid, kV3Warps), kV3Warps * 32, v3.smem_block, stream>>>(p3);
    } else {
        // a visited table per warp: `slots` rounded up to whole 32-byte buckets of 8 ids
        const uint32_t n_buckets = (uint32_t)((slots + 7) / 8);
        int rc;
        if ((rc = tables->reserve((size_t)v2.grid * kV2Warps * n_buckets * 32))) return rc;
        p2.tables = (uint32_t*)tables->p;
        p2.n_buckets = n_buckets;
        int launch_grid = balanced_grid(p2.n_work, v2.grid, kV2Warps);
        if (full_grid) launch_grid = (int)std::min<uint64_t>((uint64_t)v2.grid, ((uint64_t)p2.n_work + kV2Warps - 1) / kV2Warps);
        v2.kern<<<launch_grid, kV2Warps * 32, v2.smem_block, stream>>>(p2);
    }
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    // the whole batch: a re-run pass rewrote some of the lists
    int rc;
    if (deleted && (rc = queue_drop_deleted(idx, stream, deleted, p2.out_ids, p2.out_dists, p2.cap, nq, k_out, filtered))) return rc;
    DAB_CUDA(cudaMemcpyAsync(h_counters, d_counters, 16, cudaMemcpyDeviceToHost, stream));
    return DAB_OK;
}

int SearchJob::finish() {
    for (;;) {
        DAB_CUDA(cudaStreamSynchronize(stream));
        idx->rec_truncated += h_counters[3];
        const uint32_t n_over = h_counters[1];
        if (!recording) {  // build-time searches run on a growing graph: do not learn from them
            learn_visited(idx->hint, l_search, beam, STORE_PQ, h_counters[2]);
            if (stage == 0) {
                idx->v3_overflow_l = l_search;
                idx->v3_overflow_beam = beam;
                idx->v3_overflow_frac = (float)n_over / (float)nq;
            }
        }
        if (n_over == 0) return DAB_OK;
        // re-run the overflowed queries on (larger) global tables
        reran = true;
        int rc;
        if ((rc = take_overflow_list(stream, d_overflow, n_over, retry_list))) return rc;
        p2.query_list = (const uint32_t*)retry_list.p;
        p2.n_work = n_over;
        if (stage == 0) {
            // the overflowed queries are the largest: size the global tables from the estimate again
            stage = 1;
            slots = std::max(slots, table_slots(idx, VisitedHint{}, l_search, beam, STORE_PQ));
        } else if ((rc = grow_visited_tables(idx, pass, slots))) {
            return rc;
        }
        if ((rc = launch())) return rc;
    }
}

// Runs the search over work items on the handle's stream and waits; device pointers only.  `rec_*` optional.
int run_search(dab_index* idx, const void* d_queries, const uint32_t* d_query_rows, uint32_t nq, uint32_t k,
               uint32_t l_search, uint32_t beam, uint32_t* d_ids, float* d_dists, uint32_t* d_counts, uint32_t* d_cmps,
               uint32_t* d_hops, uint32_t* rec_ids, float* rec_dists, uint32_t* rec_counts, uint32_t rec_cap) {
    int rc;
    if ((rc = check_search_args(idx, k, l_search, beam))) return rc;
    if (nq == 0) return DAB_OK;
    if ((rc = idx->h_counters.reserve(16))) return rc;
    SearchJob job;
    job.idx = idx;
    job.stream = idx->stream;
    job.tables = &idx->s_tables;
    job.counters = &idx->s_counters;
    job.lists = &idx->s_ids;
    job.h_counters = (uint32_t*)idx->h_counters.p;
    if ((rc = job.prepare(d_queries, d_query_rows, nq, k, l_search, beam, d_ids, d_dists, d_counts, d_cmps, d_hops, rec_ids,
                          rec_dists, rec_counts, rec_cap)))
        return rc;
    if ((rc = job.launch())) return rc;
    return job.finish();
}

// ---- host-buffer calls -------------------------------------------------------------------------
// reserves the query and result buffers of a host-buffer call (`q`; ids and dists in `out`, counts / cmps / hops in
// `stats`); nothing is queued
static int reserve_host_call(const dab_index* idx, Scratch& q, Scratch& out, Scratch& stats, uint32_t nq, uint32_t k, SearchOut* d) {
    const size_t qbytes = (size_t)nq * idx->dim * elem_size(idx->dtype);
    const size_t rbytes = (size_t)nq * k * 4;
    int rc;
    if ((rc = q.reserve(qbytes)) || (rc = out.reserve(2 * rbytes)) || (rc = stats.reserve((size_t)nq * 12))) return rc;
    uint32_t* st = (uint32_t*)stats.p;
    *d = SearchOut{(uint32_t*)out.p, (float*)((uint8_t*)out.p + rbytes), st, st + nq, st + 2 * (size_t)nq};
    return DAB_OK;
}

static int queue_query_copy(const dab_index* idx, cudaStream_t stream, void* d_queries, const void* queries, uint32_t nq) {
    DAB_CUDA(cudaMemcpyAsync(d_queries, queries, (size_t)nq * idx->dim * elem_size(idx->dtype), cudaMemcpyHostToDevice, stream));
    return DAB_OK;
}

static int queue_result_copies(cudaStream_t stream, const HostCopy& c) {
    const size_t rbytes = (size_t)c.nq * c.k * 4, sbytes = (size_t)c.nq * 4;
    DAB_CUDA(cudaMemcpyAsync(c.host.ids, c.dev.ids, rbytes, cudaMemcpyDeviceToHost, stream));
    DAB_CUDA(cudaMemcpyAsync(c.host.dists, c.dev.dists, rbytes, cudaMemcpyDeviceToHost, stream));
    if (c.host.counts) DAB_CUDA(cudaMemcpyAsync(c.host.counts, c.dev.counts, sbytes, cudaMemcpyDeviceToHost, stream));
    if (c.host.cmps) DAB_CUDA(cudaMemcpyAsync(c.host.cmps, c.dev.cmps, sbytes, cudaMemcpyDeviceToHost, stream));
    if (c.host.hops) DAB_CUDA(cudaMemcpyAsync(c.host.hops, c.dev.hops, sbytes, cudaMemcpyDeviceToHost, stream));
    return DAB_OK;
}

int search_host_buffers(dab_index* idx, const char* api, const void* queries, uint32_t nq, uint32_t k, const SearchOut& out,
                        const std::function<int(const void* d_queries, const SearchOut& d_out)>& run) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", api);
    if (nq == 0) return DAB_OK;
    if (!queries || !out.ids || !out.dists) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL argument", api);
    if (k == 0) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: k must be > 0", api);
    DAB_CUDA(cudaSetDevice(idx->device));
    HostCopy c{{}, out, nq, k};
    int rc;
    if ((rc = reserve_host_call(idx, idx->s_queries, idx->s_out, idx->s_stats, nq, k, &c.dev)) ||
        (rc = queue_query_copy(idx, idx->stream, idx->s_queries.p, queries, nq)) || (rc = run(idx->s_queries.p, c.dev)) ||
        (rc = queue_result_copies(idx->stream, c)))
        return rc;
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    return DAB_OK;
}

// ---- batches in flight (dab_search_batch[_pq|_sq|_minmax][_device]_async / dab_wait) ----
void search_slots_release(dab_index* idx) {
    for (int i = 0; i < DAB_MAX_SLOTS; ++i) {
        SearchSlot* s = (SearchSlot*)idx->slots[i];
        if (!s) continue;
        if (s->stream) cudaStreamSynchronize(s->stream);
        delete s->job;
        s->tables.release(), s->counters.release(), s->queries.release(), s->out.release(), s->stats.release(), s->h_counters.release();
        s->stage.release(), s->luts.release(), s->lists.release();
        if (s->stream) cudaStreamDestroy(s->stream);
        delete s;
        idx->slots[i] = nullptr;
    }
}

int retire_quantized_stores(dab_index* idx) {
    for (int i = 0; i < DAB_MAX_SLOTS; ++i) {
        const SearchSlot* s = (const SearchSlot*)idx->slots[i];
        if (s && s->stream) DAB_CUDA(cudaStreamSynchronize(s->stream));
    }
    ++idx->stores_version;
    return DAB_OK;
}

static int slot_of(dab_index* idx, uint32_t slot, SearchSlot** out) {
    if (slot >= DAB_MAX_SLOTS) return fail(DAB_ERR_INVALID_ARGUMENT, "search: slot %u out of range (DAB_MAX_SLOTS = %d)", slot, DAB_MAX_SLOTS);
    SearchSlot* s = (SearchSlot*)idx->slots[slot];
    if (!s) {
        s = new SearchSlot();
        s->h_counters.pinned_host = true;
        if (cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking) != cudaSuccess) {
            delete s;
            return fail(DAB_ERR_CUDA, "search: cannot create the stream of slot %u", slot);
        }
        idx->slots[slot] = s;
    }
    *out = s;
    return DAB_OK;
}

int slot_submit(dab_index* idx, const char* api, uint32_t slot, bool host, const void* queries, uint32_t nq, uint32_t k,
                const SearchOut& out, const std::function<int(SearchSlot* s, const void* d_queries, const SearchOut& d_out, SlotJob** job)>& prepare) {
    DAB_CUDA(cudaSetDevice(idx->device));
    SearchSlot* s = nullptr;
    int rc;
    if ((rc = slot_of(idx, slot, &s))) return rc;
    if (s->job) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: slot %u still has a batch in flight (call dab_wait)", api, slot);
    if (nq == 0) return DAB_OK;
    HostCopy c{out, SearchOut{}, nq, k};
    if (host) {
        c.host = out;
        if ((rc = reserve_host_call(idx, s->queries, s->out, s->stats, nq, k, &c.dev))) return rc;
    }
    const void* d_queries = host ? s->queries.p : queries;
    SlotJob* job = nullptr;
    if ((rc = prepare(s, d_queries, c.dev, &job))) {
        delete job;
        return rc;
    }
    if ((host && (rc = queue_query_copy(idx, s->stream, s->queries.p, queries, nq))) || (rc = job->launch())) {
        // a launch that failed half way (a CUDA error: every buffer was reserved by prepare) may have queued work that
        // writes the caller's buffers: it completes before the error is returned, and the slot is idle
        cudaStreamSynchronize(s->stream);
        delete job;
        return rc;
    }
    s->job = job;
    s->host_out = c;
    // optimistic copies: valid as they are unless a query overflowed (then dab_wait repeats them)
    return host ? queue_result_copies(s->stream, c) : DAB_OK;
}

// a full-precision batch on slot `s`: every resident worker is launched (the next batch fills what this one leaves)
static int prepare_search_job(dab_index* idx, SearchSlot* s, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                              uint32_t beam, const SearchOut& d, SlotJob** out) {
    int rc;
    if ((rc = s->h_counters.reserve(16))) return rc;
    SearchJob* job = new SearchJob();
    *out = job;
    job->idx = idx;
    job->stream = s->stream;
    job->tables = &s->tables;
    job->counters = &s->counters;
    job->lists = &s->lists;
    job->h_counters = (uint32_t*)s->h_counters.p;
    job->full_grid = true;
    return job->prepare(d_queries, nullptr, nq, k, l_search, beam, d.ids, d.dists, d.counts, d.cmps, d.hops, nullptr, nullptr, nullptr, 0);
}

}  // namespace dab

using namespace dab;

extern "C" {

int dab_search_batch_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                            uint32_t beam_width, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts,
                            uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_search_batch: idx is NULL");
    if (nq && (!d_queries || !d_out_ids || !d_out_dists)) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_search_batch: NULL argument");
    DAB_CUDA(cudaSetDevice(idx->device));
    return run_search(idx, d_queries, nullptr, nq, k, l_search, beam_width, d_out_ids, d_out_dists, d_out_counts,
                      d_out_cmps, d_out_hops, nullptr, nullptr, nullptr, 0);
}

int dab_search_batch(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                     uint32_t beam_width, uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                     uint32_t* out_cmps, uint32_t* out_hops) {
    return search_host_buffers(idx, "dab_search_batch", queries, nq, k, SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops},
                               [&](const void* d_queries, const SearchOut& d) {
                                   return run_search(idx, d_queries, nullptr, nq, k, l_search, beam_width, d.ids, d.dists, d.counts,
                                                     d.cmps, d.hops, nullptr, nullptr, nullptr, 0);
                               });
}

// ---- asynchronous batches: launch on a slot, collect with dab_wait ---------------------------
// Host-buffer flavour: the queries are copied from `queries` on the slot's stream (pinned memory makes
// the copy asynchronous), the kernel follows, and the results are copied into the host outputs; all of
// it is queued by this call when no query can overflow its visited table on the way, i.e. nothing waits.
// dab_wait(slot) blocks until the slot's batch is complete (and, in the rare overflow case, re-runs the
// affected queries and repeats the result copies).  The buffers must stay valid until dab_wait returns.
int dab_search_batch_async(dab_index* idx, uint32_t slot, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                           uint32_t beam_width, uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps,
                           uint32_t* out_hops) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_search_batch_async: idx is NULL");
    if (nq && (!queries || !out_ids || !out_dists)) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_search_batch_async: NULL argument");
    int rc;
    if ((rc = check_search_args(idx, k, l_search, beam_width))) return rc;
    return slot_submit(idx, "dab_search_batch_async", slot, true, queries, nq, k, SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops},
                       [&](SearchSlot* s, const void* d_queries, const SearchOut& d, SlotJob** job) {
                           return prepare_search_job(idx, s, d_queries, nq, k, l_search, beam_width, d, job);
                       });
}

int dab_search_batch_device_async(dab_index* idx, uint32_t slot, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                  uint32_t beam_width, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts,
                                  uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_search_batch_device_async: idx is NULL");
    if (nq && (!d_queries || !d_out_ids || !d_out_dists)) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_search_batch_device_async: NULL argument");
    int rc;
    if ((rc = check_search_args(idx, k, l_search, beam_width))) return rc;
    return slot_submit(idx, "dab_search_batch_device_async", slot, false, d_queries, nq, k,
                       SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops},
                       [&](SearchSlot* s, const void* dq, const SearchOut& d, SlotJob** job) {
                           return prepare_search_job(idx, s, dq, nq, k, l_search, beam_width, d, job);
                       });
}

// Joins a batch of any kind.  In the rare overflow case the job's re-runs (and, for a quantized batch with rerank, the
// rerank of the whole batch) are queued again by finish: they are waited for here, after the result copies of a
// host-buffer call are queued once more.
int dab_wait(dab_index* idx, uint32_t slot) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_wait: idx is NULL");
    if (slot >= DAB_MAX_SLOTS) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_wait: slot %u out of range (DAB_MAX_SLOTS = %d)", slot, DAB_MAX_SLOTS);
    SearchSlot* s = (SearchSlot*)idx->slots[slot];
    if (!s || !s->job) return DAB_OK;
    DAB_CUDA(cudaSetDevice(idx->device));
    SlotJob* job = s->job;
    s->job = nullptr;
    DAB_CUDA(cudaStreamSynchronize(s->stream));
    int rc = job->finish();
    const bool reran = job->reran;
    delete job;
    if (rc) return rc;
    if (reran) {
        if (s->host_out.host.ids && (rc = queue_result_copies(s->stream, s->host_out))) return rc;
        DAB_CUDA(cudaStreamSynchronize(s->stream));
    }
    return DAB_OK;
}

}  // extern "C"
