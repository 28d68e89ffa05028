// search_kernel.cu — the host side of batched graph search: the visited-table policy, the one job that runs a batch of
// any kind with its overflow re-runs and post-processing (full precision; PQ, SQ and MinMax, whose kernels and rerank
// are in search_kernel_pq.cu and search_kernel_pqs.cu), the slots of batches in flight and the C entry points
// (dab_search_batch[_pq|_pq_rerank|_sq|_minmax][_device][_async], dab_search_batch_diverse[_pq|_sq|_minmax][_device],
// dab_search_batch_filtered[_pq|_sq|_minmax][_device], dab_wait).  The diverse search (search_diverse.cu), over full-precision rows or a
// quantized store, is one more kind of the job; so are the filtered search (search_filtered.cu), over full-precision
// rows or a quantized store, and the first phase of
// range search (search_range.cu), a batch over full-precision rows or a quantized store that keeps start points and
// deleted ids.
//
// A full-precision batch runs on search_kernel_v3 (visited set in shared memory) where its short lists make that the
// faster kernel, and on search_kernel_v2 (global visited tables) otherwise; queries whose visited set outgrows its table
// are re-run on v2 with larger tables, so membership stays exact.  Both kernels restate DiskANNIndex::search_internal
// (index.rs:1933-2000) bit for bit.
#include "dab_common.cuh"
#include "search_diverse.cuh"
#include "search_filtered.cuh"
#include "search_host.cuh"
#include "search_pq.cuh"
#include "search_v2.cuh"
#include "search_v3.cuh"

#include <algorithm>
#include <cmath>

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

// `hint` takes in the largest visited set of a pass at (L, beam, mode)
static void learn_visited(VisitedHint& hint, uint32_t l_search, uint32_t beam, QuantStore mode, uint32_t visited) {
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

// The `n_over` query ids a pass reported at `d_overflow` become the work list of the next pass, in `retry`
static int take_overflow_list(cudaStream_t stream, const uint32_t* d_overflow, uint32_t n_over, Scratch& retry) {
    // the pass that wrote the list is complete, so `retry` (its own work list, or empty) can be overwritten
    int rc;
    if ((rc = retry.reserve((size_t)n_over * 4))) return rc;
    DAB_CUDA(cudaMemcpyAsync(retry.p, d_overflow, (size_t)n_over * 4, cudaMemcpyDeviceToDevice, stream));
    DAB_CUDA(cudaStreamSynchronize(stream));
    return DAB_OK;
}

int stage_store_queries(const dab_index* idx, cudaStream_t stream, Scratch& stage, int store, const void* d_queries, uint32_t nq,
                        uint32_t* h_counters, StagedQueries& out) {
    if (store == STORE_SQ) return sq_stage_queries(idx, stream, stage, d_queries, nq, &out.codes, &out.meta);
    if (store == STORE_MINMAX)
        return minmax_stage_queries(idx, stream, stage, d_queries, nq, (unsigned long long*)(h_counters + 4), &out.codes, &out.meta);
    return DAB_OK;
}

// The checks of a batch that need no plan: the arguments and, for a quantized traversal, the store, its metric and the
// list length
static int check_batch_args(const dab_index* idx, uint32_t k, uint32_t l_search, uint32_t beam, int store) {
    if (store < 0) return check_search_args(idx, k, l_search, beam);
    const QuantStore mode = (QuantStore)store;
    // every entry point of a store reports under its synchronous host-buffer call's name
    const char* who = mode == STORE_PQ ? "dab_search_batch_pq" : mode == STORE_SQ ? "dab_search_batch_sq" : "dab_search_batch_minmax";
    int rc;
    if ((rc = check_search_args(idx, k, l_search, beam, false)) || (rc = check_quant_store(idx, mode, who, false))) return rc;
    if (l_search + idx->n_start > 1024)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: L + #start must be <= 1024", mode == STORE_MINMAX ? "dab_search_batch_minmax" : "dab_search_batch_pq");
    return DAB_OK;
}

// ---- one batch as a resumable job ------------------------------------------------------------------------------------
// `prepare` plans the batch (check_batch_args has passed), makes the checks of the plan and reserves every buffer the
// first pass needs; nothing is queued.  `launch` queues all of the batch and waits for nothing: the staging of the
// queries (SQ, MinMax), the first pass with the read-back of its counters into pinned memory and, optimistically, the
// post-processing (the rerank, or the filter of deleted ids).  `finish` waits for the counters, learns the visited-set
// size, re-runs the queries whose visited set outgrew its table on larger tables and then queues the post-processing of
// the whole batch again; `reran` says it did (the results were written again after the first copies were queued).
// The synchronous calls run the job on the handle's stream and scratch.  The *_async calls keep several batches in
// flight on slot-owned streams, so that the tail of one batch (workers running out of queries) is filled by the next
// batch's CTAs and the host<->device copies of neighbouring batches overlap the kernel.  A re-run of a quantized batch
// reads the store the batch was planned on: if that store was replaced since (retire_quantized_stores), finish fails.
struct SlotJob {
    dab_index* idx;
    cudaStream_t stream;
    Scratch *tables, *counters, *stage, *luts, *lists, *pinned;
    bool full_grid = false;  // full precision, batches in flight: launch every resident worker (the next batch fills what this one leaves)

    int store = -1;  // -1: full precision, else the QuantStore the traversal reads
    bool rerank = false;
    // > 0: a diverse search with at most diverse_k results per attribute value, over full-precision rows or `store`; its
    // local queues are `pool` entries for every warp a pass launches, in `pools` (the synchronous calls' own region: a
    // PQ traversal's tables stay in `luts`, as in every quantized kind)
    uint32_t diverse_k = 0;
    uint64_t pool = 0;
    Scratch* pools = nullptr;
    // set: a filtered search over full-precision rows or `store` (FilterSpec, search_filtered.cuh)
    const FilterSpec* filt = nullptr;
    const void* d_queries = nullptr;
    uint32_t nq = 0, k = 0, l_search = 0, beam = 0, cap = 0;
    SearchRecord rec{};  // searches over rows of the index (rec.query_rows set)
    // some id is deleted: a rerank drops deleted ids itself; without one (`filter`) the traversal writes every non-start
    // entry of a list (k = L + #start) to `lists` and the filter takes the first k live ones into `filtered`, the caller's
    // buffers
    const uint32_t* deleted = nullptr;
    bool filter = false;
    SearchOut out{}, filtered{};  // `out`: where the traversal writes
    uint32_t *d_counters = nullptr, *d_overflow = nullptr;
    uint32_t* h_counters = nullptr;  // pinned: the four counters of a pass, then (u64 at word 4) the MinMax NaN flag
    cudaEvent_t counted = nullptr;   // recorded after the read-back of a pass's counters
    uint64_t stores_version = 0;     // idx->stores_version when the batch was planned
    // global-table passes: the n_work queries of `work` (NULL: the whole batch), a visited table of `slots` ids for each
    // of `warps` resident warps; the overflowed queries of one pass are re-run on larger tables in the next
    const uint32_t* work = nullptr;
    uint32_t n_work = 0, warps = 0, n_buckets = 0;
    uint64_t slots = 0;
    int pass = 0;
    Scratch retry;
    bool reran = false;

    // full precision
    SearchParamsV2 p2;
    SearchParamsV3 p3;
    V2Launch v2;
    V3Launch v3;
    bool on_v3 = false;  // the first pass runs on search_kernel_v3
    // quantized: staged queries and rerank lists, which each kind's launch copies into its parameter block
    StagedQueries staged{};
    uint32_t *list_ids = nullptr, *list_counts = nullptr;
    SearchParamsPq pq;
    PqsPlan plan;
    bool use_pqs = false;
    PqKernel kern = nullptr;
    int grid = 0;
    size_t smem_block = 0;
    // diverse
    SearchParamsDiverse pd;
    WarpPlan<SearchParamsDiverse> dplan;
    // filtered
    SearchParamsFiltered pf;
    WarpPlan<SearchParamsFiltered> fplan;

    SlotJob(dab_index* idx_, cudaStream_t stream_, Scratch& tables_, Scratch& counters_, Scratch& stage_, Scratch& luts_,
            Scratch& lists_, Scratch& pinned_)
        : idx(idx_), stream(stream_), tables(&tables_), counters(&counters_), stage(&stage_), luts(&luts_), lists(&lists_), pinned(&pinned_) {}
    ~SlotJob() {
        retry.release();
        if (counted) cudaEventDestroy(counted);
    }

    int prepare(const void* d_queries_, uint32_t nq_, uint32_t k_, uint32_t l_search_, uint32_t beam_, const SearchOut& d, int store_,
                bool rerank_, const SearchRecord* rec_);
    int launch() {
        int rc;
        if ((rc = stage_queries()) || (rc = launch_pass())) return rc;
        return post();
    }
    int finish();

    int plan_full();
    int plan_quant();
    int plan_diverse();
    int plan_filtered();
    template <class P>
    int plan_store(P& p);
    int reserve_quant();
    int reserve_tables();
    int reserve_pools();
    // SQ and MinMax: the batch's queries compressed by the store's quantizer (MinMax: the NaN flag read back into h_counters)
    int stage_queries() { return stage_store_queries(idx, stream, *stage, store, d_queries, nq, h_counters, staged); }
    int launch_pass();
    int launch_full();
    int launch_quant();
    int launch_diverse();
    int launch_filtered();
    int post();

    // full precision keeps STORE_PQ in a hint of its own
    VisitedHint& hint() const { return store < 0 ? idx->hint : idx->pq_hint; }
    QuantStore mode() const { return store < 0 ? STORE_PQ : (QuantStore)store; }
    unsigned long long first_nan() const { return staged_first_nan(h_counters); }
    int nan_error() const {
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_search_batch_minmax: query %llu contains NaN after the transform (InputContainsNaN)", first_nan());
    }

    // the fields of a parameter block that every traversal's pass has
    template <class P>
    void set_batch_params(P& p) const {
        set_graph_params(idx, p);
        p.queries = d_queries;
        p.n_work = nq;
        p.k = filter ? cap : k;
        p.cap = cap;
        p.beam = beam;
        p.out_ids = out.ids, p.out_dists = out.dists, p.out_counts = out.counts, p.out_cmps = out.cmps, p.out_hops = out.hops;
        p.counters = d_counters;
        p.overflow_list = d_overflow;
    }
    // ... and those of search_kernel_v2 and _v3
    template <class P>
    void set_full_params(P& p) const {
        set_batch_params(p);
        p.vectors = idx->d_vectors;
        p.row_stride = idx->row_stride;
        p.query_rows = rec.query_rows;
        p.rec_ids = rec.ids, p.rec_dists = rec.dists, p.rec_counts = rec.counts, p.rec_cap = rec.cap;
        p.result_bound = rec.keep_starts ? idx->n_total() : idx->n_points;
    }
    // a global-table pass: its work list and tables
    template <class P>
    void set_pass_params(P& p) const {
        p.query_list = work;
        p.n_work = n_work;
        p.tables = (uint32_t*)tables->p;
        p.n_buckets = n_buckets;
    }
    // a quantized traversal's staged queries (into `q`: the block, or its StoreParams) and rerank lists
    template <class P, class Q>
    void set_quant_inputs(P& p, Q& q) const {
        q.query_codes = staged.codes, q.query_meta = staged.meta;
        p.list_ids = list_ids, p.list_counts = list_counts, p.list_cap = rerank ? cap : 0;
    }
};

int SlotJob::prepare(const void* d_queries_, uint32_t nq_, uint32_t k_, uint32_t l_search_, uint32_t beam_, const SearchOut& d,
                     int store_, bool rerank_, const SearchRecord* rec_) {
    d_queries = d_queries_, nq = nq_, k = k_, l_search = l_search_, beam = beam_, store = store_, rerank = rerank_;
    if (rec_) rec = *rec_;
    stores_version = idx->stores_version;
    // scratch.rs:195-208; a diverse search's list holds L (Diverse::create_scratch, diverse_search.rs:149-177), and a
    // filtered search's results are the first L matches
    cap = diverse_k || filt ? l_search : l_search + idx->n_start;
    int rc;
    if ((rc = pinned->reserve(24)) || (rc = counters->reserve(16 + (size_t)nq * 4))) return rc;
    h_counters = (uint32_t*)pinned->p;
    d_counters = (uint32_t*)counters->p;
    d_overflow = d_counters + 4;
    out = d;
    // searches over rows of the index ignore deletions, as the reference's insert and in-place delete do
    deleted = rec.query_rows || rec.keep_deleted ? nullptr : deleted_filter(idx);
    filter = deleted && !rerank;
    if (filter) {
        if ((rc = lists->reserve((size_t)nq * cap * 8))) return rc;
        filtered = d;
        out.ids = (uint32_t*)lists->p;
        out.dists = (float*)(out.ids + (size_t)nq * cap);
    }
    n_work = nq;
    // a diverse search visits other nodes than a k-NN search, and a filtered one's list may grow: they neither read nor
    // teach the hints; a filtered search's tables are sized for its longest list
    if (filt) slots = table_slots(idx, VisitedHint{}, std::max(l_search, filt->best_max), beam, mode());
    else slots = table_slots(idx, diverse_k ? VisitedHint{} : hint(), l_search, beam, mode());
    if ((rc = filt ? plan_filtered() : diverse_k ? plan_diverse() : store < 0 ? plan_full() : plan_quant())) return rc;
    if (!on_v3 && (rc = reserve_tables())) return rc;
    DAB_CUDA(cudaEventCreateWithFlags(&counted, cudaEventDisableTiming));
    return DAB_OK;
}

// full precision: search_kernel_v2's plan, and search_kernel_v3's for the first pass where it is the faster kernel
int SlotJob::plan_full() {
    int rc;
    memset(&p2, 0, sizeof(p2));
    if ((rc = v2_prepare(idx, l_search, beam, full_grid, p2, v2))) return rc;
    set_full_params(p2);
    warps = (uint32_t)v2.grid * kV2Warps;
    // queries that outgrow their table in search_kernel_v3 are re-run on global tables; v3 is skipped where most did so
    const uint32_t need = idx->tune.test_visited_log2 ? (1u << idx->tune.test_visited_log2) / 2 : 0;  // tests: tables that overflow
    const bool skip = idx->v3_overflow_l == l_search && idx->v3_overflow_beam == beam && idx->v3_overflow_frac > 0.25f;
    memset(&p3, 0, sizeof(p3));
    on_v3 = !skip && v3_prepare(idx, l_search, beam, need, p3, v3) == 0;
    if (on_v3) set_full_params(p3);
    return DAB_OK;
}

// PQ, SQ and MinMax: the shared-memory layout, search_kernel_pqs's plan or search_kernel_pq's grid, and the LUTs, rerank
// lists and query staging
int SlotJob::plan_quant() {
    const QuantStore mode = (QuantStore)store;
    memset(&pq, 0, sizeof(pq));
    set_batch_params(pq);
    set_store_params(idx, mode, pq);

    size_t off = 0;
    pq.off_q = 0;
    off += round_up((size_t)idx->dim * 4, 16);
    const size_t cap_pad = round_up(cap, 32) + 32;
    pq.off_qd = (uint32_t)off;
    off += cap_pad * 4;
    pq.off_qi = (uint32_t)off;
    off += cap_pad * 4;
    const size_t ncand_max = std::max<size_t>((size_t)beam * idx->max_degree, idx->n_start);
    pq.off_cid = (uint32_t)off;
    off += round_up(ncand_max * 4, 16);
    pq.off_cd = (uint32_t)off;
    off += round_up(ncand_max * 4, 16);
    pq.off_beam = (uint32_t)off;
    off += round_up((size_t)beam * 4, 16);
    pq.off_qc = (uint32_t)off;
    if (mode == STORE_SQ) off += pq.code_stride;
    if (mode == STORE_MINMAX) off += pq.code_stride + 16;  // the query's code row and its four compensations
    off = round_up(off, 16);
    pq.off_nrow = (uint32_t)off;  // search_kernel_pqs: the adjacency row copied one hop ahead
    if (mode == STORE_PQ) off += 96 * 4;
    pq.warp_smem = (uint32_t)round_up(off, 16);
    // table metrics with a pivot table that fits shared memory: search_kernel_pqs (pivots resident per SM, entries
    // computed on the fly); everything else — SQ, MinMax, DirectCosine, wide pivots, > 32 chunks — search_kernel_pq
    memset(&plan, 0, sizeof(plan));
    // (a list that keeps its start points, range search's first phase, runs on search_kernel_pq_starts)
    use_pqs = mode == STORE_PQ && !pq.direct_cosine && !rec.keep_starts && pqs_plan(idx, pq.warp_smem, nq, &plan);
    smem_block = (size_t)pq.warp_smem * kPqWarps;
    if (use_pqs) {
        pq.piv_stride = plan.piv_stride;
        pq.piv_bytes = plan.piv_bytes;
        grid = plan.grid;
        warps = (uint32_t)plan.grid * (uint32_t)plan.warps;
    } else {
        if (smem_block > 200 * 1024) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_search_batch_pq: configuration needs %zu B shared memory per CTA", smem_block);
        kern = pq_kernel(cap, mode, rec.keep_starts);
        int per_sm = ctas_per_sm(kern, kPqWarps * 32, smem_block);
        if (per_sm < 1) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_search_batch_pq: kernel does not fit");
        // every resident warp owns a LUT (n_chunks x n_centers f32: 32 KB at 32 x 256) and a visited table in
        // global memory; ADC terms and probes are L2 hits only while all of them stay L2-resident
        // (the SQ kernel has no LUT: it keeps the occupancy the shared memory allows)
        if (mode == STORE_PQ) per_sm = std::min(per_sm, 6);
        grid = (int)std::min<uint64_t>((uint64_t)per_sm * idx->sm_count, ((uint64_t)nq + kPqWarps - 1) / kPqWarps);
        warps = (uint32_t)grid * kPqWarps;
    }

    int rc;
    if ((rc = luts->reserve(std::max<size_t>(use_pqs ? 0 : pq_table_bytes(idx, store, warps, true), 16)))) return rc;
    pq.luts = (float*)luts->p;
    if (rerank && (rc = check_rerank(idx, "dab_search_batch_pq", cap))) return rc;
    return reserve_quant();
}

// diverse: the kernel's plan, the attribute table and the local queues of the first pass
int SlotJob::plan_diverse() {
    memset(&pd, 0, sizeof(pd));
    int rc;
    if ((rc = diverse_plan(idx, l_search, beam, store, pd, dplan))) return rc;
    set_batch_params(pd);
    pd.vectors = idx->d_vectors;
    pd.row_stride = idx->row_stride;
    pd.attr_values = idx->d_attr_values;
    pd.attr_present = idx->d_attr_present;
    pd.diverse_k = diverse_k;
    // diverse_priority_queue.rs:96 in 64 bits; a local queue holds distinct ids, so a capacity of n_total never fills
    // and every larger one behaves the same
    pd.local_cap = (uint32_t)std::min<uint64_t>((uint64_t)diverse_k * l_search / k, idx->n_total());
    warps = (uint32_t)dplan.grid * dplan.warps;
    if (store >= 0 && (rc = plan_store(pd))) return rc;
    pool = diverse_pool_first(idx, l_search);
    return reserve_pools();
}

// A diverse or filtered traversal over `store` (the `warps` of its grid planned): the store, a PQ table for every warp
// of the grid, and reserve_quant's buffers (the rerank's lists hold at most L ids a query: cap = L)
template <class P>
int SlotJob::plan_store(P& p) {
    set_store_params(idx, (QuantStore)store, p.store);
    int rc;
    if ((rc = luts->reserve(std::max<size_t>(pq_table_bytes(idx, store, warps), 16)))) return rc;
    p.store.luts = (float*)luts->p;
    return reserve_quant();
}

// a quantized traversal's rerank lists (at most cap ids a query, then every query's count) and the staging of its queries
int SlotJob::reserve_quant() {
    int rc;
    if (rerank) {
        if ((rc = lists->reserve(((size_t)nq * cap + nq) * 4))) return rc;
        list_ids = (uint32_t*)lists->p;
        list_counts = list_ids + (size_t)nq * cap;
    }
    return stage->reserve(store == STORE_SQ ? sq_stage_bytes(idx, nq) : store == STORE_MINMAX ? minmax_stage_bytes(idx, nq) : 0);
}

// filtered: the kernel's plan, the label table, the masks and adaptive L's table; over a store, plan_store's buffers
int SlotJob::plan_filtered() {
    memset(&pf, 0, sizeof(pf));
    int rc;
    if ((rc = filtered_plan(idx, l_search, filt->best_max, beam, store, pf, fplan))) return rc;
    set_batch_params(pf);
    pf.vectors = idx->d_vectors;
    pf.row_stride = idx->row_stride;
    pf.labels = idx->d_labels;
    pf.masks = filt->masks;
    pf.match_all = filt->match_all;
    pf.best_cap = l_search + idx->n_start;
    pf.samples = filt->adapt ? filt->samples : 0;
    pf.span = beam * idx->max_degree;
    pf.adapt = filt->adapt;
    warps = (uint32_t)fplan.grid * fplan.warps;
    return store >= 0 ? plan_store(pf) : DAB_OK;
}

// the local queues of the warps the next pass over n_work queries launches (warp_launch's grid)
int SlotJob::reserve_pools() {
    int rc;
    const uint64_t pass_warps = (uint64_t)dplan.pass_grid(n_work) * dplan.warps;
    if ((rc = pools->reserve((size_t)pass_warps * pool * 16))) return rc;
    pd.pools = (uint32_t*)pools->p;
    pd.pool_cap = (uint32_t)pool;
    return DAB_OK;
}

// a visited table of `slots` ids, in whole 32-byte buckets of 8 ids, for every resident warp
int SlotJob::reserve_tables() {
    n_buckets = (uint32_t)((slots + 7) / 8);
    return tables->reserve((size_t)warps * n_buckets * 32);
}

// one traversal pass over the queries of `work` (tables reserved) and the read-back of its counters
int SlotJob::launch_pass() {
    DAB_CUDA(cudaMemsetAsync(d_counters, 0, 16, stream));
    int rc;
    if ((rc = filt ? launch_filtered() : diverse_k ? launch_diverse() : store < 0 ? launch_full() : launch_quant())) return rc;
    DAB_CUDA(cudaMemcpyAsync(h_counters, d_counters, 16, cudaMemcpyDeviceToHost, stream));
    DAB_CUDA(cudaEventRecord(counted, stream));
    return DAB_OK;
}

int SlotJob::launch_full() {
    if (on_v3) {
        v3.kern<<<balanced_grid(nq, v3.grid, kV3Warps), kV3Warps * 32, v3.smem_block, stream>>>(p3);
    } else {
        set_pass_params(p2);
        int launch_grid = balanced_grid(n_work, v2.grid, kV2Warps);
        if (full_grid) launch_grid = (int)std::min<uint64_t>((uint64_t)v2.grid, ((uint64_t)n_work + kV2Warps - 1) / kV2Warps);
        v2.kern<<<launch_grid, kV2Warps * 32, v2.smem_block, stream>>>(p2);
    }
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    return DAB_OK;
}

int SlotJob::launch_quant() {
    set_pass_params(pq);
    set_quant_inputs(pq, pq);
    if (use_pqs) return pqs_launch(pq, plan, cap, stream);
    kern<<<grid, kPqWarps * 32, smem_block, stream>>>(pq);
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    return DAB_OK;
}

int SlotJob::launch_diverse() {
    set_pass_params(pd);
    set_quant_inputs(pd, pd.store);
    return warp_launch(pd, dplan, dplan.pass_grid(n_work), stream);
}

int SlotJob::launch_filtered() {
    set_pass_params(pf);
    set_quant_inputs(pf, pf.store);
    return warp_launch(pf, fplan, fplan.pass_grid(n_work), stream);
}

// the post-processing of the whole batch: the rerank, or the filter of deleted ids
int SlotJob::post() {
    if (rerank) return launch_rerank(idx, stream, d_queries, nq, k, cap, list_ids, list_counts, out.ids, out.dists, out.counts, deleted);
    if (filter) return queue_drop_deleted(idx, stream, deleted, out.ids, out.dists, cap, nq, k, filtered, idx->n_points);
    return DAB_OK;
}

int SlotJob::finish() {
    DAB_CUDA(cudaEventSynchronize(counted));
    if (store == STORE_MINMAX && first_nan() != ~0ull) return nan_error();
    for (;;) {
        const uint32_t n_over = h_counters[1];
        if (rec.query_rows) {
            idx->rec_truncated += h_counters[3];
        } else if (!diverse_k && !filt) {  // searches over rows run on a graph being changed: do not learn from them
            learn_visited(hint(), l_search, beam, mode(), h_counters[2]);
            if (on_v3) {
                idx->v3_overflow_l = l_search;
                idx->v3_overflow_beam = beam;
                idx->v3_overflow_frac = (float)n_over / (float)nq;
            }
        }
        if (n_over == 0) break;
        // the store the batch was planned on has been freed: its overflowed queries cannot be re-run
        if (store >= 0 && idx->stores_version != stores_version)
            return fail(DAB_ERR_INVALID_ARGUMENT, "dab_wait: a quantized store was replaced while the batch was in flight; "
                                                  "%u of its queries could not be re-run", n_over);
        int rc;
        if ((rc = take_overflow_list(stream, d_overflow, n_over, retry))) return rc;
        if (on_v3) {
            // the overflowed queries are the largest: size the global tables from the estimate again
            on_v3 = false;
            slots = std::max(slots, table_slots(idx, VisitedHint{}, l_search, beam, mode()));
        } else if ((!diverse_k || n_over > h_counters[3]) && (rc = grow_visited_tables(idx, pass, slots))) {
            // (a diverse pass counts in counters[3] the queries that stopped on their local queues instead)
            return rc;
        }
        if ((rc = reserve_tables())) return rc;
        work = (const uint32_t*)retry.p;
        n_work = n_over;
        if (diverse_k) {
            if (h_counters[3]) {
                const uint64_t grown = diverse_pool_grow(idx, pool);
                // a pool of n_total entries takes every id: it cannot overflow
                if (grown == pool)
                    return fail(DAB_ERR_VISITED_OVERFLOW, "dab_search_batch_diverse: local queues outgrew %llu entries",
                                (unsigned long long)pool);
                pool = grown;
            }
            if ((rc = reserve_pools())) return rc;
        }
        reran = true;
        if ((rc = launch_pass())) return rc;
        DAB_CUDA(cudaEventSynchronize(counted));
    }
    // the post-processing queued by launch read lists that the re-runs have since rewritten
    return reran ? post() : DAB_OK;
}

// The checks of a diverse search (DiverseSearchParams::new, diverse_search.rs:80-97; Diverse::new, :119-134), all made
// before any device work.  diverse_k > k is accepted: the reference declares DiverseKGreaterThanTotalK and never returns it.
// Over a quantized store (`store` >= 0) the store checks of the synchronous quantized call follow, reported under `api`.
static int check_diverse_args(const dab_index* idx, const char* api, uint32_t k, uint32_t l_search, uint32_t beam, uint32_t diverse_k,
                              int store = -1, bool rerank = false) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", api);
    int rc;
    if ((rc = check_search_args(idx, k, l_search, beam, store < 0))) return rc;
    if (diverse_k == 0) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: diverse k_value cannot be zero", api);
    if (l_search < k) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: l_value (%u) must be greater than or equal to total_k_value (%u)", api, l_search, k);
    if (l_search > kDiverseMaxL) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: l_value %u > %u", api, l_search, kDiverseMaxL);
    if ((rc = diverse_check_smem(idx, api, l_search, beam, store))) return rc;
    if (!idx->d_attr_values) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: no attribute table (dab_upload_attributes has not been called)", api);
    if (store < 0) return DAB_OK;
    if ((rc = check_quant_store(idx, (QuantStore)store, api, false))) return rc;
    return rerank ? check_rerank(idx, api, l_search) : DAB_OK;
}

// `diverse_k` > 0: a diverse search, whose arguments check_diverse_args has passed; `filt`: a filtered search, whose
// arguments check_filtered_args has passed
static int run_job(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam, const SearchOut& d,
                   int store, bool rerank, const SearchRecord* rec, uint32_t diverse_k, const FilterSpec* filt = nullptr) {
    int rc;
    if (!diverse_k && !filt && (rc = check_batch_args(idx, k, l_search, beam, store))) return rc;
    if (nq == 0) return DAB_OK;
    SlotJob job(idx, idx->stream, idx->s_tables, idx->s_counters, idx->s_stage, idx->s_out2, idx->s_ids, idx->h_counters);
    job.diverse_k = diverse_k;
    job.filt = filt;
    job.pools = &idx->s_pools;
    if ((rc = job.prepare(d_queries, nq, k, l_search, beam, d, store, rerank, rec)) || (rc = job.stage_queries())) return rc;
    if (rec && rec->staged) *rec->staged = job.staged;
    if (store == STORE_MINMAX) {  // a batch with a NaN query fails before any traversal is launched
        DAB_CUDA(cudaStreamSynchronize(idx->stream));
        if (job.first_nan() != ~0ull) return job.nan_error();
    }
    if ((rc = job.launch_pass()) || (rc = job.post()) || (rc = job.finish())) return rc;
    if (store < 0 && job.filter) DAB_CUDA(cudaStreamSynchronize(idx->stream));  // the filter follows the counters
    return DAB_OK;
}

int run_search(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam, const SearchOut& d,
               int store, bool rerank, const SearchRecord* rec) {
    return run_job(idx, d_queries, nq, k, l_search, beam, d, store, rerank, rec, 0);
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

// ---- the entry points' helpers: `store` -1 (full precision) or a QuantStore; `api` names the call in error messages ----
// The synchronous host-buffer calls: checks the buffers, copies the queries to the handle's scratch, runs the batch on
// them with device result buffers, copies the results to `out` and waits.
static int search_host(dab_index* idx, const char* api, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                       uint32_t beam, const SearchOut& out, int store, bool rerank, uint32_t diverse_k = 0, const FilterSpec* filt = nullptr) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", api);
    if (nq == 0) return DAB_OK;
    if (!queries || !out.ids || !out.dists) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL argument", api);
    if (k == 0) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: k must be > 0", api);
    DAB_CUDA(cudaSetDevice(idx->device));
    HostCopy c{{}, out, nq, k};
    int rc;
    if ((rc = reserve_host_call(idx, idx->s_queries, idx->s_out, idx->s_stats, nq, k, &c.dev)) ||
        (rc = queue_query_copy(idx, idx->stream, idx->s_queries.p, queries, nq)) ||
        (rc = run_job(idx, idx->s_queries.p, nq, k, l_search, beam, c.dev, store, rerank, nullptr, diverse_k, filt)) ||
        (rc = queue_result_copies(idx->stream, c)))
        return rc;
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    return DAB_OK;
}

// The synchronous device-buffer calls (run_search).  The full-precision call makes its argument checks before it returns
// for an empty batch; the quantized calls return first.
static int search_device(dab_index* idx, const char* api, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                         uint32_t beam, const SearchOut& d, int store, bool rerank, uint32_t diverse_k = 0, const FilterSpec* filt = nullptr) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", api);
    if (nq == 0 && store >= 0) return DAB_OK;
    if (nq && (!d_queries || !d.ids || !d.dists)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL argument", api);
    DAB_CUDA(cudaSetDevice(idx->device));
    return run_job(idx, d_queries, nq, k, l_search, beam, d, store, rerank, nullptr, diverse_k, filt);
}

// The diverse search over a quantized store: every argument and store check before the queries are copied; the device
// form waits for the rerank or the filter of deleted ids, so that it returns with its outputs complete
static int search_diverse_quant(dab_index* idx, const char* api, bool host, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                uint32_t beam, uint32_t diverse_k, int rerank, const SearchOut& out, QuantStore store) {
    int rc;
    if ((rc = check_diverse_args(idx, api, k, l_search, beam, diverse_k, store, rerank != 0))) return rc;
    if (host) return search_host(idx, api, queries, nq, k, l_search, beam, out, store, rerank != 0, diverse_k);
    if ((rc = search_device(idx, api, queries, nq, k, l_search, beam, out, store, rerank != 0, diverse_k))) return rc;
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    return DAB_OK;
}

// The checks of a filtered search, all made before any device work: InlineFilterSearch's (k >= 1 and L >= k from Knn::new,
// scale >= 1.0 from AdaptiveL::new, which a NaN scale does not pass either), the label table, and what the kernel holds:
// L + #start and floor(L * scale) at most kFilteredMaxL, and its shared memory.  *best_max: the longest list.  Over a
// quantized store (`store` >= 0) the store checks of the synchronous quantized call follow, reported under `api`.
static int check_filtered_args(const dab_index* idx, const char* api, uint32_t k, uint32_t l_search, uint32_t beam,
                               uint32_t adaptive_samples, double adaptive_scale, uint32_t* best_max, int store, bool rerank) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", api);
    int rc;
    if ((rc = check_search_args(idx, k, l_search, beam, store < 0))) return rc;
    if (l_search < k) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: l_value (%u) must be greater than or equal to k_value (%u)", api, l_search, k);
    if (adaptive_samples && !(adaptive_scale >= 1.0)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: adaptive L scale factor must be >= 1.0", api);
    if (!idx->d_labels) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: no label table (dab_upload_labels has not been called)", api);
    if ((uint64_t)l_search + idx->n_start > kFilteredMaxL)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: L + #start = %llu > %u", api, (unsigned long long)l_search + idx->n_start, kFilteredMaxL);
    *best_max = l_search + idx->n_start;
    if (adaptive_samples) {
        const double grown = std::floor((double)l_search * adaptive_scale);
        if (grown > kFilteredMaxL)
            return fail(DAB_ERR_INVALID_ARGUMENT, "%s: floor(L * scale) = %.17g > %u", api, grown, kFilteredMaxL);
        *best_max = std::max(*best_max, (uint32_t)grown);
    }
    if ((rc = filtered_check_smem(idx, api, l_search, *best_max, beam, store))) return rc;
    if (store < 0) return DAB_OK;
    if ((rc = check_quant_store(idx, (QuantStore)store, api, false))) return rc;
    return rerank ? check_rerank(idx, api, l_search) : DAB_OK;
}

// InlineFilterSearch::search over a batch: the checks, then the masks (host call: copied to the handle's scratch) and
// adaptive L's table on the device, then the job.  `store` -1: full-precision rows, else the traversal reads that store
// and `rerank` reorders the first L matches by full-precision distance.  The device form returns with its outputs
// complete.
static int search_filtered(dab_index* idx, const char* api, bool host, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                           uint32_t beam, const uint64_t* masks, uint32_t match_all, uint32_t adaptive_samples, double adaptive_scale,
                           const SearchOut& out, int store = -1, bool rerank = false) {
    uint32_t best_max = 0;
    int rc;
    if ((rc = check_filtered_args(idx, api, k, l_search, beam, adaptive_samples, adaptive_scale, &best_max, store, rerank))) return rc;
    if (nq == 0) return DAB_OK;
    if (!masks) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL argument", api);
    DAB_CUDA(cudaSetDevice(idx->device));
    // the sample counts distinct evaluated neighbours, data points only: past n_points it is never reached
    const bool adaptive = adaptive_samples && adaptive_samples <= idx->n_points;
    const uint32_t span = beam * idx->max_degree;
    std::vector<uint16_t> table;
    if (adaptive) table = adaptive_table(l_search, adaptive_samples, span, adaptive_scale);
    const size_t mask_bytes = host ? round_up((size_t)nq * 8, 16) : 0;
    if ((rc = idx->s_pools.reserve(mask_bytes + table.size() * 2 + 16))) return rc;
    FilterSpec spec{masks, match_all, adaptive_samples, nullptr, best_max};
    if (host) {
        DAB_CUDA(cudaMemcpyAsync(idx->s_pools.p, masks, (size_t)nq * 8, cudaMemcpyHostToDevice, idx->stream));
        spec.masks = (const uint64_t*)idx->s_pools.p;
    }
    if (adaptive) {
        spec.adapt = (const uint16_t*)((uint8_t*)idx->s_pools.p + mask_bytes);
        DAB_CUDA(cudaMemcpyAsync((void*)spec.adapt, table.data(), table.size() * 2, cudaMemcpyHostToDevice, idx->stream));
    }
    if (host) return search_host(idx, api, queries, nq, k, l_search, beam, out, store, rerank, 0, &spec);
    if ((rc = search_device(idx, api, queries, nq, k, l_search, beam, out, store, rerank, 0, &spec))) return rc;
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    return DAB_OK;
}

// ---- batches in flight (dab_search_batch*_async / dab_wait) --------------------------------------------------------
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

// The *_async calls: the job on the slot's stream and scratch.  After the argument checks, the slot is checked (in range,
// no batch in flight); nq == 0 is then a no-op.  A host-buffer call (`host`) gets device buffers in the slot's scratch.
// The job is prepared with every check the synchronous call makes before it launches; then the copy of the queries, the
// job's launch and the copies of the results are queued, and the call returns without waiting.
static int search_async(dab_index* idx, const char* api, uint32_t slot, bool host, const void* queries, uint32_t nq, uint32_t k,
                        uint32_t l_search, uint32_t beam, const SearchOut& out, int store, bool rerank) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", api);
    if (nq && (!queries || !out.ids || !out.dists)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL argument", api);
    int rc;
    if ((rc = check_batch_args(idx, k, l_search, beam, store))) return rc;
    DAB_CUDA(cudaSetDevice(idx->device));
    SearchSlot* s = nullptr;
    if ((rc = slot_of(idx, slot, &s))) return rc;
    if (s->job) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: slot %u still has a batch in flight (call dab_wait)", api, slot);
    if (nq == 0) return DAB_OK;
    HostCopy c{out, SearchOut{}, nq, k};
    if (host) {
        c.host = out;
        if ((rc = reserve_host_call(idx, s->queries, s->out, s->stats, nq, k, &c.dev))) return rc;
    }
    SlotJob* job = new SlotJob(idx, s->stream, s->tables, s->counters, s->stage, s->luts, s->lists, s->h_counters);
    job->full_grid = true;
    if ((rc = job->prepare(host ? s->queries.p : queries, nq, k, l_search, beam, c.dev, store, rerank, nullptr))) {
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

}  // namespace dab

using namespace dab;

extern "C" {

int dab_search_batch(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                     uint32_t beam_width, uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                     uint32_t* out_cmps, uint32_t* out_hops) {
    return search_host(idx, "dab_search_batch", queries, nq, k, l_search, beam_width,
                       SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, -1, false);
}

// returns with the outputs complete, the filter of deleted ids included
int dab_search_batch_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                            uint32_t beam_width, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts,
                            uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    return search_device(idx, "dab_search_batch", d_queries, nq, k, l_search, beam_width,
                         SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, -1, false);
}

int dab_search_batch_pq(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                        uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops) {
    return search_host(idx, "dab_search_batch_pq", queries, nq, k, l_search, beam_width,
                       SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, STORE_PQ, false);
}

int dab_search_batch_pq_rerank(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                               uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops) {
    return search_host(idx, "dab_search_batch_pq_rerank", queries, nq, k, l_search, beam_width,
                       SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, STORE_PQ, true);
}

// The quantized *_device calls return once the traversal is complete; the rerank or the filter may still run
int dab_search_batch_pq_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                               int rerank, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts, uint32_t* d_out_cmps,
                               uint32_t* d_out_hops) {
    return search_device(idx, "dab_search_batch_pq_device", d_queries, nq, k, l_search, beam_width,
                         SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, STORE_PQ, rerank != 0);
}

int dab_search_batch_sq(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                        int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops) {
    return search_host(idx, "dab_search_batch_sq", queries, nq, k, l_search, beam_width,
                       SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, STORE_SQ, rerank != 0);
}

int dab_search_batch_sq_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                               int rerank, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts, uint32_t* d_out_cmps,
                               uint32_t* d_out_hops) {
    return search_device(idx, "dab_search_batch_sq_device", d_queries, nq, k, l_search, beam_width,
                         SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, STORE_SQ, rerank != 0);
}

int dab_search_batch_minmax(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                            int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops) {
    return search_host(idx, "dab_search_batch_minmax", queries, nq, k, l_search, beam_width,
                       SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, STORE_MINMAX, rerank != 0);
}

int dab_search_batch_minmax_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                                   int rerank, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts, uint32_t* d_out_cmps,
                                   uint32_t* d_out_hops) {
    return search_device(idx, "dab_search_batch_minmax_device", d_queries, nq, k, l_search, beam_width,
                         SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, STORE_MINMAX, rerank != 0);
}

// Diverse::search (diverse_search.rs:189-234): every argument is checked before the queries are copied
int dab_search_batch_diverse(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                             uint32_t diverse_k, uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps,
                             uint32_t* out_hops) {
    int rc;
    if ((rc = check_diverse_args(idx, "dab_search_batch_diverse", k, l_search, beam_width, diverse_k))) return rc;
    return search_host(idx, "dab_search_batch_diverse", queries, nq, k, l_search, beam_width,
                       SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, -1, false, diverse_k);
}

// returns with the outputs complete, the filter of deleted ids included
int dab_search_batch_diverse_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                                    uint32_t diverse_k, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts,
                                    uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    int rc;
    if ((rc = check_diverse_args(idx, "dab_search_batch_diverse_device", k, l_search, beam_width, diverse_k))) return rc;
    return search_device(idx, "dab_search_batch_diverse_device", d_queries, nq, k, l_search, beam_width,
                         SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, -1, false, diverse_k);
}

int dab_search_batch_diverse_pq(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                                uint32_t diverse_k, int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps,
                                uint32_t* out_hops) {
    return search_diverse_quant(idx, "dab_search_batch_diverse_pq", true, queries, nq, k, l_search, beam_width, diverse_k, rerank,
                                SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, STORE_PQ);
}

int dab_search_batch_diverse_pq_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                       uint32_t beam_width, uint32_t diverse_k, int rerank, uint32_t* d_out_ids, float* d_out_dists,
                                       uint32_t* d_out_counts, uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    return search_diverse_quant(idx, "dab_search_batch_diverse_pq_device", false, d_queries, nq, k, l_search, beam_width, diverse_k, rerank,
                                SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, STORE_PQ);
}

int dab_search_batch_diverse_sq(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                                uint32_t diverse_k, int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps,
                                uint32_t* out_hops) {
    return search_diverse_quant(idx, "dab_search_batch_diverse_sq", true, queries, nq, k, l_search, beam_width, diverse_k, rerank,
                                SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, STORE_SQ);
}

int dab_search_batch_diverse_sq_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                       uint32_t beam_width, uint32_t diverse_k, int rerank, uint32_t* d_out_ids, float* d_out_dists,
                                       uint32_t* d_out_counts, uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    return search_diverse_quant(idx, "dab_search_batch_diverse_sq_device", false, d_queries, nq, k, l_search, beam_width, diverse_k, rerank,
                                SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, STORE_SQ);
}

int dab_search_batch_diverse_minmax(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                                    uint32_t diverse_k, int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                                    uint32_t* out_cmps, uint32_t* out_hops) {
    return search_diverse_quant(idx, "dab_search_batch_diverse_minmax", true, queries, nq, k, l_search, beam_width, diverse_k, rerank,
                                SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, STORE_MINMAX);
}

int dab_search_batch_diverse_minmax_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                           uint32_t beam_width, uint32_t diverse_k, int rerank, uint32_t* d_out_ids, float* d_out_dists,
                                           uint32_t* d_out_counts, uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    return search_diverse_quant(idx, "dab_search_batch_diverse_minmax_device", false, d_queries, nq, k, l_search, beam_width, diverse_k,
                                rerank, SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, STORE_MINMAX);
}

// InlineFilterSearch::search (inline_filter_search.rs:89-160): every argument is checked before the masks and the queries
// are copied
int dab_search_batch_filtered(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                              const uint64_t* query_masks, uint32_t match_all, uint32_t adaptive_samples, double adaptive_scale,
                              uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops) {
    return search_filtered(idx, "dab_search_batch_filtered", true, queries, nq, k, l_search, beam_width, query_masks, match_all,
                           adaptive_samples, adaptive_scale, SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops});
}

// query_masks is a device pointer; returns with the outputs complete, the filter of deleted ids included
int dab_search_batch_filtered_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                     uint32_t beam_width, const uint64_t* d_query_masks, uint32_t match_all, uint32_t adaptive_samples,
                                     double adaptive_scale, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts,
                                     uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    return search_filtered(idx, "dab_search_batch_filtered_device", false, d_queries, nq, k, l_search, beam_width, d_query_masks,
                           match_all, adaptive_samples, adaptive_scale,
                           SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops});
}

// InlineFilterSearch::search over the PQ, SQ and MinMax stores: the traversal distances of dab_search_batch_{pq,sq,minmax};
// rerank != 0 runs Pipeline<FilterStartPoints, Rerank> over the first L matches
int dab_search_batch_filtered_pq(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                                 const uint64_t* query_masks, uint32_t match_all, uint32_t adaptive_samples, double adaptive_scale,
                                 int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps,
                                 uint32_t* out_hops) {
    return search_filtered(idx, "dab_search_batch_filtered_pq", true, queries, nq, k, l_search, beam_width, query_masks, match_all,
                           adaptive_samples, adaptive_scale, SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, STORE_PQ,
                           rerank != 0);
}

int dab_search_batch_filtered_pq_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                        uint32_t beam_width, const uint64_t* d_query_masks, uint32_t match_all, uint32_t adaptive_samples,
                                        double adaptive_scale, int rerank, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts,
                                        uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    return search_filtered(idx, "dab_search_batch_filtered_pq_device", false, d_queries, nq, k, l_search, beam_width, d_query_masks,
                           match_all, adaptive_samples, adaptive_scale,
                           SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, STORE_PQ, rerank != 0);
}

int dab_search_batch_filtered_sq(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                                 const uint64_t* query_masks, uint32_t match_all, uint32_t adaptive_samples, double adaptive_scale,
                                 int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps,
                                 uint32_t* out_hops) {
    return search_filtered(idx, "dab_search_batch_filtered_sq", true, queries, nq, k, l_search, beam_width, query_masks, match_all,
                           adaptive_samples, adaptive_scale, SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, STORE_SQ,
                           rerank != 0);
}

int dab_search_batch_filtered_sq_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                        uint32_t beam_width, const uint64_t* d_query_masks, uint32_t match_all, uint32_t adaptive_samples,
                                        double adaptive_scale, int rerank, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts,
                                        uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    return search_filtered(idx, "dab_search_batch_filtered_sq_device", false, d_queries, nq, k, l_search, beam_width, d_query_masks,
                           match_all, adaptive_samples, adaptive_scale,
                           SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, STORE_SQ, rerank != 0);
}

int dab_search_batch_filtered_minmax(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search, uint32_t beam_width,
                                     const uint64_t* query_masks, uint32_t match_all, uint32_t adaptive_samples, double adaptive_scale,
                                     int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps,
                                     uint32_t* out_hops) {
    return search_filtered(idx, "dab_search_batch_filtered_minmax", true, queries, nq, k, l_search, beam_width, query_masks, match_all,
                           adaptive_samples, adaptive_scale, SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, STORE_MINMAX,
                           rerank != 0);
}

int dab_search_batch_filtered_minmax_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                            uint32_t beam_width, const uint64_t* d_query_masks, uint32_t match_all,
                                            uint32_t adaptive_samples, double adaptive_scale, int rerank, uint32_t* d_out_ids,
                                            float* d_out_dists, uint32_t* d_out_counts, uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    return search_filtered(idx, "dab_search_batch_filtered_minmax_device", false, d_queries, nq, k, l_search, beam_width, d_query_masks,
                           match_all, adaptive_samples, adaptive_scale,
                           SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, STORE_MINMAX, rerank != 0);
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
    return search_async(idx, "dab_search_batch_async", slot, true, queries, nq, k, l_search, beam_width,
                        SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, -1, false);
}

int dab_search_batch_device_async(dab_index* idx, uint32_t slot, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                  uint32_t beam_width, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts,
                                  uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    return search_async(idx, "dab_search_batch_device_async", slot, false, d_queries, nq, k, l_search, beam_width,
                        SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, -1, false);
}

int dab_search_batch_pq_async(dab_index* idx, uint32_t slot, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                              uint32_t beam_width, int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                              uint32_t* out_cmps, uint32_t* out_hops) {
    return search_async(idx, "dab_search_batch_pq_async", slot, true, queries, nq, k, l_search, beam_width,
                        SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, STORE_PQ, rerank != 0);
}

int dab_search_batch_pq_device_async(dab_index* idx, uint32_t slot, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                     uint32_t beam_width, int rerank, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts,
                                     uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    return search_async(idx, "dab_search_batch_pq_device_async", slot, false, d_queries, nq, k, l_search, beam_width,
                        SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, STORE_PQ, rerank != 0);
}

int dab_search_batch_sq_async(dab_index* idx, uint32_t slot, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                              uint32_t beam_width, int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                              uint32_t* out_cmps, uint32_t* out_hops) {
    return search_async(idx, "dab_search_batch_sq_async", slot, true, queries, nq, k, l_search, beam_width,
                        SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, STORE_SQ, rerank != 0);
}

int dab_search_batch_sq_device_async(dab_index* idx, uint32_t slot, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                     uint32_t beam_width, int rerank, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts,
                                     uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    return search_async(idx, "dab_search_batch_sq_device_async", slot, false, d_queries, nq, k, l_search, beam_width,
                        SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, STORE_SQ, rerank != 0);
}

int dab_search_batch_minmax_async(dab_index* idx, uint32_t slot, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                  uint32_t beam_width, int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                                  uint32_t* out_cmps, uint32_t* out_hops) {
    return search_async(idx, "dab_search_batch_minmax_async", slot, true, queries, nq, k, l_search, beam_width,
                        SearchOut{out_ids, out_dists, out_counts, out_cmps, out_hops}, STORE_MINMAX, rerank != 0);
}

int dab_search_batch_minmax_device_async(dab_index* idx, uint32_t slot, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                         uint32_t beam_width, int rerank, uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts,
                                         uint32_t* d_out_cmps, uint32_t* d_out_hops) {
    return search_async(idx, "dab_search_batch_minmax_device_async", slot, false, d_queries, nq, k, l_search, beam_width,
                        SearchOut{d_out_ids, d_out_dists, d_out_counts, d_out_cmps, d_out_hops}, STORE_MINMAX, rerank != 0);
}

// Joins a batch of any kind.  In the rare overflow case the job's re-runs (and then the rerank or the filter of the whole
// batch) are queued again by finish: they are waited for here, after the result copies of a host-buffer call are queued
// once more.
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
