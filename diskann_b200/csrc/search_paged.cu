// search_paged.cu — paged search on the device: DiskANNIndex::paged_search (diskann/src/graph/index.rs:2075-2155) and
// PagedSearch::next_page (graph/search/paged.rs:53-149) for a whole query batch, each query's state resident in HBM
// between pages (dab_paged_search_begin / _next / _end).
//
// The reference's session is a resizable NeighborPriorityQueue of search_param_l = L + #start (queue.rs:108-119: it grows
// and never evicts), a visited set seeded with the start ids, and the cumulative cmps / hops of search_internal.  Its
// order is total: distance ascending, later insertion first among equal distances (lower-bound insertion), NaN never
// enters.  Exploration and the pages only ever look at the first L + #start entries, so a query keeps those — the
// window — sorted (id | visited flag, distance, insertion number), and everything behind them in an unsorted tail
// with the insertion number, from which the front of the order is selected again after a page drains the window.
//
// Per query, in HBM:
//   window   [cap] distance, id | visited flag, insertion number (cap = L + #start), and the counters below;
//   tail     entries that fell behind the window (a merge that pushed them past cap, or a full window that rejected them);
//   visited  a bucketed table (search_common.cuh, 8 ids per 32-byte bucket) and an append-only log of every id inserted.
// The tail holds queued ids and the log visited ids, so both fit in the table's load limit (7/8 of its slots).
//
// A call works on the window and counters in shared memory and writes them back only when it completes.  During the
// search the tail and the log are only appended to, so a query whose table passes 7/8 full simply stops uncommitted:
// the host gives it a table four times larger, rebuilt from the log up to its committed length (the tail is copied up
// to its committed length), and runs that query's call again from its committed state.  Membership is exact at any size.
//
// The session logic (paged_queries) does not depend on how distances are made.  paged_kernel reads full-precision rows;
// paged_kernel_quant reads the PQ, SQ or MinMax store with the per-candidate code of the one-shot quantized traversal
// (quant_device.cuh), so a page carries the same quantized distances (dab_paged_search_begin_{pq,sq,minmax}).  Nothing
// a session reads between pages lives in the index's shared scratch: the compressed SQ / MinMax queries are session
// memory, and a PQ query's table is rebuilt at every call in the session's own table scratch.
#include "dab_common.cuh"
#include "search_common.cuh"
#include "search_host.cuh"
#include "search_pq.cuh"
#include "search_source.cuh"

#include <algorithm>
#include <vector>

namespace dab {

namespace {

constexpr int kPagedWarps = 4;  // warps per CTA, one query each

// where one query's growing state lives (the window and counters have fixed strides)
struct PagedQuery {
    uint32_t* table;  // n_buckets * 8 ids
    uint32_t* log;    // tcap ids
    float* td;        // tail: tcap distances, ids | visited flag, insertion numbers
    uint32_t* ti;
    uint32_t* ts;
    uint32_t n_buckets;
    uint32_t tcap;
};

// committed counters of a query
enum { C_SIZE = 0, C_CURSOR, C_TAIL, C_LOG, C_CMPS, C_HOPS, C_SEQ, C_WORDS = 8 };

struct PagedParams {
    const uint8_t* vectors;
    size_t row_stride;
    const uint32_t* adj;
    uint32_t adj_stride;
    uint64_t n_points;
    uint32_t n_start, dim, max_degree;
    const void* queries;
    const uint32_t* work;  // query ids to run (NULL: 0 .. n_work-1)
    uint32_t n_work;
    uint32_t* counters;       // [0] work taken, [1] overflowed queries
    uint32_t* overflow_list;  // the overflowed query ids
    int begin;                // 1: DiskANNIndex::paged_search, 0: next_page
    uint32_t k, cap;
    PagedQuery* qs;
    float* wd;
    uint32_t *wi, *ws, *ctr;
    uint32_t* out_ids;
    float* out_dists;
    uint32_t *out_counts, *out_cmps, *out_hops;
    uint32_t warp_smem, off_cid, off_cd, off_wd, off_wi, off_ws;
    StoreParams store;  // the quantized sessions (paged_kernel_quant); SQ / MinMax queries are the session's
};

// (distance ascending, insertion number descending) as one ascending 64-bit key; -0.0 and +0.0 compare equal
__device__ __forceinline__ uint64_t order_key(float d, uint32_t seq) {
    uint32_t b = __float_as_uint(d == 0.0f ? 0.0f : d);
    b = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    return ((uint64_t)b << 32) | (uint32_t)~seq;
}

// appends the entries of the lanes with `leave` to the tail (lane order)
__device__ __forceinline__ void tail_push(const PagedQuery& st, uint32_t& tlen, bool leave, float d, uint32_t id, uint32_t seq, int lane) {
    const unsigned m = __ballot_sync(kFull, leave);
    if (leave) {
        const uint32_t at = tlen + __popc(m & ((1u << lane) - 1u));
        st.td[at] = d;
        st.ti[at] = id;
        st.ts[at] = seq;
    }
    tlen += __popc(m);
}

// NeighborPriorityQueue::insert (queue.rs:130-171, resizable) of candidates c0 .. c0+m-1 (m <= 32, lane j owns candidate
// j, inserted in lane order) into the window: the rank merge of search_common.cuh (merge_round_chunked) in tiles of 32
// from the top, with the insertion numbers moving along, and every entry whose final position is >= cap — old or new —
// appended to the tail instead of dropped.  NaN candidates are ignored.
__device__ __forceinline__ void merge_paged(float* wd, uint32_t* wi, uint32_t* ws, uint32_t cap, uint32_t& size, uint32_t& cursor,
                                            uint32_t& seq, const PagedQuery& st, uint32_t& tlen, const uint32_t* cid,
                                            const float* cd, uint32_t c0, uint32_t m, int lane) {
    const uint32_t j = (uint32_t)lane;
    const float dj = j < m ? cd[c0 + j] : __int_as_float(0x7FC00000);
    const uint32_t idj = j < m ? cid[c0 + j] : 0;
    const bool valid = j < m && dj == dj;
    const unsigned vm = __ballot_sync(kFull, valid);
    if (!vm) return;
    const uint32_t sj = seq + __popc(vm & ((1u << lane) - 1u));
    uint32_t lo = 0, hi = size;
    while (__any_sync(kFull, lo < hi)) {
        const uint32_t mid = (lo + hi) >> 1;
        if (lo < hi) {
            if (wd[mid] < dj) lo = mid + 1;
            else hi = mid;
        }
    }
    uint32_t rn = 0;
    for (unsigned it = vm; it;) {
        const int i = __ffs(it) - 1;
        it &= it - 1;
        const float di = __shfl_sync(kFull, dj, i);
        rn += (di < dj || (di == dj && (uint32_t)i > j)) ? 1u : 0u;
    }
    const uint32_t pos = lo + rn;
    __syncwarp();
#pragma unroll 1
    for (uint32_t c = (size + 31) / 32; c-- > 0;) {
        const uint32_t e = c * 32 + j;
        const bool have = e < size;
        const float od = have ? wd[e] : __int_as_float(0x7F800000);
        const uint32_t oi = have ? wi[e] : kEmptyV2;
        const uint32_t os = have ? ws[e] : 0;
        uint32_t sh = 0;
        for (unsigned it = vm; it;) {
            const int i = __ffs(it) - 1;
            it &= it - 1;
            sh += __shfl_sync(kFull, dj, i) <= od ? 1u : 0u;
        }
        __syncwarp();  // the whole tile is in registers before any of it is overwritten
        const uint32_t ne = e + sh;
        if (have && sh != 0 && ne < cap) {
            wd[ne] = od;
            wi[ne] = oi;
            ws[ne] = os;
        }
        tail_push(st, tlen, have && ne >= cap, od, oi, os, lane);
        __syncwarp();
    }
    const bool keep = valid && pos < cap;
    if (keep) {
        wd[pos] = dj;
        wi[pos] = idj;
        ws[pos] = sj;
    }
    tail_push(st, tlen, valid && !keep, dj, idj, sj, lane);
    size = min(cap, size + (uint32_t)__popc(vm));
    cursor = min(cursor, __reduce_min_sync(kFull, keep ? pos : 0xFFFFFFFFu));
    seq += __popc(vm);
    __syncwarp();
}

// One warp's share of a pass: the session logic of paged search for every query it takes, whatever the distances are.
// Src is a distance source (search_source.cuh): load(q) runs before the query's window is read back, prepare() once
// the window is in place.
template <class Src>
__device__ __forceinline__ void paged_queries(const PagedParams& p, uint8_t* base, int lane, Src& src) {
    uint32_t* cid = reinterpret_cast<uint32_t*>(base + p.off_cid);
    float* cd = reinterpret_cast<float*>(base + p.off_cd);
    float* wd = reinterpret_cast<float*>(base + p.off_wd);
    uint32_t* wi = reinterpret_cast<uint32_t*>(base + p.off_wi);
    uint32_t* ws = reinterpret_cast<uint32_t*>(base + p.off_ws);
    const uint64_t n_total = p.n_points + p.n_start;
    const uint32_t cap = p.cap;

    for (uint32_t q; next_query(p.counters, p.n_work, p.work, lane, q);) {
        const PagedQuery st = p.qs[q];
        uint32_t* ctr = p.ctr + (size_t)q * C_WORDS;
        const uint32_t hlimit = st.n_buckets * 7;  // 87.5 % load

        __syncwarp();
        src.load(q);
        uint32_t size = 0, cursor = 0, tlen = 0, logn = 0, cmps = 0, hops = 0, seq = 0;
        if (p.begin) {
            for (uint32_t i = lane; i < st.n_buckets; i += 32) store_empty_bucket(st.table + (size_t)i * 8);
        } else {
            size = ctr[C_SIZE], cursor = ctr[C_CURSOR], tlen = ctr[C_TAIL], logn = ctr[C_LOG];
            cmps = ctr[C_CMPS], hops = ctr[C_HOPS], seq = ctr[C_SEQ];
            const size_t wo = (size_t)q * cap;
            for (uint32_t i = lane; i < size; i += 32) {
                wd[i] = p.wd[wo + i];
                wi[i] = p.wi[wo + i];
                ws[i] = p.ws[wo + i];
            }
        }
        __syncwarp();
        src.prepare();

        // HashSet::insert of one id per lane; the new ones are logged in lane order
        auto visit = [&](uint32_t id, bool ok) -> bool {
            const bool ins = ok && visit_global(st.table, st.n_buckets, id);
            const unsigned m = __ballot_sync(kFull, ins);
            if (ins) st.log[logn + __popc(m & ((1u << lane) - 1u))] = id;
            logn += __popc(m);
            return ins;
        };

        // expand_beam of one node (provider.rs:436-479): the neighbours that enter the visited set and are in bounds,
        // in adjacency order, into cid[0..)
        auto expand = [&](uint32_t node) -> uint32_t {
            const uint32_t* row = p.adj + (size_t)node * p.adj_stride;
            const uint32_t deg = min(__ldg(row), p.max_degree);
            uint32_t ncand = 0;
            for (uint32_t c0 = 0; c0 <= deg; c0 += 32) {
                const uint32_t jj = c0 + lane;
                const uint32_t word = jj < p.adj_stride ? __ldg(row + jj) : kEmptyV2;
                const bool isnew = visit(word, jj >= 1 && jj <= deg) && word < n_total;  // is_in_bounds after the insert
                push_new(isnew, word, cid, ncand, lane);
            }
            __syncwarp();
            return ncand;
        };

        auto distances = [&](uint32_t n) { src.distances(cid, cd, n); };

        auto merge = [&](uint32_t n) {
            for (uint32_t c0 = 0; c0 < n; c0 += 32)
                merge_paged(wd, wi, ws, cap, size, cursor, seq, st, tlen, cid, cd, c0, min(32u, n - c0), lane);
        };

        bool overflow = false;
        if (p.begin) {
            // paged_search_with_init_ids (index.rs:2108-2153): visited = the start ids, then one expand_beam over them;
            // the start points themselves are not queued and nothing is counted
            if (p.n_start > hlimit) overflow = true;
            for (uint32_t s0 = 0; s0 < p.n_start && !overflow; s0 += 32) visit((uint32_t)p.n_points + s0 + lane, s0 + lane < p.n_start);
            for (uint32_t s = 0; s < p.n_start && !overflow; ++s) {
                if (logn + p.max_degree > hlimit) {
                    overflow = true;
                    break;
                }
                const uint32_t n = expand((uint32_t)p.n_points + s);
                distances(n);
                merge(n);
            }
        } else {
            // search_internal with beam width 1 (index.rs:1961-1992), resumed.  After a page the cursor is 0 and
            // closest_notvisited (queue.rs:297-313) hands out entry 0 although it is visited: the first hop re-expands it
            for (;;) {
                const uint32_t lim = min(cap, size);
                if (cursor >= lim) break;
                if (logn + p.max_degree > hlimit) {  // the next node could pass the load limit: stop now
                    overflow = true;
                    break;
                }
                const uint32_t cur = cursor;
                const uint32_t node = wi[cur] & ~kFlagV2;
                __syncwarp();
                if (lane == 0) wi[cur] = node | kFlagV2;
                __syncwarp();
                cursor = first_unvisited(wi, cur + 1, lim, lane);
                const uint32_t n = expand(node);
                distances(n);
                merge(n);
                cmps += n;
                hops += 1;
            }
        }

        if (overflow) {
            report_overflow(p.counters, p.overflow_list, q, lane);
            continue;
        }

        if (!p.begin) {
            // the page: the first k entries of best.iter() (no start point is ever queued: they are visited from the
            // start), then drain_best (queue.rs:174-180) and the window refilled from the front of the tail
            const uint32_t cnt = min(p.k, size);
            for (uint32_t i = lane; i < p.k; i += 32) {
                p.out_ids[(size_t)q * p.k + i] = i < cnt ? (wi[i] & ~kFlagV2) : kEmptyV2;
                p.out_dists[(size_t)q * p.k + i] = i < cnt ? wd[i] : __int_as_float(0x7F800000);
            }
            for (uint32_t c0 = cnt; c0 < size; c0 += 32) {
                const uint32_t i = c0 + lane;
                float d = 0.0f;
                uint32_t id = 0, sq = 0;
                if (i < size) d = wd[i], id = wi[i], sq = ws[i];
                __syncwarp();
                if (i < size) wd[i - cnt] = d, wi[i - cnt] = id, ws[i - cnt] = sq;
                __syncwarp();
            }
            size -= cnt;
            for (uint32_t r = 0; r < cnt && tlen > 0; ++r) {
                uint64_t best = ~0ull;
                uint32_t at = 0;
                for (uint32_t i = lane; i < tlen; i += 32) {
                    const uint64_t key = order_key(st.td[i], st.ts[i]);
                    if (key < best) best = key, at = i;
                }
#pragma unroll
                for (int o = 16; o >= 1; o >>= 1) {
                    const uint64_t ob = __shfl_xor_sync(kFull, best, o);
                    const uint32_t oa = __shfl_xor_sync(kFull, at, o);
                    if (ob < best) best = ob, at = oa;
                }
                if (lane == 0) {
                    wd[size] = st.td[at], wi[size] = st.ti[at], ws[size] = st.ts[at];
                    const uint32_t last = tlen - 1;
                    st.td[at] = st.td[last], st.ti[at] = st.ti[last], st.ts[at] = st.ts[last];
                }
                ++size;
                --tlen;
                __syncwarp();
            }
            cursor = 0;
            if (lane == 0) {
                if (p.out_counts) p.out_counts[q] = cnt;
                if (p.out_cmps) p.out_cmps[q] = cmps;
                if (p.out_hops) p.out_hops[q] = hops;
            }
        }

        // commit
        __syncwarp();
        const size_t wo = (size_t)q * cap;
        for (uint32_t i = lane; i < size; i += 32) {
            p.wd[wo + i] = wd[i];
            p.wi[wo + i] = wi[i];
            p.ws[wo + i] = ws[i];
        }
        if (lane == 0) {
            ctr[C_SIZE] = size, ctr[C_CURSOR] = cursor, ctr[C_TAIL] = tlen, ctr[C_LOG] = logn;
            ctr[C_CMPS] = cmps, ctr[C_HOPS] = hops, ctr[C_SEQ] = seq;
        }
    }
}


template <typename TD, int KIND, int POST, int NA>
__global__ void __launch_bounds__(kPagedWarps * 32) paged_kernel(const PagedParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    uint8_t* base = smem + (size_t)wib * p.warp_smem;
    FullRowSource<TD, KIND, POST, NA, PagedParams> src(p, base, lane);
    paged_queries(p, base, lane, src);
}

template <int MODE>
__global__ void __launch_bounds__(kPagedWarps * 32) paged_kernel_quant(const PagedParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    uint8_t* base = smem + (size_t)wib * p.warp_smem;
    StoreSource<MODE, PagedParams> src(p, base, lane, blockIdx.x * kPagedWarps + wib);
    paged_queries(p, base, lane, src);
}

// Moves each listed query to the larger storage fresh[i]: the log and the tail up to their committed lengths are copied
// and the new table is rebuilt from the log.  One warp per query.
__global__ void __launch_bounds__(kPagedWarps * 32) paged_relocate_kernel(PagedQuery* qs, const uint32_t* ctr, const uint32_t* list,
                                                                          uint32_t n, const PagedQuery* fresh) {
    const int lane = threadIdx.x & 31;
    for (uint32_t w = blockIdx.x * kPagedWarps + (threadIdx.x >> 5); w < n; w += gridDim.x * kPagedWarps) {
        const uint32_t q = list[w];
        const PagedQuery a = qs[q], b = fresh[w];
        const uint32_t logn = ctr[(size_t)q * C_WORDS + C_LOG], tlen = ctr[(size_t)q * C_WORDS + C_TAIL];
        for (uint32_t i = lane; i < b.n_buckets; i += 32) store_empty_bucket(b.table + (size_t)i * 8);
        __syncwarp();
        for (uint32_t i = lane; i < tlen; i += 32) b.td[i] = a.td[i], b.ti[i] = a.ti[i], b.ts[i] = a.ts[i];
        for (uint32_t i0 = 0; i0 < logn; i0 += 32) {
            const uint32_t i = i0 + lane;
            if (i < logn) {
                const uint32_t id = a.log[i];
                b.log[i] = id;
                visit_global(b.table, b.n_buckets, id);
            }
        }
        __syncwarp();
        if (lane == 0) qs[q] = b;
    }
}

template <typename S>
void (*paged_kernel_of())(const PagedParams) {
    return paged_kernel<typename S::TD, S::KIND, S::POST, S::NA>;
}

}  // namespace

}  // namespace dab

using namespace dab;

// One session: the queries, every query's window, counters and visited storage, and the result buffers of a page.
struct dab_paged {
    dab_index* idx = nullptr;
    uint64_t generation = 0;
    dab_paged *prev = nullptr, *next = nullptr;  // the index's open sessions
    uint32_t nq = 0, l_search = 0, cap = 0;
    int store = -1;           // -1: full precision; else the QuantStore the traversal reads
    uint64_t store_writes = 0;  // idx->store_writes[store] when the session began
    PagedParams p{};
    WarpPlan<PagedParams> plan;
    void* d_queries = nullptr;
    float* d_wd = nullptr;
    uint32_t *d_wi = nullptr, *d_ws = nullptr, *d_ctr = nullptr;
    PagedQuery* d_qs = nullptr;
    PagedQuery* d_fresh = nullptr;  // the new storage of a pass's overflowed queries
    uint32_t* d_counters = nullptr;  // [0] work taken, [1] overflowed; then the overflow list [nq]
    uint32_t* d_list = nullptr;      // work list of a re-run [nq]
    uint32_t* d_out = nullptr;       // ids [nq][L], dists [nq][L], counts, cmps, hops [nq]
    uint8_t* d_qcodes = nullptr;     // SQ / MinMax: the compressed queries, codes [nq][stride] then one float4 each
    float* d_luts = nullptr;         // PQ tables: one table per warp of the grid, rebuilt at every call
    std::vector<uint64_t> slots;     // every query's table size
    std::vector<void*> chunks;       // visited storage (the first for every query, then one per growth)
};

namespace dab {
namespace {

size_t query_bytes(uint64_t slots) {
    const uint64_t nbk = (slots + 7) / 8, tcap = nbk * 7;
    return nbk * 32 + tcap * 16;  // table, log, tail (distance, id, insertion number)
}

PagedQuery carve(uint8_t*& at, uint64_t slots) {
    PagedQuery s;
    s.n_buckets = (uint32_t)((slots + 7) / 8);
    s.tcap = s.n_buckets * 7;
    s.table = (uint32_t*)at;
    at += (size_t)s.n_buckets * 32;
    s.log = (uint32_t*)at;
    at += (size_t)s.tcap * 4;
    s.td = (float*)at;
    at += (size_t)s.tcap * 4;
    s.ti = (uint32_t*)at;
    at += (size_t)s.tcap * 4;
    s.ts = (uint32_t*)at;
    at += (size_t)s.tcap * 4;
    return s;
}

void session_free(dab_paged* s) {
    cudaFree(s->d_queries);
    cudaFree(s->d_wd);
    cudaFree(s->d_wi);
    cudaFree(s->d_ws);
    cudaFree(s->d_ctr);
    cudaFree(s->d_qs);
    cudaFree(s->d_fresh);
    cudaFree(s->d_counters);
    cudaFree(s->d_list);
    cudaFree(s->d_out);
    cudaFree(s->d_qcodes);
    cudaFree(s->d_luts);
    for (void* c : s->chunks) cudaFree(c);
    delete s;
}

void unlink(dab_paged* s) {
    if (s->prev) s->prev->next = s->next;
    else s->idx->paged = s->next;
    if (s->next) s->next->prev = s->prev;
}

// Runs the session's kernel over every query (begin or one page), re-running on larger tables the queries that
// overflowed, until every query has committed.
int run_pass(dab_paged* s) {
    dab_index* idx = s->idx;
    cudaStream_t st = idx->stream;
    PagedParams p = s->p;
    p.work = nullptr;
    p.n_work = s->nq;
    std::vector<uint32_t> over;
    std::vector<PagedQuery> fresh;
    for (int pass = 0;;) {
        DAB_CUDA(cudaMemsetAsync(s->d_counters, 0, 8, st));
        int rc;
        if ((rc = warp_launch(p, s->plan, s->plan.pass_grid(p.n_work), st))) return rc;
        uint32_t n_over = 0;
        DAB_CUDA(cudaMemcpyAsync(&n_over, s->d_counters + 1, 4, cudaMemcpyDeviceToHost, st));
        DAB_CUDA(cudaStreamSynchronize(st));
        if (n_over == 0) return DAB_OK;
        over.resize(n_over);
        DAB_CUDA(cudaMemcpyAsync(over.data(), s->d_counters + 2, (size_t)n_over * 4, cudaMemcpyDeviceToHost, st));
        DAB_CUDA(cudaStreamSynchronize(st));
        // a table four times larger for each (grow_visited_tables), carved from one new allocation
        int next_pass = pass;
        size_t bytes = 0;
        for (uint32_t q : over) {
            int pq = pass;
            if ((rc = grow_visited_tables(idx, pq, s->slots[q]))) return rc;
            next_pass = pq;
            bytes += query_bytes(s->slots[q]);
        }
        pass = next_pass;
        void* chunk = nullptr;
        DAB_CUDA(cudaMalloc(&chunk, bytes));
        s->chunks.push_back(chunk);
        uint8_t* at = (uint8_t*)chunk;
        fresh.resize(n_over);
        for (uint32_t i = 0; i < n_over; ++i) fresh[i] = carve(at, s->slots[over[i]]);
        DAB_CUDA(cudaMemcpyAsync(s->d_fresh, fresh.data(), (size_t)n_over * sizeof(PagedQuery), cudaMemcpyHostToDevice, st));
        DAB_CUDA(cudaMemcpyAsync(s->d_list, over.data(), (size_t)n_over * 4, cudaMemcpyHostToDevice, st));
        const int rgrid = (int)std::min<uint64_t>((n_over + kPagedWarps - 1) / kPagedWarps, (uint64_t)idx->sm_count * 8);
        paged_relocate_kernel<<<rgrid, kPagedWarps * 32, 0, st>>>(s->d_qs, s->d_ctr, s->d_list, n_over, s->d_fresh);
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
        p.work = s->d_list;
        p.n_work = n_over;
    }
}

const char* begin_name(int store) {
    return store == STORE_PQ ? "dab_paged_search_begin_pq" : store == STORE_SQ ? "dab_paged_search_begin_sq"
           : store == STORE_MINMAX ? "dab_paged_search_begin_minmax" : "dab_paged_search_begin";
}

// the session's kernel, the shared memory of a warp — the query area (query_area_bytes), the candidates, the window — and
// the grid
int plan_kernel(dab_paged* s) {
    const dab_index* idx = s->idx;
    PagedParams& p = s->p;
    int rc;
    if ((rc = traversal_kernel(idx, s->store, [](auto m) { return paged_kernel_quant<decltype(m)::value>; },
                               [](auto sc) { return paged_kernel_of<decltype(sc)>(); }, s->plan.kern)))
        return rc;
    size_t off = query_area_bytes(idx, s->store);
    const size_t ncand = round_up(std::max<size_t>(idx->max_degree, 1) * 4, 16), win = round_up((size_t)s->cap * 4, 16);
    p.off_cid = (uint32_t)off, off += ncand;
    p.off_cd = (uint32_t)off, off += ncand;
    p.off_wd = (uint32_t)off, off += win;
    p.off_wi = (uint32_t)off, off += win;
    p.off_ws = (uint32_t)off, off += win;
    p.warp_smem = (uint32_t)round_up(off, 128);
    if (!plan_warps(idx, s->store, kPagedWarps, p.warp_smem, 200 * 1024, s->plan))
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: L=%u, dim=%u need %zu B shared memory per CTA", begin_name(s->store), s->l_search, idx->dim,
                    s->plan.smem_block);
    return DAB_OK;
}

// SQ and MinMax: the session's queries compressed by the store's quantizer into session memory (staged through the
// index's staging scratch, which other calls reuse between pages).  A MinMax query holding a NaN after the transform
// fails, naming the query.
int stage_session_queries(dab_paged* s) {
    dab_index* idx = s->idx;
    cudaStream_t st = idx->stream;
    const CodeStore& cs = s->store == STORE_SQ ? idx->sq : idx->mm;
    int rc;
    uint32_t* h_counters = nullptr;
    if (s->store == STORE_MINMAX) {
        if ((rc = idx->h_counters.reserve(24))) return rc;
        h_counters = (uint32_t*)idx->h_counters.p;
    }
    StagedQueries q{};
    if ((rc = stage_store_queries(idx, st, idx->s_stage, s->store, s->d_queries, s->nq, h_counters, q))) return rc;
    const size_t cbytes = (size_t)s->nq * cs.stride;
    DAB_CUDA(cudaMalloc(&s->d_qcodes, cbytes + (size_t)s->nq * 16));
    DAB_CUDA(cudaMemcpyAsync(s->d_qcodes, q.codes, cbytes, cudaMemcpyDeviceToDevice, st));
    DAB_CUDA(cudaMemcpyAsync(s->d_qcodes + cbytes, q.meta, (size_t)s->nq * 16, cudaMemcpyDeviceToDevice, st));
    DAB_CUDA(cudaStreamSynchronize(st));
    const unsigned long long nan = h_counters ? staged_first_nan(h_counters) : ~0ull;
    if (nan != ~0ull) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: query %llu contains NaN after the transform (InputContainsNaN)", begin_name(s->store), nan);
    s->p.store.query_codes = s->d_qcodes;
    s->p.store.query_meta = (const float4*)(s->d_qcodes + cbytes);
    return DAB_OK;
}

int begin_session(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search, int store, dab_paged* s) {
    s->idx = idx;
    s->generation = idx->generation;
    s->store = store;
    if (store >= 0) s->store_writes = idx->store_writes[store];
    s->nq = nq;
    s->l_search = l_search;
    s->cap = l_search + idx->n_start;  // PriorityQueueConfiguration::Resizable(L + #start)
    if (store >= 0) set_store_params(idx, (QuantStore)store, s->p.store);
    int rc;
    if ((rc = plan_kernel(s))) return rc;
    const size_t qbytes = (size_t)nq * idx->dim * elem_size(idx->dtype), wbytes = (size_t)nq * s->cap * 4;
    const size_t n1 = std::max<uint32_t>(nq, 1);
    DAB_CUDA(cudaMalloc(&s->d_queries, std::max<size_t>(qbytes, 16)));
    DAB_CUDA(cudaMalloc(&s->d_wd, std::max<size_t>(wbytes, 16)));
    DAB_CUDA(cudaMalloc(&s->d_wi, std::max<size_t>(wbytes, 16)));
    DAB_CUDA(cudaMalloc(&s->d_ws, std::max<size_t>(wbytes, 16)));
    DAB_CUDA(cudaMalloc(&s->d_ctr, n1 * C_WORDS * 4));
    DAB_CUDA(cudaMalloc(&s->d_qs, n1 * sizeof(PagedQuery)));
    DAB_CUDA(cudaMalloc(&s->d_fresh, n1 * sizeof(PagedQuery)));
    DAB_CUDA(cudaMalloc(&s->d_counters, 8 + n1 * 4));
    DAB_CUDA(cudaMalloc(&s->d_list, n1 * 4));
    DAB_CUDA(cudaMalloc(&s->d_out, n1 * ((size_t)l_search * 8 + 12)));
    if (nq == 0) return DAB_OK;
    // the reference's estimate of a search's visited set (or DAB_TEST_VISITED_LOG2), at least what the start points
    // and one expansion need; a query that outgrows it gets a larger table
    // (no hint is consulted, so it does not matter which store's the estimate is asked for)
    const uint64_t slots = std::max<uint64_t>(table_slots(idx, VisitedHint{}, l_search, 1, STORE_PQ),
                                              idx->tune.test_visited_log2 ? 0 : ((uint64_t)idx->n_start + idx->max_degree) * 8 / 7 + 64);
    s->slots.assign(nq, slots);
    void* chunk = nullptr;
    DAB_CUDA(cudaMalloc(&chunk, query_bytes(slots) * nq));
    s->chunks.push_back(chunk);
    std::vector<PagedQuery> qs(nq);
    uint8_t* at = (uint8_t*)chunk;
    for (uint32_t q = 0; q < nq; ++q) qs[q] = carve(at, slots);
    cudaStream_t st = idx->stream;
    DAB_CUDA(cudaMemcpyAsync(s->d_qs, qs.data(), (size_t)nq * sizeof(PagedQuery), cudaMemcpyHostToDevice, st));
    DAB_CUDA(cudaMemcpyAsync(s->d_queries, queries, qbytes, cudaMemcpyHostToDevice, st));
    DAB_CUDA(cudaMemsetAsync(s->d_ctr, 0, (size_t)nq * C_WORDS * 4, st));
    if (store == STORE_SQ || store == STORE_MINMAX) {
        if ((rc = stage_session_queries(s))) return rc;
        cudaFree(s->d_queries);  // the kernel reads the compressed queries only
        s->d_queries = nullptr;
    }
    if (const size_t tables = pq_table_bytes(idx, store, (uint64_t)s->plan.grid * s->plan.warps)) {
        DAB_CUDA(cudaMalloc(&s->d_luts, tables));
        s->p.store.luts = s->d_luts;
    }

    PagedParams& p = s->p;
    p.vectors = idx->d_vectors;
    p.row_stride = idx->row_stride;
    set_graph_params(idx, p);
    p.queries = s->d_queries;
    p.counters = s->d_counters;
    p.overflow_list = s->d_counters + 2;
    p.cap = s->cap;
    p.qs = s->d_qs;
    p.wd = s->d_wd, p.wi = s->d_wi, p.ws = s->d_ws, p.ctr = s->d_ctr;
    p.begin = 1;
    p.k = 0;
    rc = run_pass(s);
    p.begin = 0;
    return rc;
}

}  // namespace

void paged_release(dab_index* idx) {
    while (idx->paged) {
        dab_paged* s = (dab_paged*)idx->paged;
        unlink(s);
        session_free(s);
    }
}

namespace {

// dab_paged_search_begin and its quantized forms (store: -1 full precision, else the QuantStore the traversal reads)
int paged_begin(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search, int store, dab_paged** out) {
    const char* who = begin_name(store);
    if (!idx || !out || (nq && !queries)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL argument", who);
    *out = nullptr;
    int rc;
    if ((rc = check_search_args(idx, 1, l_search, 1, store < 0)) || (store >= 0 && (rc = check_quant_store(idx, (QuantStore)store, who, true)))) return rc;
    if ((uint64_t)l_search + idx->n_start > 1024)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: l_search + n_start = %llu > 1024", who, (unsigned long long)l_search + idx->n_start);
    DAB_CUDA(cudaSetDevice(idx->device));
    dab_paged* s = new dab_paged();
    if ((rc = begin_session(idx, queries, nq, l_search, store, s))) {
        cudaStreamSynchronize(idx->stream);
        session_free(s);
        return rc;
    }
    s->next = (dab_paged*)idx->paged;
    if (s->next) s->next->prev = s;
    idx->paged = s;
    *out = s;
    return DAB_OK;
}

}  // namespace

}  // namespace dab

extern "C" {

int dab_paged_search_begin(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search, dab_paged** out) {
    return paged_begin(idx, queries, nq, l_search, -1, out);
}

int dab_paged_search_begin_pq(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search, dab_paged** out) {
    return paged_begin(idx, queries, nq, l_search, STORE_PQ, out);
}

int dab_paged_search_begin_sq(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search, dab_paged** out) {
    return paged_begin(idx, queries, nq, l_search, STORE_SQ, out);
}

int dab_paged_search_begin_minmax(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search, dab_paged** out) {
    return paged_begin(idx, queries, nq, l_search, STORE_MINMAX, out);
}

int dab_paged_search_next(dab_paged* s, uint32_t k, uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps,
                          uint32_t* out_hops) {
    if (!s) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_paged_search_next: session is NULL");
    if (s->nq && (!out_ids || !out_dists)) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_paged_search_next: NULL argument");
    // PagedSearch::next_page (paged.rs:62-69): the bound is L itself, not L + #start
    if (k == 0) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_paged_search_next: k should be greater than 0");
    if (k > s->l_search)
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_paged_search_next: k should be less than or equal to search_param_l (k = %u, L = %u)", k,
                    s->l_search);
    dab_index* idx = s->idx;
    if (s->generation != idx->generation)
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_paged_search_next: index changed since the session began");
    if (s->store >= 0 && s->store_writes != idx->store_writes[s->store])
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_paged_search_next: the session's quantized store was written since the session began");
    if (s->nq == 0) return DAB_OK;
    DAB_CUDA(cudaSetDevice(idx->device));
    const size_t nq = s->nq, rk = nq * k;
    uint32_t* ids = s->d_out;
    float* dists = (float*)(ids + rk);
    uint32_t* stats = (uint32_t*)(dists + rk);
    s->p.k = k;
    s->p.out_ids = ids, s->p.out_dists = dists;
    s->p.out_counts = stats, s->p.out_cmps = stats + nq, s->p.out_hops = stats + 2 * nq;
    int rc;
    if ((rc = run_pass(s))) return rc;
    cudaStream_t st = idx->stream;
    DAB_CUDA(cudaMemcpyAsync(out_ids, ids, rk * 4, cudaMemcpyDeviceToHost, st));
    DAB_CUDA(cudaMemcpyAsync(out_dists, dists, rk * 4, cudaMemcpyDeviceToHost, st));
    if (out_counts) DAB_CUDA(cudaMemcpyAsync(out_counts, stats, nq * 4, cudaMemcpyDeviceToHost, st));
    if (out_cmps) DAB_CUDA(cudaMemcpyAsync(out_cmps, stats + nq, nq * 4, cudaMemcpyDeviceToHost, st));
    if (out_hops) DAB_CUDA(cudaMemcpyAsync(out_hops, stats + 2 * nq, nq * 4, cudaMemcpyDeviceToHost, st));
    DAB_CUDA(cudaStreamSynchronize(st));
    return DAB_OK;
}

void dab_paged_search_end(dab_paged* s) {
    if (!s) return;
    cudaSetDevice(s->idx->device);
    cudaStreamSynchronize(s->idx->stream);
    unlink(s);
    session_free(s);
}

}  // extern "C"
