// search_diverse.cu — diversity-aware batched search on the device: Diverse::search (diskann/src/graph/search/
// diverse_search.rs:189-234), i.e. search_internal (diskann/src/graph/index.rs:1933-2000) with the list a
// DiverseNeighborQueue (diskann/src/neighbor/diverse_priority_queue.rs:90-220), then its post_process and the default
// post-processing of the first L entries; and the attribute table it reads (dab_upload_attributes).
//
// One warp per query on global visited tables, over full-precision rows of every type and metric of the k-NN path
// (diverse_kernel) or the PQ, SQ and MinMax stores with the distances of their k-NN traversal and an optional
// full-precision rerank of the post-processed list (diverse_kernel_quant).  The warp keeps, per query:
//   the global list   L entries sorted as a NeighborPriorityQueue sorts them (distance ascending, a later insertion
//                     first among equal distances), each with its id | visited flag and its attribute, in shared memory;
//                     the cursor is the reference's plain index (after a removal at the cursor it may point at a visited
//                     entry, which closest_notvisited then hands out again);
//   the local queues  one pool of entries {attribute, distance, id, insertion number} in global memory: a local queue
//                     is the pool's entries of one attribute, and its order follows from (distance ascending, insertion
//                     number descending) without being stored.
// Candidates enter one at a time in expand_beam order with the three cases of DiverseNeighborQueue::insert; every
// NeighborPriorityQueue::remove looks only at the lower bound of the distance, so a removal that meets another entry
// of equal distance fails as it does in the reference and the local queues drift from the list the same way.  The pool
// holds at most L entries while no removal fails; a query whose entries outgrow the pool stops, is counted in
// counters[3] and is re-run by the job on a pool four times larger (at most n_total entries, which never overflow), so
// no query is ever answered from a truncated pool.  A query that outgrew its visited table instead gets a larger table.
#include "dab_common.cuh"
#include "search_common.cuh"
#include "search_diverse.cuh"

#include <algorithm>

namespace dab {

namespace {

// ---- the global list --------------------------------------------------------------------------------------------
// the first entry whose distance is >= d (queue.rs:229-280): the list is sorted and holds no NaN
__device__ __forceinline__ uint32_t list_lower_bound(const float* gd, uint32_t size, float d, int lane) {
    uint32_t n = 0;
    for (uint32_t b = 0; b < size; b += 32) {
        const uint32_t i = b + lane;
        const unsigned m = __ballot_sync(kFull, i < size && gd[i] < d);
        n += __popc(m);
        if (m != kFull) break;
    }
    return n;
}

// entries [from, to) move to [from + 1, to + 1), the top tile first
__device__ __forceinline__ void list_shift_up(float* gd, uint32_t* gi, uint32_t* ga, uint32_t from, uint32_t to, int lane) {
    if (to <= from) return;
    for (uint32_t t = (to - from - 1) / 32 + 1; t-- > 0;) {
        const uint32_t i = from + t * 32 + lane;
        float d = 0.0f;
        uint32_t id = 0, a = 0;
        if (i < to) d = gd[i], id = gi[i], a = ga[i];
        __syncwarp();
        if (i < to) gd[i + 1] = d, gi[i + 1] = id, ga[i + 1] = a;
        __syncwarp();
    }
}

// entries [from + 1, to) move to [from, to - 1), the bottom tile first
__device__ __forceinline__ void list_shift_down(float* gd, uint32_t* gi, uint32_t* ga, uint32_t from, uint32_t to, int lane) {
    for (uint32_t b = from + 1; b < to; b += 32) {
        const uint32_t i = b + lane;
        float d = 0.0f;
        uint32_t id = 0, a = 0;
        if (i < to) d = gd[i], id = gi[i], a = ga[i];
        __syncwarp();
        if (i < to) gd[i - 1] = d, gi[i - 1] = id, ga[i - 1] = a;
        __syncwarp();
    }
}

// NeighborPriorityQueue::insert, fixed capacity cap (queue.rs:130-171); d is not NaN
__device__ __forceinline__ void list_insert(float* gd, uint32_t* gi, uint32_t* ga, uint32_t cap, uint32_t& size, uint32_t& cursor, float d,
                                            uint32_t id, uint32_t a, int lane) {
    if (size == cap && gd[cap - 1] < d) return;
    const uint32_t at = list_lower_bound(gd, size, d, lane);
    const uint32_t end = size == cap ? cap - 1 : size;  // a full list drops its last entry
    list_shift_up(gd, gi, ga, at, end, lane);
    if (lane == 0) gd[at] = d, gi[at] = id, ga[at] = a;
    __syncwarp();
    size = end + 1;
    if (at < cursor) cursor = at;
}

// NeighborPriorityQueue::remove (queue.rs:197-224): only the entry at the lower bound of d is compared
__device__ __forceinline__ void list_remove(float* gd, uint32_t* gi, uint32_t* ga, uint32_t& size, uint32_t& cursor, float d, uint32_t id,
                                            int lane) {
    if (size == 0) return;
    const uint32_t at = list_lower_bound(gd, size, d, lane);
    if (at >= size || (gi[at] & ~kFlagV2) != id) return;
    list_shift_down(gd, gi, ga, at, size, lane);
    --size;
    if (at < cursor && cursor > 0) --cursor;
}

// ---- the local queues: one pool of entries in global memory -----------------------------------------------------
struct Pool {
    uint32_t* attr;
    float* dist;
    uint32_t* id;
    uint32_t* seq;
    uint32_t cap;
};

// x comes after y in a local queue: a larger distance, or an equal one inserted earlier
__device__ __forceinline__ bool after(float dx, uint32_t sx, float dy, uint32_t sy) { return dx > dy || (dx == dy && sx < sy); }

// one entry of a warp-wide search: its pool index (none: UINT32_MAX), distance, insertion number
struct Pick {
    uint32_t at;
    float d;
    uint32_t s;
};

// the warp's Pick that `better` prefers, on every lane
template <class Better>
__device__ __forceinline__ Pick warp_pick(Pick p, Better better) {
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
        Pick q;
        q.at = __shfl_xor_sync(kFull, p.at, o);
        q.d = __shfl_xor_sync(kFull, p.d, o);
        q.s = __shfl_xor_sync(kFull, p.s, o);
        if (q.at != kEmptyV2 && (p.at == kEmptyV2 || better(q, p))) p = q;
    }
    return p;
}

// the size of attribute a's local queue and its last entry
__device__ __forceinline__ Pick local_last(const Pool& pl, uint32_t psize, uint32_t a, uint32_t& count, int lane) {
    Pick w{kEmptyV2, 0.0f, 0};
    uint32_t n = 0;
    for (uint32_t i = lane; i < psize; i += 32) {
        if (pl.attr[i] != a) continue;
        ++n;
        const float d = pl.dist[i];
        const uint32_t s = pl.seq[i];
        if (w.at == kEmptyV2 || after(d, s, w.d, w.s)) w = Pick{i, d, s};
    }
    count = __reduce_add_sync(kFull, n);
    return warp_pick(w, [](const Pick& x, const Pick& y) { return after(x.d, x.s, y.d, y.s); });
}

// NeighborPriorityQueue::remove of (id, d) from attribute a's local queue: the first of its entries whose distance is
// >= d goes if it is `id`
__device__ __forceinline__ void local_remove(const Pool& pl, uint32_t& psize, uint32_t a, uint32_t id, float d, int lane) {
    Pick f{kEmptyV2, 0.0f, 0};
    for (uint32_t i = lane; i < psize; i += 32) {
        if (pl.attr[i] != a) continue;
        const float di = pl.dist[i];
        if (!(di >= d)) continue;
        const uint32_t s = pl.seq[i];
        if (f.at == kEmptyV2 || after(f.d, f.s, di, s)) f = Pick{i, di, s};
    }
    f = warp_pick(f, [](const Pick& x, const Pick& y) { return after(y.d, y.s, x.d, x.s); });
    if (f.at == kEmptyV2 || pl.id[f.at] != id) return;
    // the pool's last entry fills the hole
    const uint32_t last = psize - 1;
    __syncwarp();
    if (lane == 0 && f.at != last) {
        pl.attr[f.at] = pl.attr[last], pl.dist[f.at] = pl.dist[last], pl.id[f.at] = pl.id[last], pl.seq[f.at] = pl.seq[last];
    }
    __syncwarp();
    psize = last;
}

__device__ __forceinline__ void pool_put(const Pool& pl, uint32_t at, uint32_t a, float d, uint32_t id, uint32_t s, int lane) {
    __syncwarp();
    if (lane == 0) pl.attr[at] = a, pl.dist[at] = d, pl.id[at] = id, pl.seq[at] = s;
    __syncwarp();
}

// The state of one query
struct DivQuery {
    float* gd;
    uint32_t *gi, *ga;
    uint32_t cap, size, cursor;
    Pool pool;
    uint32_t psize, seq;
    uint32_t local_cap;
};

// DiverseNeighborQueue::insert (diverse_priority_queue.rs:151-220) of one candidate; false when the pool is full
__device__ __forceinline__ bool diverse_insert(const SearchParamsDiverse& p, DivQuery& q, uint32_t id, float d, int lane) {
    if (d != d) return true;  // NaN enters neither queue
    if (!(__ldg(p.attr_present + (id >> 5)) >> (id & 31) & 1u)) return true;  // no attribute: skipped
    const uint32_t a = __ldg(p.attr_values + id);
    uint32_t lsize;
    const Pick worst = local_last(q.pool, q.psize, a, lsize, lane);
    const bool local_full = lsize == q.local_cap, global_full = q.size == q.cap;
    if (!local_full && !global_full) {
        // case 1: both have room
        if (q.psize == q.pool.cap) return false;
        pool_put(q.pool, q.psize++, a, d, id, q.seq++, lane);
        list_insert(q.gd, q.gi, q.ga, q.cap, q.size, q.cursor, d, id, a, lane);
    } else if (local_full) {
        // case 2: the local queue's last entry leaves both queues (the list only if it sits at its lower bound)
        if (!(d < worst.d)) return true;
        const uint32_t wid = q.pool.id[worst.at];
        list_remove(q.gd, q.gi, q.ga, q.size, q.cursor, worst.d, wid, lane);
        pool_put(q.pool, worst.at, a, d, id, q.seq++, lane);
        list_insert(q.gd, q.gi, q.ga, q.cap, q.size, q.cursor, d, id, a, lane);
    } else {
        // case 3: the list's last entry leaves it and then its own local queue
        const float gw = q.gd[q.cap - 1];
        if (!(d < gw)) return true;
        const uint32_t gw_id = q.gi[q.cap - 1] & ~kFlagV2, gw_a = q.ga[q.cap - 1];
        if (q.psize == q.pool.cap) return false;
        pool_put(q.pool, q.psize++, a, d, id, q.seq++, lane);
        list_insert(q.gd, q.gi, q.ga, q.cap, q.size, q.cursor, d, id, a, lane);
        local_remove(q.pool, q.psize, gw_a, gw_id, gw, lane);
    }
    return true;
}

// DiverseNeighborQueue::post_process (diverse_priority_queue.rs:112-138): the entries of each local queue past
// diverse_k are cut, and the list keeps, in order, the entries whose id was not cut (queue.rs:427-456)
__device__ __forceinline__ void diverse_post_process(const SearchParamsDiverse& p, DivQuery& q, int lane) {
    // the visited flags are cleared (retain resets them) and then mark the cut entries
    for (uint32_t i = lane; i < q.size; i += 32) q.gi[i] &= ~kFlagV2;
    __syncwarp();
    const Pool& pl = q.pool;
    for (uint32_t b = 0; b < q.psize; b += 32) {
        const uint32_t e = b + lane;
        const bool have = e < q.psize;
        const uint32_t a = have ? pl.attr[e] : 0, s = have ? pl.seq[e] : 0;
        const float d = have ? pl.dist[e] : 0.0f;
        uint32_t rank = 0;  // entries of the same local queue before this one
        for (uint32_t j = 0; j < q.psize; ++j) rank += pl.attr[j] == a && after(d, s, pl.dist[j], pl.seq[j]) ? 1u : 0u;
        const uint32_t cut_id = have ? pl.id[e] : kEmptyV2;
        for (unsigned m = __ballot_sync(kFull, have && rank >= p.diverse_k); m;) {
            const int l = __ffs(m) - 1;
            m &= m - 1;
            const uint32_t id = __shfl_sync(kFull, cut_id, l);
            for (uint32_t g = lane; g < q.size; g += 32)
                if (q.gi[g] == id) q.gi[g] = id | kFlagV2;
        }
    }
    __syncwarp();
    uint32_t w = 0;
    for (uint32_t b = 0; b < q.size; b += 32) {
        const uint32_t i = b + lane;
        const bool keep = i < q.size && !(q.gi[i] & kFlagV2);
        float d = 0.0f;
        uint32_t id = 0, a = 0;
        if (keep) d = q.gd[i], id = q.gi[i], a = q.ga[i];
        const unsigned mk = __ballot_sync(kFull, keep);
        __syncwarp();
        if (keep) {
            const uint32_t at = w + __popc(mk & ((1u << lane) - 1u));
            q.gd[at] = d, q.gi[at] = id, q.ga[at] = a;
        }
        w += __popc(mk);
        __syncwarp();
    }
    q.size = w;
}

// One warp's share of a pass: the diverse search of every query it takes, whatever the distances are.  Src is a
// distance source (search_source.cuh).  LIST: with p.list_ids, the post-processed list of each query is written for
// the rerank.
template <bool LIST, class Src>
__device__ __forceinline__ void diverse_queries(const SearchParamsDiverse& p, uint8_t* base, int lane, Src& src) {
    const int wib = threadIdx.x >> 5;
    uint32_t* cid = reinterpret_cast<uint32_t*>(base + p.off_cid);
    float* cd = reinterpret_cast<float*>(base + p.off_cd);
    uint32_t* beam_ids = reinterpret_cast<uint32_t*>(base + p.off_beam);
    const uint32_t warp_slot = blockIdx.x * kDivWarps + wib;
    const uint32_t nbk = p.n_buckets;
    uint32_t* table = p.tables + (size_t)warp_slot * nbk * 8;
    const uint32_t hlimit = nbk * 7;  // 87.5 % load
    const uint64_t n_total = p.n_points + p.n_start;
    uint32_t* pool = p.pools + (size_t)warp_slot * p.pool_cap * 4;

    auto distances = [&](uint32_t n) { src.distances(cid, cd, n); };

    for (uint32_t qidx; next_query(p.counters, p.n_work, p.query_list, lane, qidx);) {
        __syncwarp();
        src.load(qidx);
        for (uint32_t i = lane; i < nbk; i += 32) store_empty_bucket(table + (size_t)i * 8);
        __syncwarp();
        src.prepare();
        DivQuery q;
        q.gd = reinterpret_cast<float*>(base + p.off_gd);
        q.gi = reinterpret_cast<uint32_t*>(base + p.off_gi);
        q.ga = reinterpret_cast<uint32_t*>(base + p.off_ga);
        q.cap = p.cap, q.size = 0, q.cursor = 0;
        q.pool = Pool{pool, reinterpret_cast<float*>(pool + p.pool_cap), pool + 2 * (size_t)p.pool_cap, pool + 3 * (size_t)p.pool_cap, p.pool_cap};
        q.psize = 0, q.seq = 0;
        q.local_cap = p.local_cap;
        uint32_t cmps = 0, hops = 0, nvisited = 0;
        bool overflow = false, pool_full = false;  // the visited table or the local queues outgrew their storage

        auto insert_all = [&](uint32_t n) {
            for (uint32_t c = 0; c < n && !overflow; ++c) overflow = pool_full = !diverse_insert(p, q, cid[c], cd[c], lane);
        };

        // ---- start points (start_point_distances, provider.rs:406-433), in id order
        for (uint32_t s0 = 0; s0 < p.n_start && !overflow; s0 += 32) {
            const uint32_t n = min(32u, p.n_start - s0);
            if ((uint32_t)lane < n) {
                const uint32_t id = (uint32_t)p.n_points + s0 + lane;
                cid[lane] = id;
                visit_global(table, nbk, id);
            }
            __syncwarp();
            distances(n);
            insert_all(n);
            nvisited += n;
            cmps += n;
        }

        // ---- search_internal: closest_notvisited x beam, expand_beam, the candidates inserted in order
        while (!overflow && q.cursor < min(q.cap, q.size)) {
            uint32_t nb = 0;
            while (nb < p.beam && q.cursor < min(q.cap, q.size)) {
                const uint32_t cur = q.cursor;
                const uint32_t node = q.gi[cur] & ~kFlagV2;
                __syncwarp();
                if (lane == 0) {
                    q.gi[cur] = node | kFlagV2;
                    beam_ids[nb] = node;
                }
                __syncwarp();
                q.cursor = first_unvisited(q.gi, cur + 1, q.size, lane);
                ++nb;
            }
            uint32_t ncand = 0;
            for (uint32_t b = 0; b < nb; ++b) {
                const uint32_t node = beam_ids[b];
                const uint32_t* row = p.adj + (size_t)node * p.adj_stride;
                const uint32_t deg = min(__ldg(row), p.max_degree);
                for (uint32_t c0 = 0; c0 < deg + 1; c0 += 32) {
                    const uint32_t j = c0 + lane;
                    const uint32_t word = j < p.adj_stride ? __ldg(row + j) : kEmptyV2;
                    const bool inserted = j >= 1 && j <= deg && visit_global(table, nbk, word);
                    push_new(inserted, inserted && word < n_total, word, cid, ncand, nvisited, lane);
                }
                if (nvisited + p.max_degree > hlimit) {
                    overflow = true;
                    break;
                }
            }
            if (overflow) break;
            __syncwarp();
            distances(ncand);
            insert_all(ncand);
            cmps += ncand;
            hops += nb;
        }

        if (overflow) {
            report_overflow(p.counters, p.overflow_list, qidx, lane);
            if (pool_full && lane == 0) atomicAdd(p.counters + 3, 1u);  // the job grows the pool, not the tables
            continue;
        }
        diverse_post_process(p, q, lane);
        if constexpr (LIST) {
            if (p.list_ids) write_list(q.gi, q.size, p.list_ids, p.list_counts, p.list_cap, qidx, lane);
        }
        const uint32_t count = write_results(q.gi, q.gd, q.size, p.n_points, p.k, p.out_ids, p.out_dists, qidx, lane);
        write_stats(p.counters, nvisited, p.out_counts, p.out_cmps, p.out_hops, qidx, count, cmps, hops, lane);
    }
}

template <typename TD, int KIND, int POST, int NA>
__global__ void __launch_bounds__(kDivWarps * 32) diverse_kernel(const SearchParamsDiverse p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    uint8_t* base = smem + (size_t)wib * p.warp_smem;
    FullRowSource<TD, KIND, POST, NA, SearchParamsDiverse> src(p, base, lane);
    diverse_queries<false>(p, base, lane, src);
}

template <int MODE>
__global__ void __launch_bounds__(kDivWarps * 32) diverse_kernel_quant(const SearchParamsDiverse p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    uint8_t* base = smem + (size_t)wib * p.warp_smem;
    StoreSource<MODE, SearchParamsDiverse> src(p, base, lane, blockIdx.x * kDivWarps + wib);
    diverse_queries<true>(p, base, lane, src);
}

template <typename S>
void (*diverse_kernel_of())(const SearchParamsDiverse) {
    return diverse_kernel<typename S::TD, S::KIND, S::POST, S::NA>;
}

}  // namespace

// A warp's shared memory: the query area (query_area_bytes), the list's distances, ids and attributes, a hop's candidate
// ids and distances, the beam; `p` (may be NULL) takes the offsets.  `store`: -1 full precision, else a QuantStore.
static size_t diverse_warp_smem(const dab_index* idx, uint32_t l_search, uint32_t beam, int store, SearchParamsDiverse* p) {
    size_t off = query_area_bytes(idx, store);
    const size_t list = round_up((size_t)l_search * 4, 16);
    const size_t ncand = round_up(std::max<size_t>((size_t)beam * idx->max_degree, 32) * 4, 16);
    SearchParamsDiverse scratch;
    SearchParamsDiverse& q = p ? *p : scratch;
    q.off_gd = (uint32_t)off, off += list;
    q.off_gi = (uint32_t)off, off += list;
    q.off_ga = (uint32_t)off, off += list;
    q.off_cid = (uint32_t)off, off += ncand;
    q.off_cd = (uint32_t)off, off += ncand;
    q.off_beam = (uint32_t)off, off += round_up((size_t)beam * 4, 16);
    return round_up(off, 128);
}

int diverse_check_smem(const dab_index* idx, const char* api, uint32_t l_search, uint32_t beam, int store) {
    const size_t smem = diverse_warp_smem(idx, l_search, beam, store, nullptr) * kDivWarps;
    if (smem > kDiverseMaxSmem)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: L=%u, beam_width=%u, dim=%u, max_degree=%u need %zu B shared memory per CTA (> %zu)", api,
                    l_search, beam, idx->dim, idx->max_degree, smem, kDiverseMaxSmem);
    return DAB_OK;
}

int diverse_plan(const dab_index* idx, uint32_t l_search, uint32_t beam, int store, SearchParamsDiverse& p, WarpPlan<SearchParamsDiverse>& plan) {
    p.warp_smem = (uint32_t)diverse_warp_smem(idx, l_search, beam, store, &p);
    int rc;
    if ((rc = traversal_kernel(idx, store, [](auto m) { return diverse_kernel_quant<decltype(m)::value>; },
                               [](auto sc) { return diverse_kernel_of<decltype(sc)>(); }, plan.kern)))
        return rc;
    if (!plan_warps(idx, store, kDivWarps, p.warp_smem, kDiverseMaxSmem, plan))
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_search_batch_diverse: L=%u, beam_width=%u, dim=%u need %zu B shared memory per CTA",
                    l_search, beam, idx->dim, plan.smem_block);
    return DAB_OK;
}

// While no removal fails the pool holds what the list holds, at most L entries; 32 more absorb a few failed removals
uint64_t diverse_pool_first(const dab_index* idx, uint32_t l_search) {
    if (idx->tune.test_diverse_pool) return idx->tune.test_diverse_pool;  // tests force the overflow re-runs
    return round_up((size_t)l_search + 32, 32);
}

// the pool never needs more entries than there are ids: each id enters the local queues at most once
uint64_t diverse_pool_grow(const dab_index* idx, uint64_t pool) {
    return std::min<uint64_t>(pool * 4, round_up(idx->n_total(), 32));
}

// ---- the attribute table -----------------------------------------------------------------------------------------
void attributes_release(dab_index* idx) {
    cudaFree(idx->d_attr_values);
    cudaFree(idx->d_attr_present);
    delete[] idx->h_attr_present;
    idx->d_attr_values = nullptr;
    idx->d_attr_present = nullptr;
    idx->h_attr_present = nullptr;
}

}  // namespace dab

using namespace dab;

extern "C" {

int dab_upload_attributes(dab_index* idx, const uint32_t* values, const uint8_t* present, uint64_t first, uint64_t count) {
    if (!idx || (count && !values)) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_upload_attributes: NULL argument");
    if (first > idx->n_total() || count > idx->n_total() - first)
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_upload_attributes: ids [%llu, %llu) out of range (%llu ids)", (unsigned long long)first,
                    (unsigned long long)(first + count), (unsigned long long)idx->n_total());
    DAB_CUDA(cudaSetDevice(idx->device));
    const uint64_t words = idx->deleted_words();
    if (!idx->h_attr_present) {
        // the table is published only once both device arrays exist and are cleared
        DevBuf values, bits;
        int rc;
        if ((rc = values.alloc(idx->n_total() * 4, "dab_upload_attributes")) || (rc = bits.alloc(words * 4, "dab_upload_attributes")))
            return rc;
        DAB_CUDA(cudaMemsetAsync(values.p, 0, idx->n_total() * 4, idx->stream));
        DAB_CUDA(cudaMemsetAsync(bits.p, 0, words * 4, idx->stream));
        DAB_CUDA(cudaStreamSynchronize(idx->stream));
        idx->h_attr_present = new uint32_t[words]();
        idx->d_attr_values = (uint32_t*)values.p;
        idx->d_attr_present = (uint32_t*)bits.p;
        values.p = bits.p = nullptr;
    }
    if (count == 0) return DAB_OK;
    for (uint64_t i = 0; i < count; ++i) {
        const uint64_t id = first + i;
        const uint32_t bit = 1u << (id & 31);
        if (!present || present[i]) idx->h_attr_present[id >> 5] |= bit;
        else idx->h_attr_present[id >> 5] &= ~bit;
    }
    const uint64_t w0 = first >> 5, w1 = (first + count - 1) >> 5;
    DAB_CUDA(cudaMemcpyAsync(idx->d_attr_values + first, values, count * 4, cudaMemcpyHostToDevice, idx->stream));
    DAB_CUDA(cudaMemcpyAsync(idx->d_attr_present + w0, idx->h_attr_present + w0, (w1 - w0 + 1) * 4, cudaMemcpyHostToDevice, idx->stream));
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    return DAB_OK;
}

}  // extern "C"
