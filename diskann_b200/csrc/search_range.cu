// search_range.cu — batched range search on the device: Range::search and range_search_internal
// (diskann/src/graph/search/range_search.rs:255-469) over full-precision rows or the PQ, SQ and MinMax stores, the
// filtered range search's pass loop (FilteredRange::search, dab_range_search_filtered[_pq|_sq|_minmax][_device]; its
// kernels are in search_filtered.cu), and the result sets they return (dab_range_search[_pq|_sq|_minmax][_device],
// dab_range_offsets, dab_range_results[_device], dab_range_free).
//
// Phase 1 is the k-NN traversal at L through run_search (search_kernel_v3 / _v2 over full-precision rows,
// search_kernel_pq_starts over a store): with k = L and start points and deleted ids kept, it writes each query's first
// L list entries, its cmps and its hops.  Phase 2 is range_kernel (full precision) or range_kernel_quant (the store's
// distances, those of its k-NN traversal), one warp per query on global visited tables:
//   in_range  the phase-1 entries with distance <= radius, in list order, in the warp's region of global memory;
//   round 2   iff |in_range| >= (f32(L) * initial_slack) as usize and |in_range| < max_returned: the visited table is
//             cleared and re-seeded with the in_range ids, and the frontier, the unconsumed suffix of in_range, is
//             expanded beam_width ids at a time in expand_beam order; each new neighbour with d <= radius * range_slack
//             is appended while |in_range| < max_returned (the cap may cut a hop short);
//   output    in_range in insertion order without start points, deleted ids, ids with d <= inner_radius (when given)
//             and ids with d > radius.
// Every distance of both phases is the store's, so over a store the output compares the store's distances.  With
// rerank, the quantized strategies' Pipeline<FilterStartPoints, Rerank> (providers inmem/product.rs:391-401,
// full_precision.rs:356-399) runs instead over each query's in_range: start points and deleted ids dropped, every other
// id's full-precision Distance<T, T> to the query (range_rerank_kernel, the rerank_kernel schemas), the entries outside
// (inner_radius, radius] of that distance dropped, and the rest sorted by it, stably (ties in in_range order, -0.0 equal
// to +0.0; the reference's sort_unstable_by leaves ties unspecified, and NaN has been filtered out before the sort).
// The hops of a query that took the second round are phase1 + (phase1 + phase2), as the reference adds its cumulative
// scratch.hops to phase 1's; cmps are phase 1's.  A hop's nodes are expanded, scored and appended one node at a time:
// the visited inserts and the appends come in the reference's order, and nothing after the cap is observable.
//
// No query is answered from truncated storage.  A query whose visited set outgrows its table, or whose in_range
// outgrows its region, stops and is re-run: on tables from grow_visited_tables, or on regions four times larger (at
// most min(max_returned, n_total) entries, which in_range, of distinct ids, cannot outgrow).  A completed query claims
// space for its filtered results in the batch's arena; one that finds no room reports its count and is re-run once the
// arena has been extended by exactly what those queries need.  A scan and a compaction then lay the results out in
// query order in the result set, which owns its memory: later writes to the index do not change it.
#include "dab_common.cuh"
#include "search_common.cuh"
#include "search_host.cuh"
#include "search_pq.cuh"
#include "search_range.cuh"
#include "search_smem.cuh"

#include <cub/device/device_segmented_sort.cuh>

#include <algorithm>

struct dab_range {
    dab_index* idx = nullptr;
    dab_range *prev = nullptr, *next = nullptr;  // the index's open result sets
    uint32_t nq = 0;
    uint64_t total = 0;
    void* d_stats = nullptr;  // offsets [nq + 1] u64, cmps [nq], hops [nq] u32, second_round [nq] u8
    void* d_results = nullptr;  // ids [total] u32, dists [total] f32
    uint64_t* offsets() const { return (uint64_t*)d_stats; }
    uint32_t* cmps() const { return (uint32_t*)(offsets() + nq + 1); }
    uint32_t* hops() const { return cmps() + nq; }
    uint8_t* second() const { return (uint8_t*)(hops() + nq); }
};

namespace dab {

namespace {

constexpr size_t kRangeMaxSmem = 200 * 1024;   // a CTA's shared memory
constexpr uint64_t kRegionBudget = 1ull << 31;  // bytes of in_range regions one pass may take

inline uint64_t round_up_pow2(uint64_t n) {
    uint64_t p = 1;
    while (p < n) p <<= 1;
    return p;
}

// One warp's share of a pass: the queries of the work list it takes, whatever the distances are.  Src is a distance
// source (search_source.cuh).  radius_filter: the output drops the ids outside (inner_radius, radius]; without it only
// start points and deleted ids are dropped (the rerank filters on its own distances).
template <class Src>
__device__ __forceinline__ void range_queries(const RangeParams& p, uint8_t* base, int lane, Src& src, bool radius_filter) {
    const int wib = threadIdx.x >> 5;
    uint32_t* cid = reinterpret_cast<uint32_t*>(base + p.off_cid);
    float* cd = reinterpret_cast<float*>(base + p.off_cd);
    const uint32_t warp_slot = blockIdx.x * kRangeWarps + wib;
    const uint32_t nbk = p.n_buckets;
    uint32_t* table = p.tables + (size_t)warp_slot * nbk * 8;
    const uint32_t hlimit = nbk * 7;  // 87.5 % load
    const uint64_t n_total = p.n_points + p.n_start;
    uint32_t* rid = p.regions + (size_t)warp_slot * p.region_cap * 2;
    float* rd = reinterpret_cast<float*>(rid + p.region_cap);
    const unsigned below = (1u << lane) - 1u;

    for (uint32_t qidx; next_query(p.counters, p.n_work, p.query_list, lane, qidx);) {
        // ---- in_range: the phase-1 prefix within the radius, in list order
        const uint32_t* li = p.list_ids + (size_t)qidx * p.l_search;
        const float* ld = p.list_dists + (size_t)qidx * p.l_search;
        const uint32_t n1 = p.list_counts[qidx];
        uint64_t size = 0;
        for (uint32_t b = 0; b < n1; b += 32) {
            const uint32_t i = b + lane;
            const float d = i < n1 ? ld[i] : 0.0f;
            const bool in = i < n1 && d <= p.radius;
            const unsigned m = __ballot_sync(kFull, in);
            const uint64_t at = size + __popc(m & below);
            if (in && at < p.region_cap) rid[at] = li[i], rd[at] = d;
            size += __popc(m);
        }
        bool region_full = size > p.region_cap, overflow = region_full;
        const bool second = size >= p.min_in_range && size < p.max_returned;
        uint32_t hops = p.list_hops[qidx], nvisited = 0;
        __syncwarp();

        if (second && !overflow) {
            // ---- range_search_internal: the visited set is the in_range ids, the frontier the suffix not yet expanded
            src.load(qidx);
            for (uint32_t i = lane; i < nbk; i += 32) store_empty_bucket(table + (size_t)i * 8);
            __syncwarp();
            src.prepare();
            for (uint32_t i = lane; i < size; i += 32) visit_global(table, nbk, rid[i]);
            __syncwarp();  // every seed is in the table before any lane probes it for a neighbour
            nvisited = (uint32_t)size;
            overflow = nvisited + p.max_degree > hlimit;
            uint64_t front = 0;
            uint32_t hops2 = 0;
            while (!overflow && front < size && size < p.max_returned) {
                const uint32_t nb = (uint32_t)min((unsigned long long)p.beam, (unsigned long long)(size - front));
                const uint64_t f0 = front;
                front += nb;
                hops2 += nb;
                for (uint32_t b = 0; b < nb && size < p.max_returned; ++b) {
                    uint32_t ncand = 0;
                    expand_node(p.adj, p.adj_stride, p.max_degree, n_total, table, nbk, rid[f0 + b], cid, ncand, nvisited, lane,
                                [](bool, uint32_t, uint32_t) {});
                    if (nvisited + p.max_degree > hlimit) {
                        overflow = true;
                        break;
                    }
                    __syncwarp();
                    src.distances(cid, cd, ncand);
                    // the appends, in order, while in_range is below max_returned
                    for (uint32_t c0 = 0; c0 < ncand && size < p.max_returned; c0 += 32) {
                        const uint32_t c = c0 + lane;
                        const float d = c < ncand ? cd[c] : 0.0f;
                        const bool ok = c < ncand && d <= p.bound;
                        const unsigned m = __ballot_sync(kFull, ok);
                        const uint32_t take = (uint32_t)min((unsigned long long)__popc(m), (unsigned long long)(p.max_returned - size));
                        if (size + take > p.region_cap) {
                            region_full = overflow = true;
                            break;
                        }
                        const uint32_t rank = __popc(m & below);
                        if (ok && rank < take) rid[size + rank] = cid[c], rd[size + rank] = d;
                        size += take;
                    }
                    __syncwarp();
                    if (overflow) break;
                }
            }
            hops = hops + (hops + hops2);
        }

        if (overflow) {
            report_overflow(p.counters, p.overflow_list, qidx, lane);
            if (region_full && lane == 0) atomicAdd(p.counters + 3, 1u);
            continue;
        }

        // ---- the output: start points, deleted ids, the inner radius and the radius filtered out
        range_emit(p, rid, rd, size, radius_filter, qidx, hops, second, nvisited, lane);
    }
}

template <typename TD, int KIND, int POST, int NA>
__global__ void __launch_bounds__(kRangeWarps * 32) range_kernel(const RangeParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    uint8_t* base = smem + (size_t)wib * p.warp_smem;
    FullRowSource<TD, KIND, POST, NA, RangeParams> src(p, base, lane);
    range_queries(p, base, lane, src, true);
}

template <int MODE>
__global__ void __launch_bounds__(kRangeWarps * 32) range_kernel_quant(const RangeParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    uint8_t* base = smem + (size_t)wib * p.warp_smem;
    StoreSource<MODE, RangeParams> src(p, base, lane, blockIdx.x * kRangeWarps + wib);
    range_queries(p, base, lane, src, !p.rerank);
}

// offsets [nq + 1] <- the exclusive prefix sums of counts, by one block of 1024 threads
__global__ void __launch_bounds__(1024) range_scan(const uint32_t* counts, uint32_t nq, uint64_t* offsets) {
    __shared__ unsigned long long part[1024];
    const uint32_t t = threadIdx.x, per = (nq + 1023) / 1024;
    const uint64_t lo = (uint64_t)t * per, hi = lo + per < nq ? lo + per : (uint64_t)nq;
    unsigned long long s = 0;
    for (uint64_t i = lo; i < hi; ++i) s += counts[i];
    part[t] = s;
    __syncthreads();
    for (uint32_t o = 1; o < 1024; o <<= 1) {
        const unsigned long long v = t >= o ? part[t - o] : 0;
        __syncthreads();
        part[t] += v;
        __syncthreads();
    }
    unsigned long long run = part[t] - s;
    for (uint64_t i = lo; i < hi; ++i) {
        offsets[i] = run;
        run += counts[i];
    }
    if (t == 1023) offsets[nq] = part[1023];
}

// The results of query q from the arena (positions below `split` in the first part, the rest in the second) to
// out [offsets[q], offsets[q + 1]), a warp per query
__global__ void range_compact(const uint64_t* q_pos, const uint32_t* q_count, const uint64_t* offsets, uint32_t nq, const uint32_t* a1_ids,
                              const float* a1_dists, const uint32_t* a2_ids, const float* a2_dists, uint64_t split, uint32_t* out_ids,
                              float* out_dists) {
    const int lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t q = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5; q < nq; q += warps) {
        const uint64_t pos = q_pos[q], dst = offsets[q];
        const uint32_t n = q_count[q];
        const uint32_t* si = pos < split ? a1_ids + pos : a2_ids + (pos - split);
        const float* sd = pos < split ? a1_dists + pos : a2_dists + (pos - split);
        for (uint32_t i = lane; i < n; i += 32) {
            out_ids[dst + i] = si[i];
            out_dists[dst + i] = sd[i];
        }
    }
}

// ---- the rerank: full-precision distances in place, the radius filter, a stable sort per query --------------------
constexpr int kRangeRerankWarps = 4;

struct RangeRerankParams {
    const uint8_t* vectors;
    size_t row_stride;
    uint32_t dim, nq;
    const void* queries;  // index dtype
    const uint64_t* offsets;  // [nq + 1]: query q's results are ids / dists [offsets[q], offsets[q + 1])
    const uint32_t* ids;
    float* dists;
    float radius, inner_radius;
    int has_inner;
    uint32_t* counts;  // [nq] results within (inner_radius, radius]
    uint32_t warp_smem;
};

__device__ __forceinline__ bool in_band(float d, float radius, int has_inner, float inner_radius) {
    return !(has_inner && d <= inner_radius) && d <= radius;
}

// One warp per query: every result's Distance<T, T> to the query written over its quantized distance, and how many lie
// within (inner_radius, radius]
template <typename TD, int KIND, int POST, int NA>
__global__ void __launch_bounds__(kRangeRerankWarps * 32) range_rerank_kernel(const RangeRerankParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    float* qf = reinterpret_cast<float*>(smem + (size_t)wib * p.warp_smem);
    for (uint32_t q = blockIdx.x * kRangeRerankWarps + wib; q < p.nq; q += gridDim.x * kRangeRerankWarps) {
        const uint64_t b = p.offsets[q];
        const uint32_t m = (uint32_t)(p.offsets[q + 1] - b);
        uint32_t count = 0;
        if (m) {
            __syncwarp();
            load_query(reinterpret_cast<const TD*>(p.queries) + (size_t)q * p.dim, (int)p.dim, 16, qf, lane);
            __syncwarp();
            rerank_distances<TD, KIND, POST, NA>(qf, p.vectors, p.row_stride, p.ids + b, m, p.dists + b, (int)p.dim, lane);
            __syncwarp();
            for (uint32_t i = lane; i < m; i += 32) count += in_band(p.dists[b + i], p.radius, p.has_inner, p.inner_radius) ? 1u : 0u;
            count = __reduce_add_sync(kFull, count);
        }
        if (lane == 0) p.counts[q] = count;
    }
}

// An f32 distance as a u32 key of the same order, -0.0 and +0.0 one key (no NaN reaches the sort)
__device__ __forceinline__ uint32_t sort_key(float d) {
    const uint32_t b = __float_as_uint(d == 0.0f ? 0.0f : d);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// The rerank's rule for a reranked distance: Range's (BOUNDED) keeps (inner_radius, radius] and no NaN reaches its sort;
// FilteredRange's checks only the inner radius (it takes its matches to be within the radius), so distances above the
// radius and NaN stay, and NaN sorts after every number (order_key)
template <bool BOUNDED>
__device__ __forceinline__ bool rerank_keeps(float d, float radius, int has_inner, float inner_radius) {
    return BOUNDED ? in_band(d, radius, has_inner, inner_radius) : !(has_inner && d <= inner_radius);
}

// FilteredRange's rule: how many results of each query rerank_keeps, over range_rerank_kernel's counts of Range's; a
// warp per query
__global__ void range_rerank_count_unbounded(const uint64_t* offsets, uint32_t nq, const float* dists, int has_inner, float inner_radius,
                                             uint32_t* counts) {
    const int lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t q = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5; q < nq; q += warps) {
        uint32_t count = 0;
        for (uint64_t i = offsets[q] + lane; i < offsets[q + 1]; i += 32) count += rerank_keeps<false>(dists[i], 0.0f, has_inner, inner_radius) ? 1u : 0u;
        count = __reduce_add_sync(kFull, count);
        if (lane == 0) counts[q] = count;
    }
}

// One warp per query: the results the rule keeps, in order, from [from[q], from[q + 1]) to [to[q], to[q + 1]) of ids /
// dists, with their sort keys and their positions
template <bool BOUNDED>
__device__ __forceinline__ void rerank_filter(const uint64_t* from, const uint64_t* to, uint32_t nq, const uint32_t* ids, const float* dists,
                                              float radius, int has_inner, float inner_radius, uint32_t* out_ids, float* out_dists, uint32_t* keys,
                                              uint32_t* pos) {
    const int lane = threadIdx.x & 31;
    const unsigned below = (1u << lane) - 1u;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t q = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5; q < nq; q += warps) {
        const uint64_t b = from[q], e = from[q + 1];
        uint64_t w = to[q];
        for (uint64_t i0 = b; i0 < e; i0 += 32) {
            const uint64_t i = i0 + lane;
            const float d = i < e ? dists[i] : 0.0f;
            const bool k = i < e && rerank_keeps<BOUNDED>(d, radius, has_inner, inner_radius);
            const unsigned m = __ballot_sync(kFull, k);
            if (k) {
                const uint64_t at = w + __popc(m & below);
                out_ids[at] = ids[i];
                out_dists[at] = d;
                keys[at] = BOUNDED ? sort_key(d) : order_key(d);
                pos[at] = (uint32_t)at;
            }
            w += __popc(m);
        }
    }
}

__global__ void range_rerank_filter(const uint64_t* from, const uint64_t* to, uint32_t nq, const uint32_t* ids, const float* dists, float radius,
                                    int has_inner, float inner_radius, uint32_t* out_ids, float* out_dists, uint32_t* keys, uint32_t* pos) {
    rerank_filter<true>(from, to, nq, ids, dists, radius, has_inner, inner_radius, out_ids, out_dists, keys, pos);
}

__global__ void range_rerank_filter_unbounded(const uint64_t* from, const uint64_t* to, uint32_t nq, const uint32_t* ids, const float* dists,
                                              float radius, int has_inner, float inner_radius, uint32_t* out_ids, float* out_dists, uint32_t* keys,
                                              uint32_t* pos) {
    rerank_filter<false>(from, to, nq, ids, dists, radius, has_inner, inner_radius, out_ids, out_dists, keys, pos);
}

// out[i] <- in[pos[i]], ids and dists
__global__ void range_rerank_gather(const uint32_t* pos, uint64_t n, const uint32_t* in_ids, const float* in_dists, uint32_t* out_ids,
                                    float* out_dists) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        out_ids[i] = in_ids[pos[i]];
        out_dists[i] = in_dists[pos[i]];
    }
}

// Instantiated here, in this order, for the module order that ptxas's register allocation of the cosine range_kernel
// instantiations depends on (traversal_kernel alone would instantiate them at the end of the file)
template __global__ void range_kernel_quant<STORE_SQ>(const RangeParams);
template __global__ void range_kernel_quant<STORE_MINMAX>(const RangeParams);
template __global__ void range_kernel_quant<STORE_PQ>(const RangeParams);

template <typename S>
void (*range_kernel_of())(const RangeParams) {
    return range_kernel<typename S::TD, S::KIND, S::POST, S::NA>;
}

// A warp's shared memory: the query area (query_area_bytes), then one node's candidate ids and distances.  `store`: -1
// full precision, else a QuantStore.
size_t range_warp_smem(const dab_index* idx, int store, RangeParams* p) {
    size_t off = query_area_bytes(idx, store);
    const size_t ncand = round_up(std::max<size_t>(idx->max_degree, 32) * 4, 16);
    RangeParams scratch;
    RangeParams& q = p ? *p : scratch;
    q.off_cid = (uint32_t)off, off += ncand;
    q.off_cd = (uint32_t)off, off += ncand;
    return round_up(off, 128);
}

// range_rerank_kernel's shared memory per warp: the query (i8 / u8 rows: as they are; float rows: f32)
size_t range_rerank_smem(const dab_index* idx) {
    const bool is_int = idx->dtype == DAB_I8 || idx->dtype == DAB_U8;
    return is_int ? round_up((size_t)idx->dim, 16) : round_up((size_t)idx->dim * 4, 16);
}

// The range search's own checks, after Range::validate_and_create's (range_search.rs:91-131) in its order.  Over a
// quantized store (`store` >= 0) the traversal reads the graph and the store only; the store checks of its k-NN call
// follow, then those of the rerank.  A filtered range search (`filtered`) checks, after beam_width, the label table, the
// filtered kernel's list (L + #start <= kFilteredMaxL) and its shared memory (with the store's query area), in place of
// the range kernel's shared memory.
int check_range_args(const dab_index* idx, const char* api, int store, bool rerank, uint32_t l_search, uint32_t beam, float radius,
                     int has_inner, float inner_radius, float initial_slack, float range_slack, uint64_t max_returned, bool filtered = false) {
    if (store < 0 && (!idx->graph_ready || !idx->vectors_ready)) return fail(DAB_ERR_NOT_READY, "%s: vectors and graph must be uploaded first", api);
    if (store >= 0 && !idx->graph_ready) return fail(DAB_ERR_NOT_READY, "%s: graph must be uploaded first", api);
    if (beam == 0) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: beam_width must be > 0 (BeamWidthZero)", api);
    if (l_search == 0) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: l_search must be > 0 (LZero)", api);
    if (max_returned != 0 && max_returned < l_search)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: max_returned (%llu) must be >= l_search (%u) (MaxReturnedLessThanInitialL)", api,
                    (unsigned long long)max_returned, l_search);
    if (!(initial_slack >= 0.0f && initial_slack <= 1.0f))
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: initial_slack %g must be in [0, 1] (StartingListSlackValueError)", api, (double)initial_slack);
    if (range_slack < 1.0f) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: range_slack %g must be >= 1 (RangeSearchSlackValueError)", api, (double)range_slack);
    if (has_inner && inner_radius > radius)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: inner_radius %g must be <= radius %g (InnerRadiusValueError)", api, (double)inner_radius, (double)radius);
    if (beam > 64) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: beam_width %u > 64", api, beam);
    if (filtered) {
        if (!idx->d_labels) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: no label table (dab_upload_labels has not been called)", api);
        if ((uint64_t)l_search + idx->n_start > kFilteredMaxL)
            return fail(DAB_ERR_INVALID_ARGUMENT, "%s: L + #start = %llu > %u", api, (unsigned long long)l_search + idx->n_start, kFilteredMaxL);
        int rc;
        if ((rc = filtered_check_smem(idx, api, l_search, l_search + idx->n_start, beam, store))) return rc;
    } else {
        const size_t smem = range_warp_smem(idx, store, nullptr) * kRangeWarps;
        if (smem > kRangeMaxSmem)
            return fail(DAB_ERR_INVALID_ARGUMENT, "%s: dim=%u, max_degree=%u need %zu B shared memory per CTA (> %zu)", api, idx->dim,
                        idx->max_degree, smem, kRangeMaxSmem);
    }
    if (store < 0) return DAB_OK;
    int rc;
    if ((rc = check_quant_store(idx, (QuantStore)store, api, false))) return rc;
    if (l_search + idx->n_start > 1024) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: L + #start must be <= 1024", api);
    if (rerank) {
        if (!idx->vectors_ready) return fail(DAB_ERR_NOT_READY, "%s: rerank needs the full-precision vectors", api);
        const size_t rsmem = range_rerank_smem(idx) * kRangeRerankWarps;
        if (rsmem > kRangeMaxSmem) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: dim=%u needs %zu B shared memory per CTA in the rerank (> %zu)", api,
                                                idx->dim, rsmem, kRangeMaxSmem);
    }
    return DAB_OK;
}

// n entries (ids and dists) of result storage, or DAB_ERR_OUT_OF_MEMORY naming what the batch needs
int alloc_entries(const dab_index* idx, const char* api, DevBuf& buf, uint64_t n, uint64_t need) {
    const uint64_t limit = idx->tune.test_range_limit ? idx->tune.test_range_limit : UINT64_MAX;
    if (n > limit || buf.alloc(n * 8, api))
        return fail(DAB_ERR_OUT_OF_MEMORY, "%s: the batch's results need %llu entries (%llu bytes), more than device memory holds", api,
                    (unsigned long long)need, (unsigned long long)need * 8);
    return DAB_OK;
}

void range_unlink(dab_range* r) {
    if (r->prev) r->prev->next = r->next;
    else r->idx->ranges = r->next;
    if (r->next) r->next->prev = r->prev;
}

void range_free(dab_range* r) {
    cudaFree(r->d_stats);
    cudaFree(r->d_results);
    delete r;
}

// The rerank of a result set whose results are every in_range id (a filtered search: every match it returns) but start
// points and deleted ids: their full-precision distances, then those the rule keeps (`bounded`: Range's, within
// (inner_radius, radius]; else FilteredRange's, above inner_radius) sorted per query by that distance, stably
int range_rerank(dab_index* idx, const char* api, const void* d_queries, uint32_t nq, float radius, int has_inner, float inner_radius,
                 bool bounded, dab_range* r) {
    cudaStream_t st = idx->stream;
    int rc;
    DevBuf counts, offsets;
    if ((rc = counts.alloc((size_t)nq * 4, api)) || (rc = offsets.alloc(((size_t)nq + 1) * 8, api))) return rc;
    RangeRerankParams p;
    memset(&p, 0, sizeof(p));
    p.vectors = idx->d_vectors;
    p.row_stride = idx->row_stride;
    p.dim = idx->dim;
    p.nq = nq;
    p.queries = d_queries;
    p.offsets = r->offsets();
    p.ids = (const uint32_t*)r->d_results;
    p.dists = (float*)((uint32_t*)r->d_results + r->total);
    p.radius = radius;
    p.inner_radius = inner_radius;
    p.has_inner = has_inner ? 1 : 0;
    p.counts = (uint32_t*)counts.p;
    p.warp_smem = (uint32_t)range_rerank_smem(idx);
    const size_t smem = (size_t)p.warp_smem * kRangeRerankWarps;
    const int grid = (int)std::min<uint64_t>(((uint64_t)nq + kRangeRerankWarps - 1) / kRangeRerankWarps, (uint64_t)idx->sm_count * 8);
    if ((rc = visit_schema<OPS_ROW>(idx->dtype, idx->metric, [&](auto sc) -> int {
             using S = decltype(sc);
             auto kern = range_rerank_kernel<typename S::TD, S::KIND, S::POST, S::NA>;
             DAB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
             kern<<<grid, kRangeRerankWarps * 32, smem, st>>>(p);
             return DAB_OK;
         })))
        return rc;
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    if (!bounded) {
        range_rerank_count_unbounded<<<grid_for(idx, (uint64_t)nq * 32), 256, 0, st>>>(p.offsets, nq, p.dists, p.has_inner, inner_radius, p.counts);
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
    }
    range_scan<<<1, 1024, 0, st>>>(p.counts, nq, (uint64_t*)offsets.p);
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    uint64_t total = 0;
    DAB_CUDA(cudaMemcpyAsync(&total, (uint64_t*)offsets.p + nq, 8, cudaMemcpyDeviceToHost, st));
    DAB_CUDA(cudaStreamSynchronize(st));

    // the filtered results with their keys and positions, then the sort (CUB counts its items in int)
    DevBuf kept, keys, out;
    if (total > (uint64_t)INT32_MAX)
        return fail(DAB_ERR_OUT_OF_MEMORY, "%s: the rerank sorts %llu entries, more than %d", api, (unsigned long long)total, INT32_MAX);
    if ((rc = alloc_entries(idx, api, kept, total, total)) || (rc = alloc_entries(idx, api, keys, 2 * total, total)) ||
        (rc = alloc_entries(idx, api, out, total, total)))
        return rc;
    uint32_t* kept_ids = (uint32_t*)kept.p;
    float* kept_dists = (float*)(kept_ids + total);
    uint32_t* k_in = (uint32_t*)keys.p;
    uint32_t* v_in = k_in + total;
    uint32_t* k_out = v_in + total;
    uint32_t* v_out = k_out + total;
    (bounded ? range_rerank_filter : range_rerank_filter_unbounded)<<<grid_for(idx, (uint64_t)nq * 32), 256, 0, st>>>(
        r->offsets(), (const uint64_t*)offsets.p, nq, p.ids, p.dists, radius, p.has_inner, inner_radius, kept_ids, kept_dists, k_in, v_in);
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    if (total) {
        const uint64_t* seg = (const uint64_t*)offsets.p;
        size_t tmp_bytes = 0;
        DAB_CUDA(cub::DeviceSegmentedSort::StableSortPairs(nullptr, tmp_bytes, k_in, k_out, v_in, v_out, (int)total, (int)nq, seg, seg + 1, st));
        DevBuf tmp;
        if ((rc = tmp.alloc(tmp_bytes, api))) return rc;
        DAB_CUDA(cub::DeviceSegmentedSort::StableSortPairs(tmp.p, tmp_bytes, k_in, k_out, v_in, v_out, (int)total, (int)nq, seg, seg + 1, st));
        DAB_LAUNCHED();
        range_rerank_gather<<<grid_for(idx, total), 256, 0, st>>>(v_out, total, kept_ids, kept_dists, (uint32_t*)out.p,
                                                                  (float*)((uint32_t*)out.p + total));
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
    }
    DAB_CUDA(cudaMemcpyAsync(r->offsets(), offsets.p, ((size_t)nq + 1) * 8, cudaMemcpyDeviceToDevice, st));
    DAB_CUDA(cudaStreamSynchronize(st));
    cudaFree(r->d_results);
    r->d_results = out.p;
    out.p = nullptr;
    r->total = total;
    return DAB_OK;
}

// A filtered range search's device masks (one per query) and mode
struct RangeFilter {
    const uint64_t* masks;
    uint32_t match_all;
};

// Both phases for nq >= 1 queries (checks passed) into a new result set: over full-precision rows (`store` -1) or a
// QuantStore, whose results `rerank` reorders by full-precision distance.  With `filt` both phases are the filtered range
// search's, in filtered_range_kernel (_quant over a store): its passes run the traversal too, and write cmps.
int range_run(dab_index* idx, const char* api, const void* d_queries, uint32_t nq, uint32_t l_search, uint32_t beam, float radius, int has_inner,
              float inner_radius, float initial_slack, float range_slack, uint64_t max_returned, int store, bool rerank, dab_range* r,
              const RangeFilter* filt) {
    cudaStream_t st = idx->stream;
    int rc;
    // ---- the result set's statistics, then phase 1: the first L entries of every list with start points and
    // deleted ids kept, its cmps (the result set's) and hops
    const size_t stat_bytes = ((size_t)nq + 1) * 8 + (size_t)nq * 9;
    DAB_CUDA(cudaMalloc(&r->d_stats, stat_bytes));
    DevBuf p1;
    const size_t lq = filt ? 0 : (size_t)nq * l_search;
    if ((rc = p1.alloc(lq * 8 + (size_t)nq * 8, api))) return rc;
    uint32_t* list_ids = (uint32_t*)p1.p;
    float* list_dists = (float*)(list_ids + lq);
    uint32_t* list_counts = (uint32_t*)(list_dists + lq);
    uint32_t* list_hops = list_counts + nq;
    SearchRecord rec{};
    rec.keep_starts = true;
    rec.keep_deleted = true;
    StagedQueries staged{};  // SQ / MinMax: the queries phase 1 compressed, which phase 2 reads too
    rec.staged = &staged;
    if (!filt && (rc = run_search(idx, d_queries, nq, l_search, l_search, beam, SearchOut{list_ids, list_dists, list_counts, r->cmps(), list_hops},
                                  store, false, &rec)))
        return rc;
    uint32_t* h = (uint32_t*)idx->h_counters.p;  // pinned: the five counters, then the three arena counters
    if (filt && (store == STORE_SQ || store == STORE_MINMAX)) {
        // the filtered traversal does not run through the job: the queries are compressed here, once for both phases
        if ((rc = idx->s_stage.reserve(store == STORE_SQ ? sq_stage_bytes(idx, nq) : minmax_stage_bytes(idx, nq))) ||
            (rc = stage_store_queries(idx, st, idx->s_stage, store, d_queries, nq, h, staged)))
            return rc;
        if (store == STORE_MINMAX) {  // a batch with a NaN query fails before any traversal is launched
            DAB_CUDA(cudaStreamSynchronize(st));
            if (staged_first_nan(h) != ~0ull)
                return fail(DAB_ERR_INVALID_ARGUMENT, "%s: query %llu contains NaN after the transform (InputContainsNaN)", api, staged_first_nan(h));
        }
    }

    // ---- phase 2
    RangeParams p;
    memset(&p, 0, sizeof(p));
    p.warp_smem = (uint32_t)range_warp_smem(idx, store, &p);
    WarpPlan<RangeParams> plan;
    FilteredRangeParams fp;
    WarpPlan<FilteredRangeParams> fplan;
    if (filt) {
        memset(&fp, 0, sizeof(fp));
        rc = filtered_range_plan(idx, l_search, beam, store, fp, fplan);
    } else if (!(rc = traversal_kernel(idx, store, [](auto m) { return range_kernel_quant<decltype(m)::value>; },
                                       [](auto sc) { return range_kernel_of<decltype(sc)>(); }, plan.kern))) {
        plan_warps(idx, store, kRangeWarps, p.warp_smem, SIZE_MAX, plan);  // (the shared memory was checked with the arguments)
    }
    if (rc) return rc;
    const int resident = filt ? fplan.grid : plan.grid, warps_per_cta = filt ? fplan.warps : plan.warps;
    if (!resident)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: dim=%u needs %zu B shared memory per CTA", api, idx->dim, filt ? fplan.smem_block : plan.smem_block);
    DevBuf luts;
    if (store >= 0) {
        set_store_params(idx, (QuantStore)store, p.store);
        p.store.query_codes = staged.codes;
        p.store.query_meta = staged.meta;
        p.rerank = rerank ? 1 : 0;
        if ((rc = luts.alloc(std::max<size_t>(pq_table_bytes(idx, store, (uint64_t)resident * warps_per_cta), 16), api))) return rc;
        p.store.luts = (float*)luts.p;
    }
    set_graph_params(idx, p);
    p.vectors = idx->d_vectors;
    p.row_stride = idx->row_stride;
    p.queries = d_queries;
    p.l_search = l_search;
    p.beam = beam;
    p.list_ids = list_ids, p.list_dists = list_dists, p.list_counts = list_counts, p.list_hops = list_hops;
    p.radius = radius;
    p.bound = radius * range_slack;  // an f32 product, as the reference's
    p.has_inner = has_inner ? 1 : 0;
    p.inner_radius = inner_radius;
    p.min_in_range = (uint64_t)((float)l_search * initial_slack);
    p.max_returned = max_returned ? max_returned : UINT64_MAX;
    p.deleted = deleted_filter(idx);
    p.out_hops = r->hops();
    p.out_second = r->second();
    if (filt) {
        // phase 1: the filtered traversal at L + #start without adaptive L; its tables, counters and work list are p's
        set_graph_params(idx, fp.f);
        fp.f.vectors = idx->d_vectors;
        fp.f.row_stride = idx->row_stride;
        fp.f.queries = d_queries;
        fp.f.cap = l_search;
        fp.f.beam = beam;
        fp.f.best_cap = l_search + idx->n_start;
        fp.f.labels = idx->d_labels;
        fp.f.masks = filt->masks;
        fp.f.match_all = filt->match_all;
        fp.f.store = p.store;
        fp.out_cmps = r->cmps();
    }

    DevBuf ctr, per_query, tables, regions, arena1, arena2;
    if ((rc = ctr.alloc(64 + (size_t)nq * 8, api)) || (rc = per_query.alloc((size_t)nq * 12, api))) return rc;
    p.arena_ctr = (unsigned long long*)ctr.p;
    p.counters = (uint32_t*)((uint8_t*)ctr.p + 32);
    p.overflow_list = (uint32_t*)((uint8_t*)ctr.p + 64);
    p.arena_fail = p.overflow_list + nq;
    p.q_pos = (uint64_t*)per_query.p;
    p.q_count = (uint32_t*)(p.q_pos + nq);
    DAB_CUDA(cudaMemsetAsync(ctr.p, 0, 64, st));

    // the in_range regions (filtered: the matches, which max_returned does not bound in phase 1) and the arena of the
    // first pass
    const uint64_t region_max = filt ? idx->n_total() : std::min<uint64_t>(p.max_returned, idx->n_total());
    uint64_t region = idx->tune.test_range_list ? idx->tune.test_range_list : round_up(std::max<uint64_t>(4ull * l_search, 1024), 32);
    region = std::min(region, region_max);
    uint64_t slots = table_slots(idx, VisitedHint{}, filt ? l_search + idx->n_start : l_search, beam, STORE_PQ);
    const uint64_t limit = idx->tune.test_range_limit ? idx->tune.test_range_limit : UINT64_MAX;
    const uint64_t arena_first = std::min<uint64_t>(idx->tune.test_range_arena ? idx->tune.test_range_arena : (uint64_t)nq * l_search, limit);
    if ((rc = alloc_entries(idx, api, arena1, arena_first, arena_first))) return rc;
    p.arena_ids = (uint32_t*)arena1.p;
    p.arena_dists = (float*)(p.arena_ids + arena_first);
    p.arena_first = 0;
    p.arena_end = arena_first;

    DevBuf retry, fronts, keys;
    if ((rc = retry.alloc((size_t)nq * 4, api))) return rc;
    p.n_work = nq;
    int pass = 0;
    bool grown = false;
    uint64_t used = 0;
    for (;;) {
        // the grid of this pass: one warp per query at most, and regions within kRegionBudget
        int grid = balanced_grid(p.n_work, resident, warps_per_cta);
        // a filtered search's warp also holds a frontier of region + L entries and the sort keys of as many
        const uint64_t front = region + l_search, key_cap = filt ? round_up_pow2(front) : 0;
        const uint64_t warp_bytes = region * 8 + (filt ? front * 8 + key_cap * 8 : 0);
        const uint64_t region_grid = std::max<uint64_t>(1, kRegionBudget / (warp_bytes * warps_per_cta));
        grid = (int)std::min<uint64_t>(grid, region_grid);
        const uint64_t warps = (uint64_t)grid * warps_per_cta;
        p.n_buckets = (uint32_t)((slots + 7) / 8);
        p.region_cap = (uint32_t)region;
        if ((rc = tables.alloc(warps * p.n_buckets * 32, api)) || (rc = regions.alloc(warps * region * 8, api))) return rc;
        p.tables = (uint32_t*)tables.p;
        p.regions = (uint32_t*)regions.p;
        DAB_CUDA(cudaMemsetAsync(p.counters, 0, 16, st));
        if (filt) {
            if ((rc = fronts.alloc(warps * front * 8, api)) || (rc = keys.alloc(warps * key_cap * 8, api))) return rc;
            fp.r = p;
            fp.f.query_list = p.query_list;
            fp.f.n_work = p.n_work;
            fp.f.tables = p.tables;
            fp.f.n_buckets = p.n_buckets;
            fp.f.counters = p.counters;
            fp.f.overflow_list = p.overflow_list;
            fp.fronts = (uint32_t*)fronts.p;
            fp.keys = (unsigned long long*)keys.p;
            fp.front_cap = (uint32_t)front;
            fp.key_cap = (uint32_t)key_cap;
        }
        if ((rc = filt ? warp_launch(fp, fplan, grid, st) : warp_launch(p, plan, grid, st))) return rc;
        DAB_CUDA(cudaMemcpyAsync(h, ctr.p, 64, cudaMemcpyDeviceToHost, st));
        DAB_CUDA(cudaStreamSynchronize(st));
        const unsigned long long* actr = (const unsigned long long*)h;
        const uint32_t* c = h + 8;
        const uint32_t n_over = c[1], n_region = c[3], n_fail = c[4];
        if (n_over) {
            // the stopped queries are the next pass's work: on larger tables, larger regions, or both
            if (n_over > n_region && (rc = grow_visited_tables(idx, pass, slots))) return rc;
            if (n_region) region = std::min(region * 4, region_max);
            DAB_CUDA(cudaMemcpyAsync(retry.p, p.overflow_list, (size_t)n_over * 4, cudaMemcpyDeviceToDevice, st));
            p.query_list = (const uint32_t*)retry.p;
            p.n_work = n_over;
            continue;
        }
        if (n_fail) {
            // every query has completed; those that found no room re-run into an arena of exactly what they need
            if (grown) return fail(DAB_ERR_CUDA, "%s: queries re-run into the extended arena found no room", api);
            used = actr[1];
            const uint64_t need = actr[2];
            if ((rc = alloc_entries(idx, api, arena2, need, used + need))) return rc;
            grown = true;
            p.arena_ids = (uint32_t*)arena2.p;
            p.arena_dists = (float*)(p.arena_ids + need);
            p.arena_first = used;
            p.arena_end = used + need;
            const unsigned long long reset[3] = {used, used, 0};
            DAB_CUDA(cudaMemcpyAsync(ctr.p, reset, sizeof(reset), cudaMemcpyHostToDevice, st));
            DAB_CUDA(cudaMemsetAsync(p.counters + 4, 0, 4, st));
            DAB_CUDA(cudaMemcpyAsync(retry.p, p.arena_fail, (size_t)n_fail * 4, cudaMemcpyDeviceToDevice, st));
            DAB_CUDA(cudaStreamSynchronize(st));  // `reset` is read from pageable host memory
            p.query_list = (const uint32_t*)retry.p;
            p.n_work = n_fail;
            continue;
        }
        break;
    }
    cudaFree(tables.p), cudaFree(regions.p), cudaFree(fronts.p), cudaFree(keys.p);
    tables.p = regions.p = fronts.p = keys.p = nullptr;

    // ---- the result set: offsets, then the results in query order
    range_scan<<<1, 1024, 0, st>>>(p.q_count, nq, r->offsets());
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    DAB_CUDA(cudaMemcpyAsync(&r->total, r->offsets() + nq, 8, cudaMemcpyDeviceToHost, st));
    DAB_CUDA(cudaStreamSynchronize(st));
    DevBuf out;
    if ((rc = alloc_entries(idx, api, out, r->total, r->total))) return rc;
    const uint64_t split = grown ? used : UINT64_MAX;
    const uint32_t* a2_ids = grown ? (const uint32_t*)arena2.p : nullptr;
    const float* a2_dists = grown ? (const float*)(a2_ids + (p.arena_end - used)) : nullptr;
    range_compact<<<grid_for(idx, (uint64_t)nq * 32), 256, 0, st>>>(p.q_pos, p.q_count, r->offsets(), nq, (const uint32_t*)arena1.p,
                                                                    (const float*)((const uint32_t*)arena1.p + arena_first), a2_ids, a2_dists,
                                                                    split, (uint32_t*)out.p, (float*)((uint32_t*)out.p + r->total));
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    DAB_CUDA(cudaStreamSynchronize(st));
    r->d_results = out.p;
    out.p = nullptr;
    if (rerank) {
        cudaFree(luts.p), cudaFree(p1.p), cudaFree(arena1.p), cudaFree(arena2.p);
        luts.p = p1.p = arena1.p = arena2.p = nullptr;
        return range_rerank(idx, api, d_queries, nq, radius, has_inner, inner_radius, !filt, r);
    }
    return DAB_OK;
}

// a batch of no queries: offsets {0}
int range_empty(dab_index* idx, dab_range* r) {
    DAB_CUDA(cudaMalloc(&r->d_stats, 8));
    DAB_CUDA(cudaMemsetAsync(r->d_stats, 0, 8, idx->stream));
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    return DAB_OK;
}

// nq >= 1 queries, from the host (`host`, copied to the handle's scratch) or the device
int range_batch(dab_index* idx, const char* api, bool host, const void* queries, uint32_t nq, uint32_t l_search, uint32_t beam, float radius,
                int has_inner, float inner_radius, float initial_slack, float range_slack, uint64_t max_returned, int store, bool rerank,
                dab_range* r, const uint64_t* masks, uint32_t match_all) {
    const void* d_queries = queries;
    if (host) {
        const size_t qbytes = (size_t)nq * idx->dim * elem_size(idx->dtype);
        int rc;
        if ((rc = idx->s_queries.reserve(qbytes))) return rc;
        d_queries = idx->s_queries.p;
        DAB_CUDA(cudaMemcpyAsync(idx->s_queries.p, queries, qbytes, cudaMemcpyHostToDevice, idx->stream));
    }
    if (!masks) return range_run(idx, api, d_queries, nq, l_search, beam, radius, has_inner, inner_radius, initial_slack, range_slack, max_returned,
                                 store, rerank, r, nullptr);
    RangeFilter filt{masks, match_all};
    if (host) {
        int rc;
        if ((rc = idx->s_pools.reserve((size_t)nq * 8))) return rc;
        DAB_CUDA(cudaMemcpyAsync(idx->s_pools.p, masks, (size_t)nq * 8, cudaMemcpyHostToDevice, idx->stream));
        filt.masks = (const uint64_t*)idx->s_pools.p;
    }
    return range_run(idx, api, d_queries, nq, l_search, beam, radius, has_inner, inner_radius, initial_slack, range_slack, max_returned, store,
                     rerank, r, &filt);
}

// `store`: -1 full precision, else the QuantStore both phases read; `rerank` (a store) reorders the results by
// full-precision distance.  `filtered`: a filtered range search with one mask per query in `masks` (host or device
// memory, as the queries) and the mode match_all.
int range_search(dab_index* idx, const char* api, bool host, const void* queries, uint32_t nq, uint32_t l_search, uint32_t beam, float radius,
                 int has_inner, float inner_radius, float initial_slack, float range_slack, uint64_t max_returned, dab_range** out,
                 int store = -1, bool rerank = false, bool filtered = false, const uint64_t* masks = nullptr, uint32_t match_all = 0) {
    if (!idx || !out || (nq && !queries) || (nq && filtered && !masks)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL argument", api);
    *out = nullptr;
    int rc;
    if ((rc = check_range_args(idx, api, store, rerank, l_search, beam, radius, has_inner, inner_radius, initial_slack, range_slack,
                               max_returned, filtered)))
        return rc;
    DAB_CUDA(cudaSetDevice(idx->device));
    if ((rc = idx->h_counters.reserve(64))) return rc;
    dab_range* r = new dab_range();
    r->idx = idx;
    r->nq = nq;
    if ((rc = nq ? range_batch(idx, api, host, queries, nq, l_search, beam, radius, has_inner, inner_radius, initial_slack, range_slack,
                               max_returned, store, rerank, r, filtered ? masks : nullptr, match_all)
                 : range_empty(idx, r))) {
        cudaStreamSynchronize(idx->stream);
        range_free(r);
        return rc;
    }
    r->next = idx->ranges;
    if (r->next) r->next->prev = r;
    idx->ranges = r;
    *out = r;
    return DAB_OK;
}

}  // namespace

void range_release(dab_index* idx) {
    while (idx->ranges) {
        dab_range* r = idx->ranges;
        range_unlink(r);
        range_free(r);
    }
}

}  // namespace dab

using namespace dab;

extern "C" {

int dab_range_search(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search, uint32_t beam_width, float radius, int has_inner_radius,
                     float inner_radius, float initial_slack, float range_slack, uint64_t max_returned, dab_range** out) {
    return range_search(idx, "dab_range_search", true, queries, nq, l_search, beam_width, radius, has_inner_radius, inner_radius, initial_slack,
                        range_slack, max_returned, out);
}

int dab_range_search_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t l_search, uint32_t beam_width, float radius,
                            int has_inner_radius, float inner_radius, float initial_slack, float range_slack, uint64_t max_returned,
                            dab_range** out) {
    return range_search(idx, "dab_range_search_device", false, d_queries, nq, l_search, beam_width, radius, has_inner_radius, inner_radius,
                        initial_slack, range_slack, max_returned, out);
}

// FilteredRange::search (filtered_range_search.rs:119-248): the masks and mode of dab_search_batch_filtered
int dab_range_search_filtered(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search, uint32_t beam_width, float radius,
                              int has_inner_radius, float inner_radius, float initial_slack, float range_slack, uint64_t max_returned,
                              const uint64_t* query_masks, uint32_t match_all, dab_range** out) {
    return range_search(idx, "dab_range_search_filtered", true, queries, nq, l_search, beam_width, radius, has_inner_radius, inner_radius,
                        initial_slack, range_slack, max_returned, out, -1, false, true, query_masks, match_all);
}

int dab_range_search_filtered_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t l_search, uint32_t beam_width, float radius,
                                     int has_inner_radius, float inner_radius, float initial_slack, float range_slack, uint64_t max_returned,
                                     const uint64_t* d_query_masks, uint32_t match_all, dab_range** out) {
    return range_search(idx, "dab_range_search_filtered_device", false, d_queries, nq, l_search, beam_width, radius, has_inner_radius,
                        inner_radius, initial_slack, range_slack, max_returned, out, -1, false, true, d_query_masks, match_all);
}

// FilteredRange::search over a store (graph::ext::labeled::Filtered over the quantized strategies, labeled.rs:118-129)
int dab_range_search_filtered_pq(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search, uint32_t beam_width, float radius,
                                 int has_inner_radius, float inner_radius, float initial_slack, float range_slack, uint64_t max_returned,
                                 const uint64_t* query_masks, uint32_t match_all, int rerank, dab_range** out) {
    return range_search(idx, "dab_range_search_filtered_pq", true, queries, nq, l_search, beam_width, radius, has_inner_radius, inner_radius,
                        initial_slack, range_slack, max_returned, out, STORE_PQ, rerank != 0, true, query_masks, match_all);
}

int dab_range_search_filtered_pq_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t l_search, uint32_t beam_width,
                                        float radius, int has_inner_radius, float inner_radius, float initial_slack, float range_slack,
                                        uint64_t max_returned, const uint64_t* d_query_masks, uint32_t match_all, int rerank, dab_range** out) {
    return range_search(idx, "dab_range_search_filtered_pq_device", false, d_queries, nq, l_search, beam_width, radius, has_inner_radius,
                        inner_radius, initial_slack, range_slack, max_returned, out, STORE_PQ, rerank != 0, true, d_query_masks, match_all);
}

int dab_range_search_filtered_sq(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search, uint32_t beam_width, float radius,
                                 int has_inner_radius, float inner_radius, float initial_slack, float range_slack, uint64_t max_returned,
                                 const uint64_t* query_masks, uint32_t match_all, int rerank, dab_range** out) {
    return range_search(idx, "dab_range_search_filtered_sq", true, queries, nq, l_search, beam_width, radius, has_inner_radius, inner_radius,
                        initial_slack, range_slack, max_returned, out, STORE_SQ, rerank != 0, true, query_masks, match_all);
}

int dab_range_search_filtered_sq_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t l_search, uint32_t beam_width,
                                        float radius, int has_inner_radius, float inner_radius, float initial_slack, float range_slack,
                                        uint64_t max_returned, const uint64_t* d_query_masks, uint32_t match_all, int rerank, dab_range** out) {
    return range_search(idx, "dab_range_search_filtered_sq_device", false, d_queries, nq, l_search, beam_width, radius, has_inner_radius,
                        inner_radius, initial_slack, range_slack, max_returned, out, STORE_SQ, rerank != 0, true, d_query_masks, match_all);
}

int dab_range_search_filtered_minmax(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search, uint32_t beam_width, float radius,
                                     int has_inner_radius, float inner_radius, float initial_slack, float range_slack, uint64_t max_returned,
                                     const uint64_t* query_masks, uint32_t match_all, int rerank, dab_range** out) {
    return range_search(idx, "dab_range_search_filtered_minmax", true, queries, nq, l_search, beam_width, radius, has_inner_radius, inner_radius,
                        initial_slack, range_slack, max_returned, out, STORE_MINMAX, rerank != 0, true, query_masks, match_all);
}

int dab_range_search_filtered_minmax_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t l_search, uint32_t beam_width,
                                            float radius, int has_inner_radius, float inner_radius, float initial_slack, float range_slack,
                                            uint64_t max_returned, const uint64_t* d_query_masks, uint32_t match_all, int rerank,
                                            dab_range** out) {
    return range_search(idx, "dab_range_search_filtered_minmax_device", false, d_queries, nq, l_search, beam_width, radius, has_inner_radius,
                        inner_radius, initial_slack, range_slack, max_returned, out, STORE_MINMAX, rerank != 0, true, d_query_masks, match_all);
}

int dab_range_search_pq(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search, uint32_t beam_width, float radius,
                        int has_inner_radius, float inner_radius, float initial_slack, float range_slack, uint64_t max_returned, int rerank,
                        dab_range** out) {
    return range_search(idx, "dab_range_search_pq", true, queries, nq, l_search, beam_width, radius, has_inner_radius, inner_radius, initial_slack,
                        range_slack, max_returned, out, STORE_PQ, rerank != 0);
}

int dab_range_search_pq_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t l_search, uint32_t beam_width, float radius,
                               int has_inner_radius, float inner_radius, float initial_slack, float range_slack, uint64_t max_returned, int rerank,
                               dab_range** out) {
    return range_search(idx, "dab_range_search_pq_device", false, d_queries, nq, l_search, beam_width, radius, has_inner_radius, inner_radius,
                        initial_slack, range_slack, max_returned, out, STORE_PQ, rerank != 0);
}

int dab_range_search_sq(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search, uint32_t beam_width, float radius,
                        int has_inner_radius, float inner_radius, float initial_slack, float range_slack, uint64_t max_returned, int rerank,
                        dab_range** out) {
    return range_search(idx, "dab_range_search_sq", true, queries, nq, l_search, beam_width, radius, has_inner_radius, inner_radius, initial_slack,
                        range_slack, max_returned, out, STORE_SQ, rerank != 0);
}

int dab_range_search_sq_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t l_search, uint32_t beam_width, float radius,
                               int has_inner_radius, float inner_radius, float initial_slack, float range_slack, uint64_t max_returned, int rerank,
                               dab_range** out) {
    return range_search(idx, "dab_range_search_sq_device", false, d_queries, nq, l_search, beam_width, radius, has_inner_radius, inner_radius,
                        initial_slack, range_slack, max_returned, out, STORE_SQ, rerank != 0);
}

int dab_range_search_minmax(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search, uint32_t beam_width, float radius,
                            int has_inner_radius, float inner_radius, float initial_slack, float range_slack, uint64_t max_returned, int rerank,
                            dab_range** out) {
    return range_search(idx, "dab_range_search_minmax", true, queries, nq, l_search, beam_width, radius, has_inner_radius, inner_radius,
                        initial_slack, range_slack, max_returned, out, STORE_MINMAX, rerank != 0);
}

int dab_range_search_minmax_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t l_search, uint32_t beam_width, float radius,
                                   int has_inner_radius, float inner_radius, float initial_slack, float range_slack, uint64_t max_returned,
                                   int rerank, dab_range** out) {
    return range_search(idx, "dab_range_search_minmax_device", false, d_queries, nq, l_search, beam_width, radius, has_inner_radius,
                        inner_radius, initial_slack, range_slack, max_returned, out, STORE_MINMAX, rerank != 0);
}

int dab_range_offsets(const dab_range* r, uint64_t* offsets, uint32_t* cmps, uint32_t* hops, uint8_t* second_round) {
    if (!r || !offsets) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_range_offsets: NULL argument");
    DAB_CUDA(cudaSetDevice(r->idx->device));
    const size_t nq = r->nq;
    DAB_CUDA(cudaMemcpy(offsets, r->offsets(), (nq + 1) * 8, cudaMemcpyDeviceToHost));
    if (nq && cmps) DAB_CUDA(cudaMemcpy(cmps, r->cmps(), nq * 4, cudaMemcpyDeviceToHost));
    if (nq && hops) DAB_CUDA(cudaMemcpy(hops, r->hops(), nq * 4, cudaMemcpyDeviceToHost));
    if (nq && second_round) DAB_CUDA(cudaMemcpy(second_round, r->second(), nq, cudaMemcpyDeviceToHost));
    return DAB_OK;
}

static int range_results(const dab_range* r, const char* api, uint32_t* ids, float* dists, cudaMemcpyKind kind) {
    if (!r || (r->total && (!ids || !dists))) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL argument", api);
    if (!r->total) return DAB_OK;
    DAB_CUDA(cudaSetDevice(r->idx->device));
    DAB_CUDA(cudaMemcpy(ids, r->d_results, r->total * 4, kind));
    DAB_CUDA(cudaMemcpy(dists, (const uint32_t*)r->d_results + r->total, r->total * 4, kind));
    return DAB_OK;
}

int dab_range_results(const dab_range* r, uint32_t* ids, float* dists) {
    return range_results(r, "dab_range_results", ids, dists, cudaMemcpyDeviceToHost);
}

int dab_range_results_device(const dab_range* r, uint32_t* d_ids, float* d_dists) {
    return range_results(r, "dab_range_results_device", d_ids, d_dists, cudaMemcpyDeviceToDevice);
}

void dab_range_free(dab_range* r) {
    if (!r) return;
    cudaSetDevice(r->idx->device);
    cudaStreamSynchronize(r->idx->stream);
    range_unlink(r);
    range_free(r);
}

}  // extern "C"
