// search_range.cuh — what the range search (search_range.cu) shares with the filtered range search (search_filtered.cu):
// the parameter block of a range pass, the per-node expand_beam of the second round, the output of a query's results
// into the batch's arena, and the launch of a filtered range pass from the range search's pass loop.
#pragma once

#include "dab_common.cuh"
#include "search_common.cuh"
#include "search_filtered.cuh"
#include "search_host.cuh"
#include "search_source.cuh"

namespace dab {

constexpr int kRangeWarps = 4;

struct RangeParams {
    const uint32_t* adj;
    uint32_t adj_stride;
    uint64_t n_points;
    uint32_t n_start;
    uint32_t dim;
    uint32_t max_degree;
    const uint8_t* vectors;
    size_t row_stride;
    const void* queries;
    const uint32_t* query_list;  // the queries of a re-run pass (NULL: 0 .. n_work-1)
    uint32_t n_work;
    uint32_t l_search, beam;
    // phase 1: the first L list entries of every query [nq][L], their number and the hops [nq]
    const uint32_t* list_ids;
    const float* list_dists;
    const uint32_t* list_counts;
    const uint32_t* list_hops;
    float radius, bound, inner_radius;  // bound: radius * range_slack
    int has_inner;
    uint64_t min_in_range;  // (f32(L) * initial_slack) as usize
    uint64_t max_returned;  // UINT64_MAX: None
    const uint32_t* deleted;  // NULL: nothing deleted
    uint32_t* tables;
    uint32_t n_buckets;
    uint32_t* regions;  // region_cap ids then region_cap dists for every warp of the pass
    uint32_t region_cap;
    // counters[0] work cursor, [1] stopped queries (listed in overflow_list), [2] largest visited set, [3] the stopped
    // queries whose region was full, [4] queries without room in the arena (listed in arena_fail)
    uint32_t* counters;
    uint32_t* overflow_list;
    uint32_t* arena_fail;
    // the arena: positions [arena_first, arena_end) are arena_ids / arena_dists [0, arena_end - arena_first);
    // arena_ctr: the next position, the entries written, the entries of the queries that found no room
    uint32_t* arena_ids;
    float* arena_dists;
    uint64_t arena_first, arena_end;
    unsigned long long* arena_ctr;
    uint64_t* q_pos;
    uint32_t *q_count, *out_hops;
    uint8_t* out_second;
    uint32_t warp_smem, off_cid, off_cd;
    StoreParams store;  // the quantized stores (range_kernel_quant)
    int rerank;  // the output keeps every in_range id but start points and deleted ids, for range_rerank
};

// A filtered range pass (filtered_range_kernel, search_filtered.cu): phase 1 is the filtered traversal of `f` (its
// tables, counters and work list those of `r`), the rest reads `r`.  Every warp owns, next to r's region of matches
// (region_cap ids and dists), a frontier of front_cap = region_cap + L ids and dists and key_cap (a power of two
// >= front_cap) sort keys.
struct FilteredRangeParams {
    SearchParamsFiltered f;
    RangeParams r;
    uint32_t* fronts;
    unsigned long long* keys;
    uint32_t front_cap, key_cap;
    uint32_t* out_cmps;  // [nq]
};

// expand_beam of one node (provider.rs:436-479): its unvisited, in-bounds neighbours in adjacency order appended to
// cid[ncand..]; every id that enters the visited set counts in nvisited.  Before each 32-word step is collected,
// on_new(isnew, word, ncand) sees the lanes' words (the filtered search reads the label sets there).
template <class OnNew>
__device__ __forceinline__ void expand_node(const uint32_t* adj, uint32_t adj_stride, uint32_t max_degree, uint64_t n_total, uint32_t* table,
                                            uint32_t nbk, uint32_t node, uint32_t* cid, uint32_t& ncand, uint32_t& nvisited, int lane,
                                            OnNew&& on_new) {
    const uint32_t* row = adj + (size_t)node * adj_stride;
    const uint32_t deg = min(__ldg(row), max_degree);
    for (uint32_t c0 = 0; c0 < deg + 1; c0 += 32) {
        const uint32_t j = c0 + lane;
        const uint32_t word = j < adj_stride ? __ldg(row + j) : kEmptyV2;
        const bool inserted = j >= 1 && j <= deg && visit_global(table, nbk, word);
        const bool isnew = inserted && word < n_total;
        on_new(isnew, word, ncand);
        push_new(inserted, isnew, word, cid, ncand, nvisited, lane);
    }
}

// The output of one completed query: of rid / rd [0, size), the ids that are not start points or deleted (and with
// radius_filter, within (inner_radius, radius]), in order, into the batch's arena, or the query listed in arena_fail
// when the arena has no room for them; then its count, position, hops and second-round flag
__device__ __forceinline__ void range_emit(const RangeParams& p, const uint32_t* rid, const float* rd, uint64_t size, bool radius_filter,
                                           uint32_t qidx, uint32_t hops, bool second, uint32_t nvisited, int lane) {
    const unsigned below = (1u << lane) - 1u;
    auto keep = [&](uint64_t i) {
        if (i >= size) return false;
        const uint32_t id = rid[i];
        const float d = rd[i];
        if (id >= p.n_points) return false;
        if (p.deleted && (__ldg(p.deleted + (id >> 5)) >> (id & 31) & 1u)) return false;
        if (!radius_filter) return true;
        if (p.has_inner && d <= p.inner_radius) return false;
        return d <= p.radius;
    };
    uint32_t count = 0;
    for (uint64_t b = 0; b < size; b += 32) count += __popc(__ballot_sync(kFull, keep(b + lane)));
    unsigned long long pos = 0;
    int fits = 1;
    if (lane == 0 && count) {
        pos = atomicAdd(p.arena_ctr, (unsigned long long)count);
        fits = pos + count <= p.arena_end;
        if (fits) {
            atomicAdd(p.arena_ctr + 1, (unsigned long long)count);
        } else {
            p.arena_fail[atomicAdd(p.counters + 4, 1u)] = qidx;
            atomicAdd(p.arena_ctr + 2, (unsigned long long)count);
        }
    }
    pos = __shfl_sync(kFull, pos, 0);
    fits = __shfl_sync(kFull, fits, 0);
    if (fits && count) {
        uint32_t w = 0;
        for (uint64_t b = 0; b < size; b += 32) {
            const uint64_t i = b + lane;
            const bool k = keep(i);
            const unsigned m = __ballot_sync(kFull, k);
            if (k) {
                const uint64_t at = pos - p.arena_first + w + __popc(m & below);
                p.arena_ids[at] = rid[i];
                p.arena_dists[at] = rd[i];
            }
            w += __popc(m);
        }
    }
    if (lane == 0) {
        atomicMax(p.counters + 2, nvisited);
        p.q_count[qidx] = count;
        p.q_pos[qidx] = pos;
        p.out_hops[qidx] = hops;
        p.out_second[qidx] = second ? 1 : 0;
    }
}

// fast_distance's order as an unsigned key: -0.0 and +0.0 equal, every NaN after every number
__device__ __forceinline__ uint32_t order_key(float d) {
    if (d != d) return 0xFFFFFFFFu;
    const uint32_t u = __float_as_uint(d == 0.0f ? 0.0f : d);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// ---- host (search_filtered.cu) ----------------------------------------------------------------------------------------
// The filtered range kernel of this index's schema (store -1) or of `store`, and its shape (plan.grid 0: no CTA fits,
// which the range search reports; its passes cap the grid); fills p.f's shared-memory offsets
int filtered_range_plan(const dab_index* idx, uint32_t l_search, uint32_t beam, int store, FilteredRangeParams& p,
                        WarpPlan<FilteredRangeParams>& plan);

}  // namespace dab
