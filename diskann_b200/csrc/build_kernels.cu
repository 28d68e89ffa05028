// build_kernels.cu — build-side reuse of the distance path: robust_prune on the device and a
// batched Vamana construction (SURVEY.md §8f.2).
//
//   * robust_prune (diskann/src/graph/internal/prune.rs:106-259) runs one warp per pool: the
//     pool is sorted by (source distance, arrival order) in shared memory, the lazy
//     candidate x neighbour distances are data x data Distance<T,T> evaluations in the
//     reference's SIMD order (several neighbours gathered per pass, applied in order with the
//     reference's early break), PruneKind rules from graph/config/mod.rs:80-103.
//   * dab_build inserts points in batches (DiskANNIndex::multi_insert semantics,
//     diskann/src/graph/index.rs:815): the batch is searched against the current graph with
//     the search kernel recording the expanded nodes (VisitedSearchRecord, index.rs:276-282),
//     pruned (index.rs:2349-2380), and the back-edges are grouped by destination (stable radix
//     sort, cub) and applied one at a time per destination exactly like add_edge_and_prune
//     (index.rs:2264-2341) -> robust_prune_list (index.rs:2397-2454).
#include "dab_common.cuh"
#include "distance_device.cuh"
#include "search_host.cuh"

#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cfloat>
#include <vector>

namespace dab {

constexpr int kPruneWarps = 4;
constexpr uint32_t kMaxOcclusion = 750;  // graph/config/defaults.rs:13
constexpr int kPairsPerPass = 4;         // neighbour rows gathered per pass

struct PruneSmem {
    uint32_t* ids;      // [P] candidate ids (sorted by distance)
    float* d;           // [P] source distances
    float* occl;        // [P] State::occlude_factor
    uint16_t* last;     // [P] State::last_checked
    uint16_t* nbr;      // [P] State::neighbor
    uint32_t* order;    // [P] sort tie-break (arrival order)
};

__device__ __forceinline__ PruneSmem carve(uint8_t* base, uint32_t P) {
    PruneSmem s;
    s.ids = reinterpret_cast<uint32_t*>(base);
    s.d = reinterpret_cast<float*>(base + 4 * (size_t)P);
    s.occl = reinterpret_cast<float*>(base + 8 * (size_t)P);
    s.order = reinterpret_cast<uint32_t*>(base + 12 * (size_t)P);
    s.last = reinterpret_cast<uint16_t*>(base + 16 * (size_t)P);
    s.nbr = reinterpret_cast<uint16_t*>(base + 18 * (size_t)P);
    return s;
}
__host__ __device__ inline size_t prune_smem_bytes(uint32_t P) { return 20 * (size_t)P; }

// PruneKind::update_occlude_factor, graph/config/mod.rs:80-103 (kind 0 triangle, 1 occluding)
__device__ __forceinline__ float update_occlude(int kind, float d_ik, float d_jk, float cur, float alpha) {
    if (kind == 0) {
        if (d_jk == 0.0f) return FLT_MAX;
        return fmaxf(cur, __fdiv_rn(d_ik, d_jk));
    }
    if (d_jk < __fmul_rn(alpha, d_ik)) return __fadd_rn(alpha, 0.01f);
    return cur;
}

// Bitonic sort of the first n (padded to pow2 P2 <= P) entries by (distance, arrival order):
// SortedNeighbors::new (graph/internal/sorted_neighbors.rs:26-44); ties are unspecified in the
// reference (unstable sort), this kernel breaks them by arrival order (as do the parity tests).
__device__ __forceinline__ void warp_sort_pool(PruneSmem s, uint32_t n, uint32_t P2, int lane, bool preset_order = false) {
    for (uint32_t i = n + lane; i < P2; i += 32) {
        s.d[i] = __int_as_float(0x7F800000);
        s.ids[i] = kNoId;
        s.order[i] = 0xFFFFFFFFu;
    }
    if (!preset_order)
        for (uint32_t i = lane; i < n; i += 32) s.order[i] = i;
    __syncwarp();
    for (uint32_t k = 2; k <= P2; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t t = lane; t < P2; t += 32) {
                const uint32_t o = t ^ j;
                if (o > t) {
                    const float da = s.d[t], db = s.d[o];
                    const uint32_t oa = s.order[t], ob = s.order[o];
                    const bool a_less = da < db || (da == db && oa < ob);
                    const bool asc = (t & k) == 0;
                    if (asc ? !a_less : a_less) {
                        const uint32_t ia = s.ids[t];
                        s.d[t] = db;
                        s.d[o] = da;
                        s.order[t] = ob;
                        s.order[o] = oa;
                        s.ids[t] = s.ids[o];
                        s.ids[o] = ia;
                    }
                }
            }
            __syncwarp();
        }
    }
}

// data x data distance between row a and up to G rows b[g]; returns post-op'ed values on all lanes
template <typename TD, int NA, int KIND, int POST, bool IS_INT, bool SIGNED>
__device__ __forceinline__ void warp_row_distances(const uint8_t* vectors, size_t row_stride, int dim, uint32_t a,
                                                   const uint32_t (&b)[kPairsPerPass], int lane, float (&out)[kPairsPerPass]) {
    if constexpr (IS_INT) {
        const uint8_t* q = vectors + (size_t)a * row_stride;
        const uint8_t* rows[kPairsPerPass];
#pragma unroll
        for (int g = 0; g < kPairsPerPass; ++g) rows[g] = vectors + (size_t)b[g] * row_stride;
        const int qq = KIND == KIND_IP ? 0 : warp_int_self<SIGNED>(q, dim, lane);
        float r[kPairsPerPass];
        warp_int_multi<SIGNED, KIND, kPairsPerPass>(q, rows, dim, lane, qq, r);
#pragma unroll
        for (int g = 0; g < kPairsPerPass; ++g) out[g] = post_op<POST>(r[g]);
    } else {
        constexpr int S = 8 * NA, TEAMS = 32 / S;
        constexpr int U = kPairsPerPass / TEAMS;
        const int team = lane / S, slot = lane % S;
        const TD* q = reinterpret_cast<const TD*>(vectors + (size_t)a * row_stride);
        const TD* rows[U];
#pragma unroll
        for (int u = 0; u < U; ++u) rows[u] = reinterpret_cast<const TD*>(vectors + (size_t)b[u * TEAMS + team] * row_stride);
        float r[U];
        team_float_multi<NA, KIND, U>(q, rows, dim, slot, r);
#pragma unroll
        for (int u = 0; u < U; ++u) {
#pragma unroll
            for (int t = 0; t < TEAMS; ++t) out[u * TEAMS + t] = post_op<POST>(__shfl_sync(kFull, r[u], t * S));
        }
    }
}

// robust_prune over the sorted pool in shared memory (prune.rs:106-259); returns `found`,
// selected pool positions in s.nbr[0..found).
template <typename TD, int NA, int KIND, int POST, bool IS_INT, bool SIGNED>
__device__ __forceinline__ uint32_t warp_robust_prune(PruneSmem s, uint32_t n, uint32_t location, uint32_t degree, float alpha,
                                                      int prune_kind, const uint8_t* vectors, size_t row_stride, int dim,
                                                      int lane) {
    for (uint32_t i = lane; i < n; i += 32) {
        s.occl[i] = 0.0f;
        s.last[i] = 0;
        s.nbr[i] = 0;
    }
    __syncwarp();
    uint32_t found = 0;
    float current_alpha = 1.0f;
    const float increment = fminf(alpha, 1.2f);
    while (found < degree) {
        for (uint32_t i = 0; i < n; ++i) {
            if (found >= degree) break;
            float of = s.occl[i];
            uint32_t lc = s.last[i];
            if (of > current_alpha) continue;
            const uint32_t cand = s.ids[i];
            if (cand == location) {  // sorted_cache entry None (index.rs:2608-2614)
                __syncwarp();
                if (lane == 0) s.occl[i] = FLT_MAX;
                __syncwarp();
                continue;
            }
            const float d_ik = s.d[i];
            while (lc != found) {
                // gather the next neighbours that actually need a distance
                uint32_t rows[kPairsPerPass], rpos[kPairsPerPass];
                int cnt = 0;
#pragma unroll
                for (int g = 0; g < kPairsPerPass; ++g) {
                    rpos[g] = lc + g < found ? s.nbr[lc + g] : 0xFFFFFFFFu;
                    const bool need = rpos[g] != 0xFFFFFFFFu && rpos[g] < i;
                    rows[g] = need ? s.ids[rpos[g]] : cand;
                    cnt += rpos[g] != 0xFFFFFFFFu;
                }
                float dist[kPairsPerPass];
                warp_row_distances<TD, NA, KIND, POST, IS_INT, SIGNED>(vectors, row_stride, dim, cand, rows, lane, dist);
                bool stop = false;
#pragma unroll
                for (int g = 0; g < kPairsPerPass; ++g) {
                    if (g < cnt && !stop) {
                        ++lc;
                        if (rpos[g] < i) {
                            of = update_occlude(prune_kind, d_ik, dist[g], of, current_alpha);
                            if (of > current_alpha) stop = true;
                        }
                    }
                }
                if (stop) break;
            }
            __syncwarp();
            if (lane == 0) {
                s.last[i] = (uint16_t)lc;
                if (of > current_alpha) {
                    s.occl[i] = of;
                } else {
                    s.occl[i] = FLT_MAX;
                    s.nbr[found] = (uint16_t)i;
                }
            }
            __syncwarp();
            if (!(of > current_alpha)) ++found;
        }
        if (current_alpha == alpha) break;
        current_alpha = fminf(__fmul_rn(current_alpha, increment), alpha);
    }
    return found;
}

struct PruneParams {
    const uint8_t* vectors;
    size_t row_stride;
    int dim;
    uint32_t P;            // smem slots per warp (pow2)
    // pools
    const uint32_t* pool_ids;   // [n_pools][pool_cap]
    const float* pool_d;        // [n_pools][pool_cap]
    const uint32_t* pool_len;   // [n_pools]
    uint32_t pool_cap;
    const uint32_t* locations;  // [n_pools] id excluded from its own pool
    uint32_t n_pools;
    uint32_t degree;
    float alpha;
    int prune_kind;
    // outputs
    uint32_t* out_ids;          // [n_pools][degree]
    uint32_t* out_counts;       // [n_pools]
    uint32_t* adj;              // optional: also write adj[location] = [count, ids]
    uint32_t adj_stride;
};

template <typename TD, int NA, int KIND, int POST, bool IS_INT, bool SIGNED>
__global__ void __launch_bounds__(kPruneWarps * 32) prune_pools_kernel(const PruneParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    PruneSmem s = carve(smem + (size_t)wib * prune_smem_bytes(p.P), p.P);
    const uint32_t nwarps = gridDim.x * kPruneWarps;
    for (uint32_t w = blockIdx.x * kPruneWarps + wib; w < p.n_pools; w += nwarps) {
        uint32_t n = min(p.pool_len[w], p.pool_cap);
        __syncwarp();
        for (uint32_t i = lane; i < n; i += 32) {
            s.ids[i] = p.pool_ids[(size_t)w * p.pool_cap + i];
            s.d[i] = p.pool_d[(size_t)w * p.pool_cap + i];
        }
        uint32_t P2 = 1;
        while (P2 < n) P2 <<= 1;
        if (P2 < 2) P2 = 2;
        __syncwarp();
        warp_sort_pool(s, n, P2, lane);
        n = min(n, kMaxOcclusion);
        const uint32_t loc = p.locations[w];
        const uint32_t found = warp_robust_prune<TD, NA, KIND, POST, IS_INT, SIGNED>(s, n, loc, p.degree, p.alpha, p.prune_kind,
                                                                                     p.vectors, p.row_stride, p.dim, lane);
        __syncwarp();
        for (uint32_t f = lane; f < found; f += 32) {
            const uint32_t id = s.ids[s.nbr[f]];
            if (p.out_ids) p.out_ids[(size_t)w * p.degree + f] = id;
            if (p.adj) p.adj[(size_t)loc * p.adj_stride + 1 + f] = id;
        }
        if (lane == 0) {
            if (p.out_counts) p.out_counts[w] = found;
            if (p.adj) p.adj[(size_t)loc * p.adj_stride] = found;
        }
    }
}

// ------------------------------------------------------------------ back-edges
// this lane's share of: src is kNoId (no target) or appears in vals[start, e)
__device__ __forceinline__ bool segment_repeats(const uint32_t* vals, uint32_t start, uint32_t e, uint32_t src, int lane) {
    bool hit = src == kNoId;
    for (uint32_t f = start + lane; f < e; f += 32) hit |= vals[f] == src;
    return hit;
}

// id in the ascending a[0, n)
__device__ __forceinline__ bool sorted_contains(const uint32_t* a, uint32_t n, uint32_t id) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(a + mid) < id)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo < n && __ldg(a + lo) == id;
}

struct BackedgeParams {
    const uint8_t* vectors;
    size_t row_stride;
    int dim;
    uint32_t P;
    const uint32_t* keys;   // sorted destinations (kNoId = padding)
    const uint32_t* vals;   // sources
    uint32_t n_pairs;
    uint32_t degree, max_degree;
    float alpha;
    int prune_kind;
    uint32_t* adj;
    uint32_t adj_stride;
    // in-place deletes (inplace_backedge_kernel): the ids every visited list loses, ascending
    const uint32_t* remove;
    uint32_t n_remove;
    uint64_t n_total;  // ids at or above it have no row: left out of a prune pool
};

__global__ void make_pairs_kernel(const uint32_t* __restrict__ batch_ids, const uint32_t* __restrict__ nbr_ids,
                                  const uint32_t* __restrict__ nbr_counts, uint32_t n_batch, uint32_t degree,
                                  uint32_t max_backedges, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const uint32_t total = n_batch * degree;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const uint32_t b = i / degree, j = i % degree;
        const bool ok = j < nbr_counts[b] && j < max_backedges;
        keys[i] = ok ? nbr_ids[i] : kNoId;
        vals[i] = batch_ids[b];
    }
}

// One warp per destination segment: add_edge_and_prune (index.rs:2264-2341) with all the incoming
// edges of the batch at once; on overflow robust_prune_list (index.rs:2397-2454).
// REMOVE (in-place deletes): the segment's key is add_edge_and_prune's `source` and its values are the targets, in the
// order they are appended; the ids of p.remove are first taken out of the list (to_remove), a list that lost one is
// written even when nothing is added, a target already appended earlier in the segment is not appended again
// (extend_from_slice), a value kNoId only makes the source visited, and a stray id (>= n_total) in an overflowing list
// is left out of the prune pool.
template <typename TD, int NA, int KIND, int POST, bool IS_INT, bool SIGNED, bool REMOVE>
__device__ __forceinline__ void backedge_segments(const BackedgeParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    uint8_t* base = smem + (size_t)wib * (prune_smem_bytes(p.P) + 4 * (size_t)p.P);
    PruneSmem s = carve(base, p.P);
    uint32_t* list = reinterpret_cast<uint32_t*>(base + prune_smem_bytes(p.P));
    const uint32_t nwarps = gridDim.x * kPruneWarps;
    const uint32_t nchunks = (p.n_pairs + 31) / 32;
    for (uint32_t c = blockIdx.x * kPruneWarps + wib; c < nchunks; c += nwarps) {
        const uint32_t i = c * 32 + lane;
        const uint32_t key = i < p.n_pairs ? p.keys[i] : kNoId;
        const uint32_t prev = (i > 0 && i < p.n_pairs) ? p.keys[i - 1] : kNoId;
        unsigned heads = __ballot_sync(kFull, key != kNoId && (i == 0 || prev != key));
        while (heads) {
            const int hl = __ffs(heads) - 1;
            heads &= heads - 1;
            const uint32_t start = c * 32 + hl;
            const uint32_t q = __shfl_sync(kFull, key, hl);
            uint32_t* row = p.adj + (size_t)q * p.adj_stride;
            uint32_t deg = min(row[0], p.max_degree);
            __syncwarp();
            for (uint32_t t = lane; t < deg; t += 32) list[t] = row[1 + t];
            __syncwarp();
            bool did_remove = false;
            if constexpr (REMOVE) {
                uint32_t kept = 0;
                for (uint32_t c0 = 0; c0 < deg; c0 += 32) {
                    const uint32_t id = c0 + lane < deg ? list[c0 + lane] : kNoId;
                    const bool keep = c0 + lane < deg && !sorted_contains(p.remove, p.n_remove, id);
                    const unsigned m = __ballot_sync(kFull, keep);
                    __syncwarp();
                    if (keep) list[kept + __popc(m & ((1u << lane) - 1u))] = id;
                    __syncwarp();
                    kept += __popc(m);
                }
                did_remove = kept != deg;
                deg = kept;
            }
            // add_edge_and_prune(sorted sources, q) (index.rs:2264-2341, called once per target by
            // multi_insert, index.rs:986-1003): extend_from_slice appends every source that is not yet
            // in the list (sources arrive in ascending id order: the radix sort is stable and the
            // pairs are generated in batch order); if the extended list still fits it is kept,
            // otherwise robust_prune_list (index.rs:2397-2454) runs ONCE over all of it: pool =
            // (id, Distance(q, id)) for id in list, id != q, sorted by distance and cut to the 750
            // closest (SortedNeighbors::new).  A hub can receive thousands of in-edges from one large
            // batch, so the pool is streamed: whenever its P slots are full it is sorted by
            // (distance, arrival index) and cut to 750 — the same 750 a single sort would keep.
            const uint32_t deg0 = deg;
            uint32_t n_new = 0;
            for (uint32_t e = start; e < p.n_pairs && p.keys[e] == q; ++e) {
                const uint32_t src = p.vals[e];
                if (src == q) continue;
                bool present = false;
                for (uint32_t t = lane; t < deg0; t += 32) present |= list[t] == src;
                if constexpr (REMOVE) present |= segment_repeats(p.vals, start, e, src, lane);
                if (!__any_sync(kFull, present)) ++n_new;
            }
            if (n_new == 0 && !did_remove) continue;
            bool changed = true;
            if (deg0 + n_new <= p.max_degree) {
                for (uint32_t e = start; e < p.n_pairs && p.keys[e] == q; ++e) {
                    const uint32_t src = p.vals[e];
                    if (src == q) continue;
                    bool present = false;
                    for (uint32_t t = lane; t < deg0; t += 32) present |= list[t] == src;
                    if constexpr (REMOVE) present |= segment_repeats(p.vals, start, e, src, lane);
                    if (__any_sync(kFull, present)) continue;
                    if (lane == 0) list[deg] = src;
                    ++deg;
                    __syncwarp();
                }
            } else {
                uint32_t n = 0, arrival = 0;
                uint32_t pend[kPairsPerPass];
                int npend = 0;
                auto flush = [&]() {  // distances of the pending ids, appended to the pool in order
                    if (npend == 0) return;
                    uint32_t rows[kPairsPerPass];
#pragma unroll
                    for (int g = 0; g < kPairsPerPass; ++g) rows[g] = pend[g < npend ? g : npend - 1];
                    float dist[kPairsPerPass];
                    warp_row_distances<TD, NA, KIND, POST, IS_INT, SIGNED>(p.vectors, p.row_stride, p.dim, q, rows, lane, dist);
#pragma unroll
                    for (int g = 0; g < kPairsPerPass; ++g) {
                        if (g < npend) {
                            if (n == p.P) {
                                __syncwarp();
                                warp_sort_pool(s, n, p.P, lane, true);
                                n = kMaxOcclusion;
                            }
                            if (lane == 0) {
                                s.ids[n] = rows[g];
                                s.d[n] = dist[g];
                                s.order[n] = arrival;
                            }
                            ++n;
                            ++arrival;
                        }
                    }
                    npend = 0;
                    __syncwarp();
                };
                for (uint32_t t = 0; t < deg0; ++t) {
                    const uint32_t id = list[t];
                    if (id == q) continue;
                    if constexpr (REMOVE)
                        if (id >= p.n_total) continue;  // a stray id: robust_prune_list's fill finds no row for it
                    pend[npend++] = id;
                    if (npend == kPairsPerPass) flush();
                }
                for (uint32_t e = start; e < p.n_pairs && p.keys[e] == q; ++e) {
                    const uint32_t src = p.vals[e];
                    if (src == q) continue;
                    bool present = false;
                    for (uint32_t t = lane; t < deg0; t += 32) present |= list[t] == src;
                    if constexpr (REMOVE) present |= segment_repeats(p.vals, start, e, src, lane);
                    if (__any_sync(kFull, present)) continue;
                    pend[npend++] = src;
                    if (npend == kPairsPerPass) flush();
                }
                flush();
                uint32_t P2 = 2;
                while (P2 < n) P2 <<= 1;
                warp_sort_pool(s, n, P2, lane, true);
                n = min(n, kMaxOcclusion);
                const uint32_t found = warp_robust_prune<TD, NA, KIND, POST, IS_INT, SIGNED>(
                    s, n, q, p.degree, p.alpha, p.prune_kind, p.vectors, p.row_stride, p.dim, lane);
                __syncwarp();
                for (uint32_t f = lane; f < found; f += 32) list[f] = s.ids[s.nbr[f]];
                deg = found;
                __syncwarp();
            }
            if (changed) {
                for (uint32_t t = lane; t < deg; t += 32) row[1 + t] = list[t];
                if (lane == 0) row[0] = deg;
            }
            __syncwarp();
        }
    }
}

template <typename TD, int NA, int KIND, int POST, bool IS_INT, bool SIGNED>
__global__ void __launch_bounds__(kPruneWarps * 32) backedge_kernel(const BackedgeParams p) {
    backedge_segments<TD, NA, KIND, POST, IS_INT, SIGNED, false>(p);
}

template <typename TD, int NA, int KIND, int POST, bool IS_INT, bool SIGNED>
__global__ void __launch_bounds__(kPruneWarps * 32) inplace_backedge_kernel(const BackedgeParams p) {
    backedge_segments<TD, NA, KIND, POST, IS_INT, SIGNED, true>(p);
}

// ------------------------------------------------------------------ consolidation
// DiskANNIndex::consolidate_vector (index.rs:1819-1931) for every node at once.  Node v's new list depends only on v's
// list, the lists of its deleted neighbours and the deletion table, and no deleted node's list is ever written, so one
// pass in any order equals the reference's sequential loop; rows are rewritten in place.  One warp per node:
//   * a deleted v is left alone; a v with no deleted (or out-of-range) neighbour and at most `degree` distinct live
//     neighbours is left alone (lists no longer than `degree` skip the distinct count);
//   * the pool is a set in a canonical order: v's live neighbours in list order, then for each deleted neighbour in
//     list order its live neighbours in list order, first occurrence kept (the reference's HashSet leaves the order
//     unspecified).  An id >= n_total is a deleted neighbour with no neighbours.  Membership is a per-warp open-
//     addressing table in global memory, cleared after each node through the slots the pool recorded;
//   * v is then dropped; a pool of fewer than `degree` ids is the new list as it is, otherwise robust_prune_list
//     (index.rs:2397-2454): Distance<T,T>(v, u), sorted by (distance, arrival order) and cut to the 750 smallest —
//     streamed through the prune's shared-memory pool as in backedge_kernel, since a pool can hold
//     max_degree * (max_degree + 1) ids — then occlude_list without saturation.
// RANGE (prune_range_kernel): DiskANNIndex::prune_range (index.rs:2656-2700) over the nodes of p.ids (every id when
// NULL), each listed once.  The deletion table is not read (the full-precision PruneAccessor::fill finds a row for every
// id, deleted or not): a deleted node is pruned like any other and its deleted neighbours stay in its pool.  A node whose
// list holds at most `degree` ids is left alone; any other list goes through robust_prune_list with the pool of its
// distinct ids, itself and the ids >= n_total (no row: view.get finds nothing) left out, however short that pool is.
// Each prune reads only its own list and rows, so one pass equals the reference's loop.
constexpr uint32_t kConsolidateP = 1024;  // shared-memory pool slots per warp (> kMaxOcclusion)

struct ConsolidateParams {
    const uint8_t* vectors;
    size_t row_stride;
    int dim;
    uint32_t* adj;
    uint32_t adj_stride, max_degree;
    uint64_t n_points, n_total;
    const uint32_t* deleted;  // NULL: nothing deleted
    uint32_t degree;
    float alpha;
    int prune_kind;
    uint32_t* hash;  // per warp: 1 << hash_bits ids, kNoId = empty
    int hash_bits;
    uint32_t* pool;       // per warp: pool_cap ids
    uint32_t* pool_slot;  // per warp: the hash slot of each pool id
    uint32_t pool_cap;
    uint32_t* counters;  // [0] next node, [1] lists rewritten
};

struct PruneRangeParams : ConsolidateParams {
    const uint32_t* ids;  // the nodes to prune, n_ids of them (NULL: ids [0, n_ids))
    uint32_t n_ids;
};

template <typename TD, int NA, int KIND, int POST, bool IS_INT, bool SIGNED, bool RANGE, class Params>
__device__ __forceinline__ void consolidate_nodes(const Params p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    PruneSmem s = carve(smem + (size_t)wib * prune_smem_bytes(kConsolidateP), kConsolidateP);
    const uint32_t warp = blockIdx.x * kPruneWarps + wib;
    const uint32_t hmask = (1u << p.hash_bits) - 1u;
    uint32_t* hash = p.hash + ((size_t)warp << p.hash_bits);
    uint32_t* pool = p.pool + (size_t)warp * p.pool_cap;
    uint32_t* pslot = p.pool_slot + (size_t)warp * p.pool_cap;
    auto dead = [&](uint32_t id) {  // deleted, or a status lookup that fails; RANGE: no row
        return id >= p.n_total || (!RANGE && p.deleted && (__ldg(p.deleted + (id >> 5)) >> (id & 31) & 1u));
    };
    uint32_t n = 0;  // pool size
    // every lane calls; `want`: this lane offers `id`.  New ids are appended in lane order; among lanes offering the
    // same id the first one inserts it.
    auto add = [&](uint32_t id, bool want) {
        const unsigned peers = __match_any_sync(kFull, want ? id : kNoId);
        uint32_t slot = kNoId;
        if (want && __ffs(peers) - 1 == lane) {
            uint32_t h = (id * 0x9E3779B1u) >> (32 - p.hash_bits);
            for (;;) {
                const uint32_t old = atomicCAS(hash + h, kNoId, id);
                if (old == kNoId) {
                    slot = h;
                    break;
                }
                if (old == id) break;
                h = (h + 1) & hmask;
            }
        }
        const unsigned mn = __ballot_sync(kFull, slot != kNoId);
        if (slot != kNoId) {
            const uint32_t pos = n + __popc(mn & ((1u << lane) - 1u));
            pool[pos] = id;
            pslot[pos] = slot;
        }
        n += __popc(mn);
    };
    for (;;) {
        uint32_t v = 0;
        if (lane == 0) v = atomicAdd(p.counters, 1u);
        v = __shfl_sync(kFull, v, 0);
        if constexpr (RANGE) {
            if (v >= p.n_ids) break;
            if (p.ids) v = p.ids[v];
        } else {
            if (v >= p.n_total) break;
            if (dead(v)) continue;  // ConsolidateKind::Deleted
        }
        uint32_t* row = p.adj + (size_t)v * p.adj_stride;
        const uint32_t deg = min(row[0], p.max_degree);
        bool any_dead = false;
        if constexpr (!RANGE) {
            for (uint32_t j = lane; j < deg; j += 32) any_dead |= dead(row[1 + j]);
            any_dead = __any_sync(kFull, any_dead);
        }
        if (!any_dead && deg <= p.degree) continue;
        n = 0;
        for (uint32_t c = 0; c < deg; c += 32) {
            const uint32_t j = c + lane;
            const uint32_t id = j < deg ? row[1 + j] : kNoId;
            add(id, j < deg && !dead(id));
        }
        // the early exit counts a self-loop
        if (RANGE || any_dead || n > p.degree) {
            if constexpr (!RANGE) {  // the deleted neighbours' lists join the pool
                for (uint32_t c = 0; c < deg; c += 32) {
                    const uint32_t j = c + lane;
                    const uint32_t id = j < deg ? row[1 + j] : kNoId;
                    unsigned dm = __ballot_sync(kFull, j < deg && dead(id));
                    while (dm) {
                        const int src = __ffs(dm) - 1;
                        dm &= dm - 1;
                        const uint32_t u = __shfl_sync(kFull, id, src);
                        if (u >= p.n_total) continue;
                        const uint32_t* urow = p.adj + (size_t)u * p.adj_stride;
                        const uint32_t udeg = min(urow[0], p.max_degree);
                        for (uint32_t c2 = 0; c2 < udeg; c2 += 32) {
                            const uint32_t j2 = c2 + lane;
                            const uint32_t w = j2 < udeg ? urow[1 + j2] : kNoId;
                            add(w, j2 < udeg && !dead(w));
                        }
                    }
                }
            }
            // drop v (a self-loop): its table slot is cleared and the pool after it moves down one place
            uint32_t pv = kNoId;
            for (uint32_t c = 0; c < n; c += 32) {
                const unsigned m = __ballot_sync(kFull, c + lane < n && pool[c + lane] == v);
                if (m) pv = c + __ffs(m) - 1;
            }
            if (pv != kNoId) {
                if (lane == 0) hash[pslot[pv]] = kNoId;
                for (uint32_t c = pv; c + 1 < n; c += 32) {
                    const uint32_t j = c + lane;
                    uint32_t id = 0, slot = 0;
                    if (j + 1 < n) id = pool[j + 1], slot = pslot[j + 1];
                    __syncwarp();
                    if (j + 1 < n) pool[j] = id, pslot[j] = slot;
                    __syncwarp();
                }
                --n;
            }
            if (!RANGE && n < p.degree) {
                for (uint32_t j = lane; j < n; j += 32) row[1 + j] = pool[j];
                if (lane == 0) row[0] = n;
            } else {
                // Distance<T,T>(v, u) for the pool in arrival order, streamed into the shared pool: whenever its slots
                // are full it is sorted by (distance, arrival) and cut to 750, which keeps what one sort would keep
                uint32_t ns = 0;
                for (uint32_t j0 = 0; j0 < n; j0 += kPairsPerPass) {
                    const uint32_t cnt = min(n - j0, (uint32_t)kPairsPerPass);
                    uint32_t rows[kPairsPerPass];
#pragma unroll
                    for (int g = 0; g < kPairsPerPass; ++g) rows[g] = pool[j0 + min((uint32_t)g, cnt - 1)];
                    float dist[kPairsPerPass];
                    warp_row_distances<TD, NA, KIND, POST, IS_INT, SIGNED>(p.vectors, p.row_stride, p.dim, v, rows, lane, dist);
#pragma unroll
                    for (int g = 0; g < kPairsPerPass; ++g) {
                        if ((uint32_t)g < cnt) {
                            if (ns == kConsolidateP) {
                                __syncwarp();
                                warp_sort_pool(s, ns, kConsolidateP, lane, true);
                                ns = kMaxOcclusion;
                            }
                            if (lane == 0) {
                                s.ids[ns] = rows[g];
                                s.d[ns] = dist[g];
                                s.order[ns] = j0 + g;
                            }
                            ++ns;
                        }
                    }
                    __syncwarp();
                }
                uint32_t P2 = 2;
                while (P2 < ns) P2 <<= 1;
                warp_sort_pool(s, ns, P2, lane, true);
                ns = min(ns, kMaxOcclusion);
                const uint32_t found = warp_robust_prune<TD, NA, KIND, POST, IS_INT, SIGNED>(s, ns, v, p.degree, p.alpha, p.prune_kind,
                                                                                             p.vectors, p.row_stride, p.dim, lane);
                __syncwarp();
                for (uint32_t f = lane; f < found; f += 32) row[1 + f] = s.ids[s.nbr[f]];
                if (lane == 0) row[0] = found;
            }
            if (lane == 0) atomicAdd(p.counters + 1, 1u);
        }
        for (uint32_t j = lane; j < n; j += 32) hash[pslot[j]] = kNoId;
        __syncwarp();
    }
}

// 96 registers: below that ptxas spills the pool-building and prune state of the float schemas
template <typename TD, int NA, int KIND, int POST, bool IS_INT, bool SIGNED>
__global__ void __maxnreg__(96) consolidate_kernel(const ConsolidateParams p) {
    consolidate_nodes<TD, NA, KIND, POST, IS_INT, SIGNED, false>(p);
}

template <typename TD, int NA, int KIND, int POST, bool IS_INT, bool SIGNED>
__global__ void __maxnreg__(96) prune_range_kernel(const PruneRangeParams p) {
    consolidate_nodes<TD, NA, KIND, POST, IS_INT, SIGNED, true>(p);
}

// ------------------------------------------------------------------ in-place deletes
// inplace_delete_inner (index.rs:1585-1749) for every member of a chunk, one warp per member, on the graph as it was
// before the chunk, every member already deleted.  The member's replace candidates and in-neighbours (the three
// candidate routines, index.rs:1139-1336), then its scored edges as (source, target) pairs, member-major: each
// in-neighbour c's pairs (c, r) for the num_to_replace candidates r nearest to c, or one (c, kNoId) when there are none,
// then for each live neighbour a in list order the pairs (r, a) for the candidates r nearest to a.  Candidates are
// ordered by (Distance<T,T>, position in the replace candidates): warp_sort_pool with the positions as arrival order.
// An in-neighbour listed twice yields the same pairs twice, which add_edge_and_prune's extend_from_slice makes a
// no-op, as the reference's HashMap::insert replacing the entry with an equal one.  The count pass (keys NULL) writes
// each member's pair count without computing a distance; the write pass writes the pairs from offsets[w].
struct WorklistParams {
    const uint8_t* vectors;
    size_t row_stride;
    int dim;
    const uint32_t* adj;
    uint32_t adj_stride, max_degree;
    uint64_t n_total;
    const uint32_t* deleted;  // the table, the chunk's members marked
    const uint32_t* members;
    uint32_t n_members;
    int method;
    uint32_t num_to_replace, k_value;
    const uint32_t* topk;    // VisitedAndTopK: each member's filtered search list [n_members][topk_cap], topk_n long
    const uint32_t* topk_n;
    uint32_t topk_cap;
    uint32_t P;  // shared-memory pool slots per warp: a power of two >= the longest replace-candidate list
    // per warp: the member's live neighbours [max_degree], in-neighbours [inn_cap]; TwoHopAndOneHop: the two-hop set
    // [cand_cap] with the table slot of each id, and an open-addressing table of 1 << hash_bits ids (kNoId = empty)
    uint32_t *onehop, *inn, *cand, *cand_slot, *hash;
    uint32_t inn_cap, cand_cap;
    int hash_bits;
    uint32_t* counts;          // count pass: [n_members] pairs
    const uint32_t* offsets;   // write pass: [n_members] first pair
    uint32_t *keys, *vals;     // write pass: sources, targets
};

template <typename TD, int NA, int KIND, int POST, bool IS_INT, bool SIGNED>
__global__ void __launch_bounds__(kPruneWarps * 32) inplace_worklist_kernel(const WorklistParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    PruneSmem s = carve(smem + (size_t)wib * prune_smem_bytes(p.P), p.P);
    const uint32_t warp = blockIdx.x * kPruneWarps + wib, nwarps = gridDim.x * kPruneWarps;
    uint32_t* onehop = p.onehop + (size_t)warp * p.max_degree;
    uint32_t* inn = p.inn + (size_t)warp * p.inn_cap;
    uint32_t* cand = p.cand + (size_t)warp * p.cand_cap;
    uint32_t* cslot = p.cand_slot + (size_t)warp * p.cand_cap;
    uint32_t* hash = p.hash + ((size_t)warp << p.hash_bits);
    const uint32_t hmask = (1u << p.hash_bits) - 1u;
    const bool write = p.keys != nullptr;
    auto dead = [&](uint32_t id) { return id >= p.n_total || (__ldg(p.deleted + (id >> 5)) >> (id & 31) & 1u); };
    // every lane calls: the ids of the lanes with `want` go to out[n..] in lane order
    auto append = [&](uint32_t* out, uint32_t& n, uint32_t id, bool want) {
        const unsigned m = __ballot_sync(kFull, want);
        if (want) out[n + __popc(m & ((1u << lane) - 1u))] = id;
        n += __popc(m);
    };
    for (uint32_t w = warp; w < p.n_members; w += nwarps) {
        const uint32_t m = p.members[w];
        const uint32_t* mrow = p.adj + (size_t)m * p.adj_stride;
        const uint32_t mdeg = min(mrow[0], p.max_degree);
        uint32_t n1 = 0;  // live neighbours, list order (get_undeleted_neighbors)
        for (uint32_t c0 = 0; c0 < mdeg; c0 += 32) {
            const uint32_t id = c0 + lane < mdeg ? mrow[1 + c0 + lane] : kNoId;
            append(onehop, n1, id, c0 + lane < mdeg && !dead(id));
        }
        __syncwarp();
        const uint32_t *rc = onehop, *cands = onehop;  // replace candidates; the ids whose lists may hold m
        uint32_t nrc = n1, ncand = n1;
        if (p.method == DAB_INPLACE_VISITED_AND_TOPK) {
            cands = rc = p.topk + (size_t)w * p.topk_cap;
            ncand = p.topk_n[w];
            nrc = min(ncand, p.k_value);
        } else if (p.method == DAB_INPLACE_TWO_HOP_AND_ONE_HOP) {
            // the live ids of {one-hop} and their neighbours, first occurrence kept
            ncand = 0;
            auto add = [&](uint32_t id, bool want) {
                const unsigned peers = __match_any_sync(kFull, want ? id : kNoId);
                uint32_t slot = kNoId;
                if (want && __ffs(peers) - 1 == lane) {
                    uint32_t h = (id * 0x9E3779B1u) >> (32 - p.hash_bits);
                    for (;;) {
                        const uint32_t old = atomicCAS(hash + h, kNoId, id);
                        if (old == kNoId) {
                            slot = h;
                            break;
                        }
                        if (old == id) break;
                        h = (h + 1) & hmask;
                    }
                }
                const unsigned mn = __ballot_sync(kFull, slot != kNoId);
                if (slot != kNoId) {
                    const uint32_t pos = ncand + __popc(mn & ((1u << lane) - 1u));
                    cand[pos] = id;
                    cslot[pos] = slot;
                }
                ncand += __popc(mn);
            };
            for (uint32_t c0 = 0; c0 < n1; c0 += 32) add(c0 + lane < n1 ? onehop[c0 + lane] : kNoId, c0 + lane < n1);
            for (uint32_t i = 0; i < n1; ++i) {
                const uint32_t* r = p.adj + (size_t)onehop[i] * p.adj_stride;
                const uint32_t deg = min(r[0], p.max_degree);
                for (uint32_t c0 = 0; c0 < deg; c0 += 32) {
                    const uint32_t id = c0 + lane < deg ? r[1 + c0 + lane] : kNoId;
                    add(id, c0 + lane < deg && !dead(id));
                }
            }
            __syncwarp();
            cands = cand;
        }
        // in-neighbours: the candidates whose list holds m (return_refs_to_deleted_vertex)
        uint32_t nin = 0;
        for (uint32_t i = 0; i < ncand; ++i) {
            const uint32_t c = cands[i];
            const uint32_t* r = p.adj + (size_t)c * p.adj_stride;
            const uint32_t deg = min(r[0], p.max_degree);
            bool hit = false;
            for (uint32_t j = lane; j < deg; j += 32) hit |= r[1 + j] == m;
            if (__any_sync(kFull, hit)) {
                if (lane == 0) inn[nin] = c;
                ++nin;
            }
        }
        if (p.method == DAB_INPLACE_TWO_HOP_AND_ONE_HOP)
            for (uint32_t j = lane; j < ncand; j += 32) hash[cslot[j]] = kNoId;
        __syncwarp();
        // the scored edges of every in-neighbour, then of every live neighbour
        uint32_t npairs = 0;
        uint32_t* keys = write ? p.keys + p.offsets[w] : nullptr;
        uint32_t* vals = write ? p.vals + p.offsets[w] : nullptr;
        for (uint32_t j = 0; j < nin + n1; ++j) {
            const bool in = j < nin;
            const uint32_t x = in ? inn[j] : onehop[j - nin];
            uint32_t self = 0;
            for (uint32_t c0 = 0; c0 < nrc; c0 += 32) self += __popc(__ballot_sync(kFull, c0 + lane < nrc && rc[c0 + lane] == x));
            const uint32_t take = min(p.num_to_replace, nrc - self);
            if (write && take > 0) {
                uint32_t n = 0;
                for (uint32_t i0 = 0; i0 < nrc; i0 += kPairsPerPass) {
                    const uint32_t cnt = min(nrc - i0, (uint32_t)kPairsPerPass);
                    uint32_t rows[kPairsPerPass];
#pragma unroll
                    for (int g = 0; g < kPairsPerPass; ++g) rows[g] = rc[i0 + min((uint32_t)g, cnt - 1)];
                    float dist[kPairsPerPass];
                    warp_row_distances<TD, NA, KIND, POST, IS_INT, SIGNED>(p.vectors, p.row_stride, p.dim, x, rows, lane, dist);
#pragma unroll
                    for (int g = 0; g < kPairsPerPass; ++g) {
                        if ((uint32_t)g < cnt && rows[g] != x) {
                            if (lane == 0) {
                                s.ids[n] = rows[g];
                                s.d[n] = dist[g];
                                s.order[n] = i0 + g;
                            }
                            ++n;
                        }
                    }
                }
                __syncwarp();
                uint32_t P2 = 2;
                while (P2 < n) P2 <<= 1;
                warp_sort_pool(s, n, P2, lane, true);
                for (uint32_t t = lane; t < take; t += 32) {
                    keys[npairs + t] = in ? x : s.ids[t];
                    vals[npairs + t] = in ? s.ids[t] : x;
                }
                __syncwarp();
            }
            if (in && take == 0 && write && lane == 0) {  // edges[c] is set, empty
                keys[npairs] = x;
                vals[npairs] = kNoId;
            }
            npairs += in ? max(take, 1u) : take;
        }
        if (!write && lane == 0) p.counts[w] = npairs;
    }
}

__global__ void iota_kernel(uint32_t* p, uint32_t first, uint32_t n) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) p[i] = first + i;
}

// ------------------------------------------------------------------ host dispatch
static uint32_t pow2_at_least(uint32_t v) {
    uint32_t p = 2;
    while (p < v) p <<= 1;
    return p;
}

static int launch_prune(const dab_index* idx, PruneParams& p) {
    p.vectors = idx->d_vectors;
    p.row_stride = idx->row_stride;
    p.dim = (int)idx->dim;
    p.prune_kind = idx->metric == DAB_INNER_PRODUCT ? 1 : 0;  // PruneKind::from_metric, config/mod.rs:69-76
    p.P = pow2_at_least(std::max<uint32_t>(p.pool_cap, 2));
    const size_t smem = prune_smem_bytes(p.P) * kPruneWarps;
    if (smem > 200 * 1024) return fail(DAB_ERR_INVALID_ARGUMENT, "prune: pool capacity %u too large", p.pool_cap);
    const int grid = (int)std::min<uint64_t>(((uint64_t)p.n_pools + kPruneWarps - 1) / kPruneWarps, (uint64_t)idx->sm_count * 8);
    const int rc = visit_schema<OPS_ROW>(idx->dtype, idx->metric, [&](auto s) -> int {
        using S = decltype(s);
        auto kern = prune_pools_kernel<KernelRow<S>, S::NA, S::KIND, S::POST, S::IS_INT, S::SIGNED>;
        DAB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, kPruneWarps * 32, smem, idx->stream>>>(p);
        return DAB_OK;
    });
    if (rc) return rc;
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    return DAB_OK;
}

// `remove`: inplace_backedge_kernel, with p.remove set
static int launch_backedges(const dab_index* idx, BackedgeParams& p, bool remove = false) {
    p.vectors = idx->d_vectors;
    p.row_stride = idx->row_stride;
    p.dim = (int)idx->dim;
    p.prune_kind = idx->metric == DAB_INNER_PRODUCT ? 1 : 0;
    // the list of a destination holds its current neighbours plus every in-edge of the batch
    p.P = std::max<uint32_t>(1024, pow2_at_least(idx->max_degree + 2));
    p.adj = idx->d_adj;
    p.adj_stride = idx->adj_stride;
    p.max_degree = idx->max_degree;
    const size_t smem = (prune_smem_bytes(p.P) + 4 * (size_t)p.P) * kPruneWarps;
    if (smem > 200 * 1024) return fail(DAB_ERR_INVALID_ARGUMENT, "build: max_degree %u too large", idx->max_degree);
    const uint32_t chunks = (p.n_pairs + 31) / 32;
    const int grid = (int)std::min<uint64_t>(((uint64_t)chunks + kPruneWarps - 1) / kPruneWarps, (uint64_t)idx->sm_count * 8);
    const int rc = visit_schema<OPS_ROW>(idx->dtype, idx->metric, [&](auto s) -> int {
        using S = decltype(s);
        auto kern = remove ? inplace_backedge_kernel<KernelRow<S>, S::NA, S::KIND, S::POST, S::IS_INT, S::SIGNED>
                           : backedge_kernel<KernelRow<S>, S::NA, S::KIND, S::POST, S::IS_INT, S::SIGNED>;
        DAB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, kPruneWarps * 32, smem, idx->stream>>>(p);
        return DAB_OK;
    });
    if (rc) return rc;
    DAB_LAUNCHED();
    DAB_CUDA(cudaGetLastError());
    return DAB_OK;
}

// One multi_insert (index.rs:815-1030, intra_batch_candidates = None, no bootstrap) over the ids in `batch`, on the graph
// the previous step left; dab_build and dab_insert run their batches through it.
//   1. every member is searched against the graph as it was before the step (beam 1, l_build), recording the nodes it
//      expanded (VisitedSearchRecord, index.rs:276-282; the record is sized generously and a search that still outgrows
//      it is counted in rec_truncated);
//   2. each member's record is pruned to pruned_degree (index.rs:2349-2380) and its out-list written;
//   3. the back-edges are grouped by target (aggregate_backedges, index.rs:123-143; stable radix sort) and each target
//      gets one add_edge_and_prune (index.rs:2264-2341) with max_backedges = pruned_degree.
// backedge_kernel takes a target's sources in the order the pairs arrive, and add_edge_and_prune takes them sorted
// (index.rs:986-992): the ids in `batch` must be ascending.  Steps 1 and 2 do not depend on the members' order.
struct LinkStep {
    DevBuf batch, rec_ids, rec_d, rec_n, nbr, nbr_n, keys, vals, keys2, vals2, tmp, res_ids, res_d;
    size_t tmp_bytes = 0;
    uint32_t rec_cap = 0, pruned_degree = 0, l_build = 0;
    float alpha = 0.0f;

    // buffers for steps of up to `cap` ids
    int alloc(dab_index* idx, uint32_t cap, uint32_t pruned_degree_, uint32_t l_build_, float alpha_) {
        pruned_degree = pruned_degree_, l_build = l_build_, alpha = alpha_;
        rec_cap = std::min<uint32_t>(2048, 4 * l_build + 64);
        idx->rec_truncated = 0;
        int rc;
        const size_t B = cap;
        if ((rc = batch.alloc(B * 4)) || (rc = rec_ids.alloc(B * rec_cap * 4)) || (rc = rec_d.alloc(B * rec_cap * 4)) ||
            (rc = rec_n.alloc(B * 4)) || (rc = nbr.alloc(B * pruned_degree * 4)) || (rc = nbr_n.alloc(B * 4)) ||
            (rc = keys.alloc(B * pruned_degree * 4)) || (rc = vals.alloc(B * pruned_degree * 4)) ||
            (rc = keys2.alloc(B * pruned_degree * 4)) || (rc = vals2.alloc(B * pruned_degree * 4)) || (rc = res_ids.alloc(B * 4)) ||
            (rc = res_d.alloc(B * 4)))
            return rc;
        cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, (const uint32_t*)keys.p, (uint32_t*)keys2.p, (const uint32_t*)vals.p,
                                        (uint32_t*)vals2.p, (int)(B * pruned_degree), 0, 32, idx->stream);
        return tmp.alloc(tmp_bytes);
    }

    // one step over batch[0, b)
    int run(dab_index* idx, uint32_t b) {
        cudaStream_t st = idx->stream;
        int rc;
        const SearchRecord rec{(const uint32_t*)batch.p, (uint32_t*)rec_ids.p, (float*)rec_d.p, (uint32_t*)rec_n.p, rec_cap};
        // 1. search the batch against the current graph, recording expanded nodes
        if ((rc = run_search(idx, nullptr, b, 1, l_build, 1, SearchOut{(uint32_t*)res_ids.p, (float*)res_d.p, nullptr, nullptr, nullptr},
                             -1, false, &rec)))
            return rc;
        // 2. robust_prune each point's visited pool -> out-edges
        PruneParams pp;
        memset(&pp, 0, sizeof(pp));
        pp.pool_ids = (const uint32_t*)rec_ids.p;
        pp.pool_d = (const float*)rec_d.p;
        pp.pool_len = (const uint32_t*)rec_n.p;
        pp.pool_cap = rec_cap;
        pp.locations = (const uint32_t*)batch.p;
        pp.n_pools = b;
        pp.degree = pruned_degree;
        pp.alpha = alpha;
        pp.out_ids = (uint32_t*)nbr.p;
        pp.out_counts = (uint32_t*)nbr_n.p;
        pp.adj = idx->d_adj;
        pp.adj_stride = idx->adj_stride;
        if ((rc = launch_prune(idx, pp))) return rc;
        // 3. back-edges grouped by destination
        const uint32_t n_pairs = b * pruned_degree;
        make_pairs_kernel<<<(n_pairs + 255) / 256, 256, 0, st>>>((const uint32_t*)batch.p, (const uint32_t*)nbr.p, (const uint32_t*)nbr_n.p, b,
                                                                 pruned_degree, pruned_degree, (uint32_t*)keys.p, (uint32_t*)vals.p);
        DAB_LAUNCHED();
        cudaError_t e = cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, (const uint32_t*)keys.p, (uint32_t*)keys2.p, (const uint32_t*)vals.p,
                                                        (uint32_t*)vals2.p, (int)n_pairs, 0, 32, st);
        if (e != cudaSuccess) return fail(DAB_ERR_CUDA, "build: radix sort failed: %s", cudaGetErrorString(e));
        DAB_LAUNCHED();
        BackedgeParams bp;
        memset(&bp, 0, sizeof(bp));
        bp.keys = (const uint32_t*)keys2.p;
        bp.vals = (const uint32_t*)vals2.p;
        bp.n_pairs = n_pairs;
        bp.degree = pruned_degree;
        bp.alpha = alpha;
        return launch_backedges(idx, bp);
    }

    // after the last step: truncated records, reported under `who`
    int report(dab_index* idx, const char* who) {
        DAB_CUDA(cudaStreamSynchronize(idx->stream));
        if (idx->rec_truncated)
            return fail(DAB_ERR_INVALID_ARGUMENT, "%s: %llu insert searches expanded more than %u nodes; their prune pools were cut "
                        "(the graph is usable but not the reference's)", who, (unsigned long long)idx->rec_truncated, rec_cap);
        return DAB_OK;
    }
};

// The work-list kernel's shared-memory pool slots per warp: a power of two >= the longest replace-candidate list
static uint32_t inplace_pool_slots(const dab_index* idx, int method, uint32_t k_value, uint32_t l_value) {
    uint32_t longest = idx->max_degree;
    if (method == DAB_INPLACE_VISITED_AND_TOPK) longest = std::max(longest, std::min(k_value, l_value));
    return pow2_at_least(std::max<uint32_t>(longest, 2));
}

// Whether the work-list and apply kernels' shared memory fits one CTA (checked before anything is changed)
static bool inplace_fits(const dab_index* idx, int method, uint32_t k_value, uint32_t l_value) {
    const uint32_t pb = std::max<uint32_t>(1024, pow2_at_least(idx->max_degree + 2));  // launch_backedges' pool
    return prune_smem_bytes(inplace_pool_slots(idx, method, k_value, l_value)) * kPruneWarps <= 200 * 1024 &&
           (prune_smem_bytes(pb) + 4 * (size_t)pb) * kPruneWarps <= 200 * 1024;
}

// Grows `b` to at least `bytes` (contents not kept)
static int grow(DevBuf& b, size_t& have, size_t bytes) {
    if (bytes <= have) return DAB_OK;
    have = bytes;
    return b.alloc(bytes);
}

// One chunk of multi_inplace_delete; `chunk` holds its ids in the caller's order, already marked deleted
struct InplaceDelete {
    int method;
    uint32_t num_to_replace, k_value, l_value, pruned_degree;
    float alpha;
    DevBuf members, sorted, lists, topk, topk_n, scratch, counts, offsets, keys, vals, keys2, vals2, tmp;
    size_t cap_members = 0, cap_sorted = 0, cap_lists = 0, cap_topk = 0, cap_topk_n = 0, cap_scratch = 0, cap_counts = 0,
           cap_offsets = 0, cap_keys = 0, cap_vals = 0, cap_keys2 = 0, cap_vals2 = 0, cap_tmp = 0;

    int run(dab_index* idx, const uint32_t* chunk, uint32_t b) {
        cudaStream_t st = idx->stream;
        int rc;
        if ((rc = grow(members, cap_members, (size_t)b * 4)) || (rc = grow(sorted, cap_sorted, (size_t)b * 4)) ||
            (rc = grow(counts, cap_counts, (size_t)b * 4)) || (rc = grow(offsets, cap_offsets, (size_t)b * 4)))
            return rc;
        std::vector<uint32_t> ascending(chunk, chunk + b);
        std::sort(ascending.begin(), ascending.end());
        DAB_CUDA(cudaMemcpyAsync(members.p, chunk, (size_t)b * 4, cudaMemcpyHostToDevice, st));
        DAB_CUDA(cudaMemcpyAsync(sorted.p, ascending.data(), (size_t)b * 4, cudaMemcpyHostToDevice, st));
        WorklistParams p;
        memset(&p, 0, sizeof(p));
        p.vectors = idx->d_vectors;
        p.row_stride = idx->row_stride;
        p.dim = (int)idx->dim;
        p.adj = idx->d_adj;
        p.adj_stride = idx->adj_stride;
        p.max_degree = idx->max_degree;
        p.n_total = idx->n_total();
        p.deleted = idx->d_deleted;
        p.members = (const uint32_t*)members.p;
        p.n_members = b;
        p.method = method;
        p.num_to_replace = num_to_replace;
        p.k_value = k_value;
        p.P = inplace_pool_slots(idx, method, k_value, l_value);
        p.inn_cap = idx->max_degree;
        if (method == DAB_INPLACE_VISITED_AND_TOPK) {
            // search_internal from each member's row, beam 1, L = l_value, start points kept; then the first l_value
            // entries that are not deleted (RemoveDeletedIdsAndCopy, which keeps start points)
            const uint32_t cap = l_value + idx->n_start;
            if ((rc = grow(lists, cap_lists, (size_t)b * cap * 8)) || (rc = grow(topk, cap_topk, (size_t)b * l_value * 8)) ||
                (rc = grow(topk_n, cap_topk_n, (size_t)b * 4)))
                return rc;
            uint32_t* l_ids = (uint32_t*)lists.p;
            float* l_d = (float*)(l_ids + (size_t)b * cap);
            SearchRecord rec{};
            rec.query_rows = (const uint32_t*)members.p;
            rec.keep_starts = true;
            if ((rc = run_search(idx, nullptr, b, cap, l_value, 1, SearchOut{l_ids, l_d, nullptr, nullptr, nullptr}, -1, false, &rec)))
                return rc;
            uint32_t* t_ids = (uint32_t*)topk.p;
            if ((rc = queue_drop_deleted(idx, st, idx->d_deleted, l_ids, l_d, cap, b, l_value,
                                         SearchOut{t_ids, (float*)(t_ids + (size_t)b * l_value), (uint32_t*)topk_n.p, nullptr, nullptr},
                                         idx->n_total())))
                return rc;
            p.topk = t_ids;
            p.topk_n = (const uint32_t*)topk_n.p;
            p.topk_cap = l_value;
            p.inn_cap = std::max(p.inn_cap, l_value);
        }
        if (method == DAB_INPLACE_TWO_HOP_AND_ONE_HOP) {
            // distinct ids: the live neighbours and theirs, never more than the index holds
            p.cand_cap = (uint32_t)std::min<uint64_t>(idx->n_total(), (uint64_t)idx->max_degree * (idx->max_degree + 1));
            p.hash_bits = 5;
            while ((1ull << p.hash_bits) < 2ull * p.cand_cap) ++p.hash_bits;  // at most half full
            p.inn_cap = std::max(p.inn_cap, p.cand_cap);
        }
        const size_t smem = prune_smem_bytes(p.P) * kPruneWarps;
        const size_t warp_words = (size_t)idx->max_degree + p.inn_cap + 2ull * p.cand_cap + (p.cand_cap ? 1ull << p.hash_bits : 0);
        rc = visit_schema<OPS_ROW>(idx->dtype, idx->metric, [&](auto sch) -> int {
            using S = decltype(sch);
            auto kern = inplace_worklist_kernel<KernelRow<S>, S::NA, S::KIND, S::POST, S::IS_INT, S::SIGNED>;
            const int per_sm = ctas_per_sm(kern, kPruneWarps * 32, smem);
            if (per_sm < 1) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_inplace_delete: the work-list kernel does not fit");
            // every resident warp, within 2 GB of per-warp lists and tables
            uint64_t blocks = (uint64_t)per_sm * idx->sm_count;
            blocks = std::max<uint64_t>(1, std::min<uint64_t>(blocks, (2ull << 30) / (warp_words * 4 * kPruneWarps)));
            blocks = std::min<uint64_t>(blocks, ((uint64_t)b + kPruneWarps - 1) / kPruneWarps);
            const size_t warps = blocks * kPruneWarps;
            int rc2;
            if ((rc2 = grow(scratch, cap_scratch, warps * warp_words * 4))) return rc2;
            p.onehop = (uint32_t*)scratch.p;
            p.inn = p.onehop + warps * idx->max_degree;
            p.cand = p.inn + warps * p.inn_cap;
            p.cand_slot = p.cand + warps * p.cand_cap;
            p.hash = p.cand_slot + warps * p.cand_cap;
            if (p.cand_cap) DAB_CUDA(cudaMemsetAsync(p.hash, 0xFF, (warps << p.hash_bits) * 4, st));
            // count pass, offsets, write pass
            p.counts = (uint32_t*)counts.p;
            kern<<<(int)blocks, kPruneWarps * 32, smem, st>>>(p);
            DAB_LAUNCHED();
            DAB_CUDA(cudaGetLastError());
            std::vector<uint32_t> n_of(b), first(b);
            DAB_CUDA(cudaMemcpyAsync(n_of.data(), counts.p, (size_t)b * 4, cudaMemcpyDeviceToHost, st));
            DAB_CUDA(cudaStreamSynchronize(st));
            uint64_t total = 0;
            for (uint32_t i = 0; i < b; ++i) {
                first[i] = (uint32_t)total;
                total += n_of[i];
            }
            if (total >= 0x7FFFFFFFull) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_inplace_delete: %llu edges in one chunk (use a smaller batch_size)",
                                                    (unsigned long long)total);
            n_pairs = (uint32_t)total;
            if (n_pairs == 0) return DAB_OK;
            if ((rc2 = grow(keys, cap_keys, total * 4)) || (rc2 = grow(vals, cap_vals, total * 4)) ||
                (rc2 = grow(keys2, cap_keys2, total * 4)) || (rc2 = grow(vals2, cap_vals2, total * 4)))
                return rc2;
            DAB_CUDA(cudaMemcpyAsync(offsets.p, first.data(), (size_t)b * 4, cudaMemcpyHostToDevice, st));
            p.counts = nullptr;
            p.offsets = (const uint32_t*)offsets.p;
            p.keys = (uint32_t*)keys.p;
            p.vals = (uint32_t*)vals.p;
            kern<<<(int)blocks, kPruneWarps * 32, smem, st>>>(p);
            DAB_LAUNCHED();
            DAB_CUDA(cudaGetLastError());
            return DAB_OK;
        });
        if (rc) return rc;
        if (n_pairs) {
            // the targets of each source in the members' order (a stable sort), then one add_edge_and_prune per source
            size_t need = 0;
            cub::DeviceRadixSort::SortPairs(nullptr, need, (const uint32_t*)keys.p, (uint32_t*)keys2.p, (const uint32_t*)vals.p,
                                            (uint32_t*)vals2.p, (int)n_pairs, 0, 32, st);
            if ((rc = grow(tmp, cap_tmp, need))) return rc;
            cudaError_t e = cub::DeviceRadixSort::SortPairs(tmp.p, need, (const uint32_t*)keys.p, (uint32_t*)keys2.p, (const uint32_t*)vals.p,
                                                            (uint32_t*)vals2.p, (int)n_pairs, 0, 32, st);
            if (e != cudaSuccess) return fail(DAB_ERR_CUDA, "dab_inplace_delete: radix sort failed: %s", cudaGetErrorString(e));
            DAB_LAUNCHED();
            BackedgeParams bp;
            memset(&bp, 0, sizeof(bp));
            bp.keys = (const uint32_t*)keys2.p;
            bp.vals = (const uint32_t*)vals2.p;
            bp.n_pairs = n_pairs;
            bp.degree = pruned_degree;
            bp.alpha = alpha;
            bp.remove = (const uint32_t*)sorted.p;
            bp.n_remove = b;
            bp.n_total = idx->n_total();
            if ((rc = launch_backedges(idx, bp, true))) return rc;
        }
        // drop_adj_list of every member
        if ((rc = clear_rows(idx, (const uint32_t*)members.p, b))) return rc;
        DAB_CUDA(cudaStreamSynchronize(st));
        return DAB_OK;
    }
    uint32_t n_pairs = 0;
};

}  // namespace dab

using namespace dab;

extern "C" {

// PruneAccessor::fill + robust_prune over caller-provided pools (unsorted).  Exposed for the
// prune parity tests and for host-driven builds.
int dab_robust_prune(dab_index* idx, const uint32_t* pool_ids, const float* pool_dists, const uint32_t* pool_lens,
                     const uint32_t* locations, uint32_t n_pools, uint32_t pool_cap, uint32_t degree, float alpha,
                     uint32_t* out_ids, uint32_t* out_counts) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_robust_prune: idx is NULL");
    if (!idx->vectors_ready) return fail(DAB_ERR_NOT_READY, "dab_robust_prune: vectors not uploaded");
    if (n_pools == 0) return DAB_OK;
    if (!pool_ids || !pool_dists || !pool_lens || !locations || !out_ids || !out_counts)
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_robust_prune: NULL argument");
    // launch_prune holds a whole pool in shared memory: 20 bytes a slot, four warps a CTA, at most 200 KB
    if (degree == 0 || pool_cap == 0 || pool_cap > 2048)
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_robust_prune: degree must be > 0 and pool_cap in [1, 2048]");
    DAB_CUDA(cudaSetDevice(idx->device));
    DevBuf b_ids, b_d, b_len, b_loc, b_out, b_cnt;
    int rc;
    const size_t np = n_pools, pc = pool_cap;
    if ((rc = b_ids.alloc(np * pc * 4)) || (rc = b_d.alloc(np * pc * 4)) || (rc = b_len.alloc(np * 4)) || (rc = b_loc.alloc(np * 4)) ||
        (rc = b_out.alloc(np * degree * 4)) || (rc = b_cnt.alloc(np * 4)))
        return rc;
    DAB_CUDA(cudaMemcpyAsync(b_ids.p, pool_ids, np * pc * 4, cudaMemcpyHostToDevice, idx->stream));
    DAB_CUDA(cudaMemcpyAsync(b_d.p, pool_dists, np * pc * 4, cudaMemcpyHostToDevice, idx->stream));
    DAB_CUDA(cudaMemcpyAsync(b_len.p, pool_lens, np * 4, cudaMemcpyHostToDevice, idx->stream));
    DAB_CUDA(cudaMemcpyAsync(b_loc.p, locations, np * 4, cudaMemcpyHostToDevice, idx->stream));
    DAB_CUDA(cudaMemsetAsync(b_out.p, 0xFF, np * degree * 4, idx->stream));
    PruneParams p;
    memset(&p, 0, sizeof(p));
    p.pool_ids = (const uint32_t*)b_ids.p;
    p.pool_d = (const float*)b_d.p;
    p.pool_len = (const uint32_t*)b_len.p;
    p.pool_cap = pool_cap;
    p.locations = (const uint32_t*)b_loc.p;
    p.n_pools = n_pools;
    p.degree = degree;
    p.alpha = alpha;
    p.out_ids = (uint32_t*)b_out.p;
    p.out_counts = (uint32_t*)b_cnt.p;
    if ((rc = launch_prune(idx, p))) return rc;
    DAB_CUDA(cudaMemcpyAsync(out_ids, b_out.p, np * degree * 4, cudaMemcpyDeviceToHost, idx->stream));
    DAB_CUDA(cudaMemcpyAsync(out_counts, b_cnt.p, np * 4, cudaMemcpyDeviceToHost, idx->stream));
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    return DAB_OK;
}

int dab_consolidate(dab_index* idx, uint32_t pruned_degree, float alpha, uint64_t* out_rewritten) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_consolidate: idx is NULL");
    int rc;
    if ((rc = refuse_in_flight(idx, "dab_consolidate"))) return rc;
    if (!idx->vectors_ready || !idx->graph_ready) return fail(DAB_ERR_NOT_READY, "dab_consolidate: vectors and graph must be uploaded first");
    if (pruned_degree == 0 || pruned_degree > idx->max_degree)
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_consolidate: pruned_degree must be in [1, max_degree]");
    if (!(alpha >= 1.0f)) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_consolidate: alpha must be >= 1");
    DAB_CUDA(cudaSetDevice(idx->device));
    ConsolidateParams p;
    memset(&p, 0, sizeof(p));
    p.vectors = idx->d_vectors;
    p.row_stride = idx->row_stride;
    p.dim = (int)idx->dim;
    p.adj = idx->d_adj;
    p.adj_stride = idx->adj_stride;
    p.max_degree = idx->max_degree;
    p.n_points = idx->n_points;
    p.n_total = idx->n_total();
    p.deleted = deleted_filter(idx);
    p.degree = pruned_degree;
    p.alpha = alpha;
    p.prune_kind = idx->metric == DAB_INNER_PRODUCT ? 1 : 0;  // PruneKind::from_metric, config/mod.rs:69-76
    // a pool holds distinct ids: at most max_degree live neighbours plus max_degree per deleted one, and n_total
    p.pool_cap = (uint32_t)std::min<uint64_t>(idx->n_total(), (uint64_t)idx->max_degree * (idx->max_degree + 1));
    p.hash_bits = 5;
    while ((1ull << p.hash_bits) < 2ull * p.pool_cap) ++p.hash_bits;  // at most half full
    const size_t warp_bytes = ((1ull << p.hash_bits) + 2ull * p.pool_cap) * 4;
    const size_t smem = prune_smem_bytes(kConsolidateP) * kPruneWarps;
    DevBuf b_scratch, b_counters;
    uint32_t counters[2] = {0, 0};
    rc = visit_schema<OPS_ROW>(idx->dtype, idx->metric, [&](auto s) -> int {
        using S = decltype(s);
        auto kern = consolidate_kernel<KernelRow<S>, S::NA, S::KIND, S::POST, S::IS_INT, S::SIGNED>;
        const int per_sm = ctas_per_sm(kern, kPruneWarps * 32, smem);
        // every resident warp, within 2 GB of tables and pools
        uint64_t blocks = std::max(1, per_sm) * (uint64_t)idx->sm_count;
        blocks = std::max<uint64_t>(1, std::min<uint64_t>(blocks, (2ull << 30) / (warp_bytes * kPruneWarps)));
        blocks = std::min<uint64_t>(blocks, (idx->n_total() + kPruneWarps - 1) / kPruneWarps);
        int rc2;
        if ((rc2 = b_scratch.alloc(blocks * kPruneWarps * warp_bytes)) || (rc2 = b_counters.alloc(8))) return rc2;
        p.hash = (uint32_t*)b_scratch.p;
        p.pool = p.hash + (blocks * kPruneWarps << p.hash_bits);
        p.pool_slot = p.pool + blocks * kPruneWarps * p.pool_cap;
        p.counters = (uint32_t*)b_counters.p;
        DAB_CUDA(cudaMemsetAsync(p.hash, 0xFF, (blocks * kPruneWarps << p.hash_bits) * 4, idx->stream));
        DAB_CUDA(cudaMemsetAsync(p.counters, 0, 8, idx->stream));
        kern<<<(int)blocks, kPruneWarps * 32, smem, idx->stream>>>(p);
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
        DAB_CUDA(cudaMemcpyAsync(counters, p.counters, 8, cudaMemcpyDeviceToHost, idx->stream));
        DAB_CUDA(cudaStreamSynchronize(idx->stream));
        return DAB_OK;
    });
    if (rc) return rc;
    if (counters[1]) ++idx->generation;  // adjacency rows were written: open paged sessions fail their next page
    if (out_rewritten) *out_rewritten = counters[1];
    return DAB_OK;
}

int dab_prune_range(dab_index* idx, const uint32_t* ids, uint64_t n, uint32_t pruned_degree, float alpha, uint64_t* out_rewritten) {
    static const char* who = "dab_prune_range";
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", who);
    if (!ids && n) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: ids is NULL with n > 0", who);
    int rc;
    if ((rc = refuse_in_flight(idx, who))) return rc;
    if (!idx->vectors_ready || !idx->graph_ready) return fail(DAB_ERR_NOT_READY, "%s: vectors and graph must be uploaded first", who);
    if (pruned_degree == 0 || pruned_degree > idx->max_degree)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: pruned_degree must be in [1, max_degree]", who);
    if (!(alpha >= 1.0f)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: alpha must be >= 1", who);
    // each id once, in first-occurrence order: a repeat is a no-op in the reference, and two warps must not share a row
    std::vector<uint32_t> distinct;
    if (ids) {
        std::vector<uint32_t> seen(idx->deleted_words(), 0u);
        for (uint64_t i = 0; i < n; ++i) {
            const uint32_t id = ids[i];
            if (id >= idx->n_total())
                return fail(DAB_ERR_INVALID_ARGUMENT, "%s: id %u out of range (%llu ids)", who, id, (unsigned long long)idx->n_total());
            if (seen[id >> 5] >> (id & 31) & 1u) continue;
            seen[id >> 5] |= 1u << (id & 31);
            distinct.push_back(id);
        }
    }
    const uint64_t n_ids = ids ? distinct.size() : idx->n_total();
    if (out_rewritten) *out_rewritten = 0;
    if (n_ids == 0) return DAB_OK;
    DAB_CUDA(cudaSetDevice(idx->device));
    PruneRangeParams p;
    memset(&p, 0, sizeof(p));
    p.vectors = idx->d_vectors;
    p.row_stride = idx->row_stride;
    p.dim = (int)idx->dim;
    p.adj = idx->d_adj;
    p.adj_stride = idx->adj_stride;
    p.max_degree = idx->max_degree;
    p.n_points = idx->n_points;
    p.n_total = idx->n_total();
    p.degree = pruned_degree;
    p.alpha = alpha;
    p.prune_kind = idx->metric == DAB_INNER_PRODUCT ? 1 : 0;  // PruneKind::from_metric, config/mod.rs:69-76
    p.pool_cap = (uint32_t)std::min<uint64_t>(idx->n_total(), idx->max_degree);  // the distinct ids of one list
    p.hash_bits = 5;
    while ((1ull << p.hash_bits) < 2ull * p.pool_cap) ++p.hash_bits;  // at most half full
    p.n_ids = (uint32_t)n_ids;
    const size_t warp_bytes = ((1ull << p.hash_bits) + 2ull * p.pool_cap) * 4;
    const size_t smem = prune_smem_bytes(kConsolidateP) * kPruneWarps;
    DevBuf b_ids, b_scratch, b_counters;
    if (ids) {
        if ((rc = b_ids.alloc(n_ids * 4))) return rc;
        DAB_CUDA(cudaMemcpyAsync(b_ids.p, distinct.data(), n_ids * 4, cudaMemcpyHostToDevice, idx->stream));
        p.ids = (const uint32_t*)b_ids.p;
    }
    uint32_t counters[2] = {0, 0};
    rc = visit_schema<OPS_ROW>(idx->dtype, idx->metric, [&](auto s) -> int {
        using S = decltype(s);
        auto kern = prune_range_kernel<KernelRow<S>, S::NA, S::KIND, S::POST, S::IS_INT, S::SIGNED>;
        const int per_sm = ctas_per_sm(kern, kPruneWarps * 32, smem);
        if (per_sm < 1) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: the prune kernel does not fit", who);
        uint64_t blocks = (uint64_t)per_sm * idx->sm_count;
        blocks = std::min<uint64_t>(blocks, (n_ids + kPruneWarps - 1) / kPruneWarps);
        int rc2;
        if ((rc2 = b_scratch.alloc(blocks * kPruneWarps * warp_bytes)) || (rc2 = b_counters.alloc(8))) return rc2;
        p.hash = (uint32_t*)b_scratch.p;
        p.pool = p.hash + (blocks * kPruneWarps << p.hash_bits);
        p.pool_slot = p.pool + blocks * kPruneWarps * p.pool_cap;
        p.counters = (uint32_t*)b_counters.p;
        DAB_CUDA(cudaMemsetAsync(p.hash, 0xFF, (blocks * kPruneWarps << p.hash_bits) * 4, idx->stream));
        DAB_CUDA(cudaMemsetAsync(p.counters, 0, 8, idx->stream));
        kern<<<(int)blocks, kPruneWarps * 32, smem, idx->stream>>>(p);
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
        DAB_CUDA(cudaMemcpyAsync(counters, p.counters, 8, cudaMemcpyDeviceToHost, idx->stream));
        DAB_CUDA(cudaStreamSynchronize(idx->stream));
        return DAB_OK;
    });
    if (rc) return rc;
    if (counters[1]) ++idx->generation;  // adjacency rows were written: open paged sessions fail their next page
    if (out_rewritten) *out_rewritten = counters[1];
    return DAB_OK;
}

int dab_inplace_delete(dab_index* idx, const uint32_t* ids, uint64_t n, int method, uint32_t num_to_replace, uint32_t k_value,
                       uint32_t l_value, uint32_t pruned_degree, float alpha, uint32_t batch_size) {
    static const char* who = "dab_inplace_delete";
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", who);
    if (n && !ids) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL argument", who);
    if (method != DAB_INPLACE_VISITED_AND_TOPK && method != DAB_INPLACE_TWO_HOP_AND_ONE_HOP && method != DAB_INPLACE_ONE_HOP)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: unknown method %d", who, method);
    if (pruned_degree == 0 || pruned_degree > idx->max_degree)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: pruned_degree must be in [1, max_degree]", who);
    if (!(alpha >= 1.0f)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: alpha must be >= 1", who);
    if (method == DAB_INPLACE_VISITED_AND_TOPK && (l_value == 0 || (uint64_t)l_value + idx->n_start > 1024))
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: l_value must be > 0 and l_value + #start <= 1024", who);
    int rc;
    if ((rc = refuse_in_flight(idx, who))) return rc;
    std::vector<uint32_t> seen((idx->n_points + 31) / 32, 0u);
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t id = ids[i];
        if (id >= idx->n_points)
            return fail(DAB_ERR_INVALID_ARGUMENT, "%s: id %u is not a data point (n_points %llu; start points cannot be deleted)", who, id,
                        (unsigned long long)idx->n_points);
        if (seen[id >> 5] >> (id & 31) & 1u) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: id %u is repeated", who, id);
        seen[id >> 5] |= 1u << (id & 31);
    }
    if (!idx->vectors_ready || !idx->graph_ready) return fail(DAB_ERR_NOT_READY, "%s: vectors and graph must be uploaded first", who);
    if (!inplace_fits(idx, method, k_value, l_value))
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: max_degree %u (or k_value) too large for the kernels' shared memory", who, idx->max_degree);
    if (n == 0) return DAB_OK;
    DAB_CUDA(cudaSetDevice(idx->device));
    const uint32_t cap = (uint32_t)std::min<uint64_t>(batch_size ? batch_size : n, n);
    InplaceDelete del;
    del.method = method;
    del.num_to_replace = num_to_replace;
    del.k_value = k_value;
    del.l_value = l_value;
    del.pruned_degree = pruned_degree;
    del.alpha = alpha;
    ++idx->generation;  // every chunk empties its members' lists: open paged sessions fail their next page
    for (uint64_t first = 0; first < n; first += cap) {
        const uint32_t b = (uint32_t)std::min<uint64_t>(cap, n - first);
        // every member is deleted before any list is read
        if ((rc = deleted_mark(idx, ids + first, b)) || (rc = del.run(idx, ids + first, b))) return rc;
    }
    return DAB_OK;
}

int dab_build(dab_index* idx, uint32_t pruned_degree, uint32_t l_build, float alpha, uint32_t batch_size) {
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_build: idx is NULL");
    if (!idx->vectors_ready) return fail(DAB_ERR_NOT_READY, "dab_build: vectors (including start rows) must be uploaded first");
    if (idx->n_start == 0) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_build: the index needs at least one start point");
    if (pruned_degree == 0 || pruned_degree > idx->max_degree)
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_build: pruned_degree must be in [1, max_degree]");
    if (l_build == 0) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_build: l_build must be > 0");
    if (!(alpha >= 1.0f)) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_build: alpha must be >= 1");
    DAB_CUDA(cudaSetDevice(idx->device));
    const uint32_t n = (uint32_t)idx->n_points;
    if (batch_size == 0) batch_size = std::max<uint32_t>(1024, std::min<uint32_t>(65536, n / 16));
    cudaStream_t st = idx->stream;

    DAB_CUDA(cudaMemsetAsync(idx->d_adj, 0, idx->n_total() * (size_t)idx->adj_stride * 4, st));
    idx->graph_ready = true;
    ++idx->generation;

    LinkStep step;
    int rc;
    if ((rc = step.alloc(idx, batch_size, pruned_degree, l_build, alpha))) return rc;
    uint32_t inserted = 0;
    while (inserted < n) {
        // batches grow with the graph so that early points are not all inserted blind
        uint32_t b = std::min<uint32_t>(batch_size, std::max<uint32_t>(1, inserted / 8));
        b = std::min(b, n - inserted);
        iota_kernel<<<(b + 255) / 256, 256, 0, st>>>((uint32_t*)step.batch.p, inserted, b);
        DAB_LAUNCHED();
        if ((rc = step.run(idx, b))) return rc;
        inserted += b;
    }
    return step.report(idx, "dab_build");
}

int dab_insert(dab_index* idx, const uint32_t* ids, const void* rows, uint64_t n, uint32_t pruned_degree, uint32_t l_build, float alpha,
               uint32_t batch_size) {
    static const char* who = "dab_insert";
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", who);
    if (n && (!ids || !rows)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: NULL argument", who);
    if (pruned_degree == 0 || pruned_degree > idx->max_degree)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: pruned_degree must be in [1, max_degree]", who);
    if (l_build == 0) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: l_build must be > 0", who);
    if (!(alpha >= 1.0f)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: alpha must be >= 1", who);
    int rc;
    if ((rc = refuse_in_flight(idx, who))) return rc;
    if ((rc = insert_check_ids(idx, ids, n, who))) return rc;
    if (!idx->vectors_ready) return fail(DAB_ERR_NOT_READY, "%s: vectors (including start rows) must be uploaded first", who);
    if (idx->n_start == 0) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: the index needs at least one start point", who);
    if (n == 0) return DAB_OK;
    DAB_CUDA(cudaSetDevice(idx->device));
    // set_element: the rows and every store that holds rows; nothing is written when an encoder's check fails
    if ((rc = insert_rows(idx, ids, rows, n, who))) return rc;
    cudaStream_t st = idx->stream;
    if (!idx->graph_ready) {  // never uploaded or built: start from empty adjacency, as dab_build does
        DAB_CUDA(cudaMemsetAsync(idx->d_adj, 0, idx->n_total() * (size_t)idx->adj_stride * 4, st));
        idx->graph_ready = true;
    }
    ++idx->generation;
    if (batch_size == 0) batch_size = 65536;  // the cap of dab_build's default batch size
    const uint32_t cap = (uint32_t)std::min<uint64_t>(batch_size, n);
    LinkStep step;
    if ((rc = step.alloc(idx, cap, pruned_degree, l_build, alpha))) return rc;
    // consecutive chunks in the caller's order, each one multi_insert; a chunk goes to the step sorted ascending
    std::vector<uint32_t> chunk;
    for (uint64_t first = 0; first < n; first += cap) {
        const uint32_t b = (uint32_t)std::min<uint64_t>(cap, n - first);
        chunk.assign(ids + first, ids + first + b);
        std::sort(chunk.begin(), chunk.end());
        DAB_CUDA(cudaMemcpyAsync(step.batch.p, chunk.data(), (size_t)b * 4, cudaMemcpyHostToDevice, st));
        if ((rc = step.run(idx, b))) return rc;
    }
    return step.report(idx, who);
}

}  // extern "C"
