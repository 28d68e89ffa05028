// search_filtered.cu — label-filtered batched search on the device: InlineFilterSearch::search (diskann/src/graph/search/
// inline_filter_search.rs:89-160), i.e. inline_filter_search_internal (:166-282) with its optional AdaptiveL, then the
// default post-processing of the first L matches; and the label table it reads (dab_upload_labels).
//
// One warp per query on global visited tables, over full-precision rows of every type and metric of the k-NN path
// (filtered_kernel; filtered_range_kernel for FilteredRange::search, _quant over a store) or the PQ, SQ and MinMax stores with the distances of their k-NN traversal and an optional
// full-precision rerank of the first L matches (filtered_kernel_quant).  The traversal is search_internal's: every
// evaluated neighbour enters the list, accepted or not.  Next to it the warp keeps, in shared memory:
//   the matched list  the accepted start points and neighbours, at most L of them, ordered by distance with a later
//                     match after an earlier one at an equal distance (-0.0 equal to +0.0, NaN after every number).
//                     That is a stable sort of all matches followed by take(L): the reference sorts with
//                     sort_unstable_by(fast_distance), which leaves the order of exactly equal distances (and of NaN)
//                     open, and this is the one place where the device fixes an order the reference leaves open.
// A candidate's label set is read (8 B) next to its visited probe, when it is collected.  Adaptive L: after the hop in
// which the evaluated neighbours reach `samples`, the list's capacity becomes the new L of the host's table (computed
// with the reference's f64 expression, never in device math) if that is above L; NeighborPriorityQueue::reconfigure
// (queue.rs:339-353) cuts a longer list, so a "grown" L below L + #start shortens it.  A query whose visited set outgrows
// its table is re-run from its start points by the job, and so takes the same decision again.
#include "dab_common.cuh"
#include "search_common.cuh"
#include "search_filtered.cuh"
#include "search_range.cuh"

#include <algorithm>
#include <cmath>

namespace dab {

namespace {

__device__ __forceinline__ bool label_accepts(uint64_t labels, uint64_t mask, uint32_t match_all) {
    const uint64_t x = labels & mask;
    return match_all ? x == mask : x != 0;
}

// The accepted ones among candidates c0 .. c0+m-1 (m <= 32; lane j owns candidate j) into the matched list of at most
// `cap` entries: a new entry goes after every entry of an equal key, old or new, and an entry pushed past cap is dropped.
// Old entries move right by #new(key < theirs); the list is walked in tiles of 32 from the top, as merge_round_chunked
// does, so no tile overwrites an entry a lower tile still has to read.
__device__ __forceinline__ void matched_merge(float* md, uint32_t* mi, uint32_t cap, uint32_t& size, const uint32_t* cid, const float* cd,
                                              const uint32_t* ca, uint32_t c0, uint32_t m, int lane) {
    const uint32_t j = (uint32_t)lane;
    const bool acc = j < m && ca[c0 + j];
    const float dj = acc ? cd[c0 + j] : 0.0f;
    const uint32_t kj = order_key(dj);
    const bool valid = acc && !(size == cap && kj >= order_key(md[cap - 1]));
    const unsigned vm = __ballot_sync(kFull, valid);
    if (!vm) return;
    uint32_t lo = 0, hi = size;  // upper bound among the old entries
    while (__any_sync(kFull, lo < hi)) {
        const uint32_t mid = (lo + hi) >> 1;
        if (lo < hi) {
            if (order_key(md[mid]) <= kj) lo = mid + 1;
            else hi = mid;
        }
    }
    uint32_t rn = 0;
    for (unsigned it = vm; it;) {
        const int i = __ffs(it) - 1;
        it &= it - 1;
        const uint32_t ki = __shfl_sync(kFull, kj, i);
        rn += (ki < kj || (ki == kj && (uint32_t)i < j)) ? 1u : 0u;
    }
    const uint32_t pos = lo + rn;
    const bool keep_new = valid && pos < cap;
    const uint32_t idj = valid ? cid[c0 + j] : 0;
    __syncwarp();
#pragma unroll 1
    for (uint32_t t = (size + 31) / 32; t-- > 0;) {
        const uint32_t e = t * 32 + lane;
        const float od = e < size ? md[e] : 0.0f;
        const uint32_t oi = e < size ? mi[e] : 0, ke = order_key(od);
        uint32_t sh = 0;
        for (unsigned it = vm; it;) {
            const int i = __ffs(it) - 1;
            it &= it - 1;
            sh += __shfl_sync(kFull, kj, i) < ke ? 1u : 0u;
        }
        __syncwarp();
        if (e < size && sh != 0 && e + sh < cap) md[e + sh] = od, mi[e + sh] = oi;
        __syncwarp();
    }
    if (keep_new) md[pos] = dj, mi[pos] = idj;
    size = min(cap, size + (uint32_t)__popc(vm));
    __syncwarp();
}

// The matched list of InlineFilterSearch: the first L matches, written as the query's results
struct MatchedTopL {
    static constexpr bool kRange = false;
};

// One warp's share of a pass.  Src is a distance source (search_source.cuh).
// LIST: with p.list_ids, the matched list of each query (start points included) is written for the rerank.  Sink: where
// the matches go, MatchedTopL or a sink with kRange (FilteredRangeSink), which sees every hop's candidates through
// matches() and finishes each query that did not overflow.
template <bool LIST, class Src, class Sink = MatchedTopL>
__device__ __forceinline__ void filtered_queries(const SearchParamsFiltered& p, uint8_t* base, int lane, Src& src, Sink* sink = nullptr) {
    const int wib = threadIdx.x >> 5;
    float* bd = reinterpret_cast<float*>(base + p.off_bd);
    uint32_t* bi = reinterpret_cast<uint32_t*>(base + p.off_bi);
    float* md = reinterpret_cast<float*>(base + p.off_md);
    uint32_t* mi = reinterpret_cast<uint32_t*>(base + p.off_mi);
    uint32_t* cid = reinterpret_cast<uint32_t*>(base + p.off_cid);
    float* cd = reinterpret_cast<float*>(base + p.off_cd);
    uint32_t* ca = reinterpret_cast<uint32_t*>(base + p.off_ca);
    uint32_t* beam_ids = reinterpret_cast<uint32_t*>(base + p.off_beam);
    const uint32_t nbk = p.n_buckets;
    uint32_t* table = p.tables + (size_t)(blockIdx.x * kFiltWarps + wib) * nbk * 8;
    const uint32_t hlimit = nbk * 7;  // 87.5 % load
    const uint64_t n_total = p.n_points + p.n_start;

    for (uint32_t qidx; next_query(p.counters, p.n_work, p.query_list, lane, qidx);) {
        __syncwarp();
        src.load(qidx);
        for (uint32_t i = lane; i < nbk; i += 32) store_empty_bucket(table + (size_t)i * 8);
        __syncwarp();
        src.prepare();
        const uint64_t mask = __ldg(p.masks + qidx);
        uint32_t cap = p.best_cap, size = 0, cursor = 0, msize = 0;
        uint32_t cmps = 0, hops = 0, nvisited = 0, sample_visited = 0, sample_matched = 0;
        bool adjusted = p.samples == 0, overflow = false;
        if constexpr (Sink::kRange) sink->begin();

        // the candidates cid[0..n) (with their decisions in ca) into the list and the matched list, in order
        auto insert_all = [&](uint32_t n) {
            for (uint32_t c0 = 0; c0 < n; c0 += 32) {
                const uint32_t m = min(32u, n - c0);
                merge_round_chunked<8>(bd, bi, cap, size, cursor, cid, cd, c0, m, lane);
                if constexpr (Sink::kRange) sink->matches(cid, cd, ca, c0, m);
                else matched_merge(md, mi, p.cap, msize, cid, cd, ca, c0, m, lane);
            }
        };

        // ---- start points (start_point_distances, provider.rs:406-433), in id order; they count in neither cmps nor
        // the sample
        for (uint32_t s0 = 0; s0 < p.n_start; s0 += 32) {
            const uint32_t n = min(32u, p.n_start - s0);
            if ((uint32_t)lane < n) {
                const uint32_t id = (uint32_t)p.n_points + s0 + lane;
                cid[lane] = id;
                ca[lane] = label_accepts(__ldg(p.labels + id), mask, p.match_all);
                visit_global(table, nbk, id);
            }
            __syncwarp();
            src.distances(cid, cd, n);
            insert_all(n);
            nvisited += n;
        }

        // ---- closest_notvisited x beam, expand_beam_filtered, every neighbour into the list and the accepted ones into
        // the matched list; then the adaptive-L decision of the hop
        for (;;) {
            const uint32_t nb = pick_beam(bi, size, p.beam, cursor, beam_ids, lane);
            if (nb == 0) break;
            uint32_t ncand = 0;
            for (uint32_t b = 0; b < nb; ++b) {
                const uint32_t* row = p.adj + (size_t)beam_ids[b] * p.adj_stride;
                const uint32_t deg = min(__ldg(row), p.max_degree);
                for (uint32_t c0 = 0; c0 < deg + 1; c0 += 32) {
                    const uint32_t j = c0 + lane;
                    const uint32_t word = j < p.adj_stride ? __ldg(row + j) : kEmptyV2;
                    const bool inserted = j >= 1 && j <= deg && visit_global(table, nbk, word);
                    const bool isnew = inserted && word < n_total;
                    const bool acc = isnew && label_accepts(__ldg(p.labels + word), mask, p.match_all);
                    const unsigned mn = __ballot_sync(kFull, isnew);
                    if (isnew) ca[ncand + __popc(mn & ((1u << lane) - 1u))] = acc;
                    push_new(inserted, isnew, word, cid, ncand, nvisited, lane);
                }
                if (nvisited + p.max_degree > hlimit) {
                    overflow = true;
                    break;
                }
            }
            if (overflow) break;
            __syncwarp();
            src.distances(cid, cd, ncand);
            insert_all(ncand);
            uint32_t matched = 0;
            for (uint32_t c = lane; c < ncand; c += 32) matched += ca[c];
            sample_matched += __reduce_add_sync(kFull, matched);
            sample_visited += ncand;
            cmps += ncand;
            hops += nb;
            if (!adjusted && sample_visited >= p.samples) {
                adjusted = true;
                const uint32_t new_l = p.adapt[(size_t)(sample_visited - p.samples) * (p.samples + p.span) + sample_matched];
                if (new_l > p.cap) {
                    // reconfigure(new_l): the capacity is new_l, a longer list is cut
                    cap = new_l;
                    size = min(size, new_l);
                    cursor = min(cursor, new_l);
                }
            }
        }

        if (overflow) {
            report_overflow(p.counters, p.overflow_list, qidx, lane);
            continue;
        }
        if constexpr (Sink::kRange) {
            sink->finish(qidx, bi, bd, size, mask, table, cmps, hops, nvisited);
        } else {
            if constexpr (LIST) {
                if (p.list_ids) write_list(mi, msize, p.list_ids, p.list_counts, p.list_cap, qidx, lane);
            }
            // post-processing of matched_results.take(L): start points dropped, the first k kept
            const uint32_t count = write_results(mi, md, msize, p.n_points, p.k, p.out_ids, p.out_dists, qidx, lane);
            write_stats(p.counters, nvisited, p.out_counts, p.out_cmps, p.out_hops, qidx, count, cmps, hops, lane);
        }
    }
}

template <typename TD, int KIND, int POST, int NA>
__global__ void __launch_bounds__(kFiltWarps * 32) filtered_kernel(const SearchParamsFiltered p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    uint8_t* base = smem + (size_t)wib * p.warp_smem;
    FullRowSource<TD, KIND, POST, NA, SearchParamsFiltered> src(p, base, lane);
    filtered_queries<false>(p, base, lane, src);
}

template <int MODE>
__global__ void __launch_bounds__(kFiltWarps * 32) filtered_kernel_quant(const SearchParamsFiltered p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    uint8_t* base = smem + (size_t)wib * p.warp_smem;
    StoreSource<MODE, SearchParamsFiltered> src(p, base, lane, blockIdx.x * kFiltWarps + wib);
    filtered_queries<true>(p, base, lane, src);
}

// ---- the filtered range search (FilteredRange::search, filtered_range_search.rs:119-248) ---------------------------
// 64-bit keys a[0, n), n a power of two, into ascending order: a bitonic network run by one warp in global memory
__device__ __forceinline__ void warp_sort_keys(unsigned long long* a, uint32_t n, int lane) {
    for (uint32_t k = 2; k <= n; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t i = lane; i < n; i += 32) {
                const uint32_t l = i ^ j;
                if (l > i) {
                    const unsigned long long x = a[i], y = a[l];
                    if ((x > y) == ((i & k) == 0)) a[i] = y, a[l] = x;
                }
            }
            __syncwarp();
        }
    }
}

__device__ __forceinline__ uint32_t pow2_at_least(uint32_t n) { return n <= 1 ? 1u : 1u << (32 - __clz(n - 1)); }

// The sink of filtered_queries for a filtered range search.  Phase 1 (the traversal at L + #start, no adaptive L) hands
// it every hop's candidates: the accepted ones within the radius are appended to the warp's region of matches, in
// evaluation order, start points first.  finish() then runs the rest of the query on the warp's frontier and key regions:
//   matched   the matches sorted by distance, stably (order_key: -0.0 equal to +0.0; the reference's sort_unstable_by
//             leaves exact ties open, the earlier match goes first as in InlineFilterSearch);
//   in_range  the list's first L entries within the radius and the matches, sorted by (distance, id), each id once;
//   round 2   iff |in_range| >= min_in_range and |matched| < max_returned: the visited table is cleared and seeded with
//             the in_range ids, which are also the FIFO frontier.  While it is not empty and |matched| < max_returned,
//             up to beam ids are popped and expanded one node at a time (expand_beam_filtered, the label read next to
//             the visited probe); every neighbour with d <= radius * range_slack is pushed onto the frontier, and the
//             accepted ones with d <= radius are appended to matched while it is below max_returned.  The cap does not
//             cut a hop short.  cmps and hops count both phases.
//   output    matched.take(max_returned) in order without start points, deleted ids and ids with d <= inner_radius;
//             without radius_filter (a store's call with rerank) only start points and deleted ids are dropped, and
//             range_rerank applies the inner radius to the full-precision distances.
// A full region of matches or frontier stops the query, which the job re-runs on regions four times larger.
template <class Src>
struct FilteredRangeSink {
    static constexpr bool kRange = true;
    const FilteredRangeParams& fp;
    Src& src;
    int lane;
    uint32_t *cid, *ca;  // the hop's candidates and their decisions (shared memory)
    float* cd;
    uint32_t* mid;  // the matches: region_cap ids, then dists
    float* md;
    uint32_t* fid;  // the frontier: front_cap ids, then dists (the sort's scratch)
    float* fd;
    unsigned long long* keys;
    uint64_t m;  // matches within the radius, counted past region_cap
    bool radius_filter;

    __device__ __forceinline__ FilteredRangeSink(const FilteredRangeParams& p, Src& s, uint8_t* base, int ln, size_t slot, bool rf)
        : fp(p), src(s), lane(ln), radius_filter(rf) {
        cid = reinterpret_cast<uint32_t*>(base + p.f.off_cid);
        cd = reinterpret_cast<float*>(base + p.f.off_cd);
        ca = reinterpret_cast<uint32_t*>(base + p.f.off_ca);
        mid = p.r.regions + slot * p.r.region_cap * 2;
        md = reinterpret_cast<float*>(mid + p.r.region_cap);
        fid = p.fronts + slot * p.front_cap * 2;
        fd = reinterpret_cast<float*>(fid + p.front_cap);
        keys = p.keys + slot * p.key_cap;
    }

    __device__ __forceinline__ void begin() { m = 0; }

    // the accepted candidates within the radius among c0 .. c0+n-1 (n <= 32, lane j owns candidate j), in order
    __device__ __forceinline__ void matches(const uint32_t* ids, const float* ds, const uint32_t* acc, uint32_t c0, uint32_t n) {
        const uint32_t j = (uint32_t)lane;
        const float d = j < n ? ds[c0 + j] : 0.0f;
        const bool ok = j < n && acc[c0 + j] && d <= fp.r.radius;
        const unsigned b = __ballot_sync(kFull, ok);
        const uint64_t at = m + __popc(b & ((1u << lane) - 1u));
        if (ok && at < fp.r.region_cap) mid[at] = ids[c0 + j], md[at] = d;
        m += __popc(b);
    }

    __device__ __forceinline__ void finish(uint32_t qidx, const uint32_t* bi, const float* bd, uint32_t size, uint64_t mask, uint32_t* table,
                                           uint32_t cmps, uint32_t hops, uint32_t nvisited) {
        const RangeParams& p = fp.r;
        const unsigned below = (1u << lane) - 1u;
        const uint32_t nbk = p.n_buckets, hlimit = nbk * 7;
        const uint64_t n_total = p.n_points + p.n_start;
        bool region_full = m > p.region_cap, overflow = region_full, second = false;
        uint32_t M = (uint32_t)m;
        if (!overflow) {
            __syncwarp();
            // ---- matched_results sorted by (distance, evaluation order)
            uint32_t n = pow2_at_least(M);
            for (uint32_t i = lane; i < n; i += 32) keys[i] = i < M ? (unsigned long long)order_key(md[i]) << 32 | i : ~0ull;
            __syncwarp();
            warp_sort_keys(keys, n, lane);
            for (uint32_t i = lane; i < M; i += 32) {
                const uint32_t s = (uint32_t)keys[i];
                fid[i] = mid[s], fd[i] = md[s];
            }
            __syncwarp();
            for (uint32_t i = lane; i < M; i += 32) mid[i] = fid[i], md[i] = fd[i];
            // ---- in_range: the list's first L entries within the radius and the matches, by (distance, id), deduplicated
            const uint32_t n1 = min(size, p.l_search);
            uint32_t t = 0;
            for (uint32_t b = 0; b < n1; b += 32) {
                const uint32_t i = b + lane;
                const float d = i < n1 ? bd[i] : 0.0f;
                const bool in = i < n1 && d <= p.radius;
                const unsigned bb = __ballot_sync(kFull, in);
                if (in) keys[t + __popc(bb & below)] = (unsigned long long)order_key(d) << 32 | (bi[i] & ~kFlagV2);  // expanded: flagged
                t += __popc(bb);
            }
            __syncwarp();
            for (uint32_t i = lane; i < M; i += 32) keys[t + i] = (unsigned long long)order_key(md[i]) << 32 | mid[i];
            const uint32_t T = t + M;
            n = pow2_at_least(T);
            for (uint32_t i = T + lane; i < n; i += 32) keys[i] = ~0ull;
            __syncwarp();
            warp_sort_keys(keys, n, lane);
            // an id in both sources has the same distance bits there, so its two keys are equal and adjacent
            uint32_t F = 0;
            for (uint32_t b = 0; b < T; b += 32) {
                const uint32_t i = b + lane;
                const bool first = i < T && (i == 0 || keys[i] != keys[i - 1]);
                const unsigned bb = __ballot_sync(kFull, first);
                if (first) fid[F + __popc(bb & below)] = (uint32_t)keys[i];
                F += __popc(bb);
            }
            __syncwarp();
            second = F >= p.min_in_range && M < p.max_returned;
            if (second) {
                // ---- filtered_range_search_internal
                for (uint32_t i = lane; i < nbk; i += 32) store_empty_bucket(table + (size_t)i * 8);
                __syncwarp();
                for (uint32_t i = lane; i < F; i += 32) visit_global(table, nbk, fid[i]);
                __syncwarp();  // every seed is in the table before any lane probes it for a neighbour
                nvisited = F;
                overflow = nvisited + p.max_degree > hlimit;
                uint32_t head = 0;
                while (!overflow && head < F && M < p.max_returned) {
                    const uint32_t nb = min(p.beam, F - head), f0 = head;
                    head += nb;
                    hops += nb;
                    for (uint32_t b = 0; b < nb && !overflow; ++b) {
                        uint32_t ncand = 0;
                        expand_node(p.adj, p.adj_stride, p.max_degree, n_total, table, nbk, fid[f0 + b], cid, ncand, nvisited, lane,
                                    [&](bool isnew, uint32_t word, uint32_t at) {
                                        const bool acc = isnew && label_accepts(__ldg(fp.f.labels + word), mask, fp.f.match_all);
                                        const unsigned mn = __ballot_sync(kFull, isnew);
                                        if (isnew) ca[at + __popc(mn & below)] = acc;
                                    });
                        if (nvisited + p.max_degree > hlimit) {
                            overflow = true;
                            break;
                        }
                        __syncwarp();
                        src.distances(cid, cd, ncand);
                        cmps += ncand;
                        // every neighbour within the navigation radius onto the frontier; the accepted ones within the
                        // radius into matched while it is below max_returned
                        for (uint32_t c0 = 0; c0 < ncand; c0 += 32) {
                            const uint32_t c = c0 + lane;
                            const float d = c < ncand ? cd[c] : 0.0f;
                            const bool nav = c < ncand && d <= p.bound;
                            const bool acc = nav && d <= p.radius && ca[c];
                            const unsigned bn = __ballot_sync(kFull, nav), ba = __ballot_sync(kFull, acc);
                            const uint32_t take = (uint32_t)min((unsigned long long)__popc(ba), (unsigned long long)(p.max_returned - M));
                            if (F + __popc(bn) > fp.front_cap || M + take > p.region_cap) {
                                region_full = overflow = true;
                                break;
                            }
                            if (nav) fid[F + __popc(bn & below)] = cid[c];
                            const uint32_t rank = __popc(ba & below);
                            if (acc && rank < take) mid[M + rank] = cid[c], md[M + rank] = d;
                            F += __popc(bn);
                            M += take;
                        }
                        __syncwarp();
                    }
                }
            }
        }
        if (overflow) {
            report_overflow(p.counters, p.overflow_list, qidx, lane);
            if (region_full && lane == 0) atomicAdd(p.counters + 3, 1u);
            return;
        }
        if (lane == 0) fp.out_cmps[qidx] = cmps;
        range_emit(p, mid, md, min((uint64_t)M, p.max_returned), radius_filter, qidx, hops, second, nvisited, lane);
    }
};

template <typename TD, int KIND, int POST, int NA>
__global__ void __launch_bounds__(kFiltWarps * 32) filtered_range_kernel(const FilteredRangeParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    uint8_t* base = smem + (size_t)wib * p.f.warp_smem;
    FullRowSource<TD, KIND, POST, NA, SearchParamsFiltered> src(p.f, base, lane);
    FilteredRangeSink<decltype(src)> sink(p, src, base, lane, (size_t)blockIdx.x * kFiltWarps + wib, true);
    filtered_queries<false>(p.f, base, lane, src, &sink);
}

// Over a store: the distances of filtered_kernel_quant (p.f.store), the warp's grid index its PQ-table slot; with
// p.r.rerank the output keeps every match but start points and deleted ids, for range_rerank
template <int MODE>
__global__ void __launch_bounds__(kFiltWarps * 32) filtered_range_kernel_quant(const FilteredRangeParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    uint8_t* base = smem + (size_t)wib * p.f.warp_smem;
    const uint32_t slot = blockIdx.x * kFiltWarps + wib;
    StoreSource<MODE, SearchParamsFiltered> src(p.f, base, lane, slot);
    FilteredRangeSink<decltype(src)> sink(p, src, base, lane, slot, !p.r.rerank);
    filtered_queries<false>(p.f, base, lane, src, &sink);
}

// Instantiated here, in this order, rather than by traversal_kernel in filtered_range_plan: ptxas's register allocation
// of some kernels depends on their order in the module, and with this placement every other kernel keeps its SASS
template __global__ void filtered_range_kernel_quant<STORE_SQ>(const FilteredRangeParams);
template __global__ void filtered_range_kernel_quant<STORE_MINMAX>(const FilteredRangeParams);
template __global__ void filtered_range_kernel_quant<STORE_PQ>(const FilteredRangeParams);

template <typename S>
void (*filtered_kernel_of())(const SearchParamsFiltered) {
    return filtered_kernel<typename S::TD, S::KIND, S::POST, S::NA>;
}

}  // namespace

uint32_t adaptive_l(uint32_t base_l, uint64_t visited, uint64_t matched, double scale) {
    if (matched == 0 || visited == 0) return (uint32_t)((double)base_l * scale);
    const double specificity = (double)matched / (double)visited;
    double multiplier;
    if (specificity >= 0.5) multiplier = 1.0;
    else if (specificity >= 0.1) multiplier = 2.0;
    else multiplier = std::pow(2.0, -std::log10(specificity));
    multiplier = std::min(std::max(multiplier, 1.0), scale);  // f64::clamp(1.0, scale)
    return (uint32_t)((double)base_l * multiplier);
}

std::vector<uint16_t> adaptive_table(uint32_t l_search, uint32_t samples, uint32_t span, double scale) {
    const size_t width = (size_t)samples + span;
    std::vector<uint16_t> t((size_t)span * width, 0);
    for (uint32_t r = 0; r < span; ++r) {
        const uint64_t visited = (uint64_t)samples + r;
        for (uint64_t m = 0; m <= visited; ++m) t[r * width + m] = (uint16_t)adaptive_l(l_search, visited, m, scale);
    }
    return t;
}

// A warp's shared memory: the query area (query_area_bytes), the list's distances and ids (best_max entries), the matched
// list's (L), a hop's candidate ids, distances and decisions, the beam.  `store`: -1 full precision, else a QuantStore.
static size_t filtered_warp_smem(const dab_index* idx, uint32_t l_search, uint32_t best_max, uint32_t beam, int store,
                                 SearchParamsFiltered* p) {
    size_t off = query_area_bytes(idx, store);
    const size_t best = round_up((size_t)best_max * 4, 16), matched = round_up((size_t)l_search * 4, 16);
    const size_t ncand = round_up(std::max<size_t>((size_t)beam * idx->max_degree, 32) * 4, 16);
    SearchParamsFiltered scratch;
    SearchParamsFiltered& q = p ? *p : scratch;
    q.off_bd = (uint32_t)off, off += best;
    q.off_bi = (uint32_t)off, off += best;
    q.off_md = (uint32_t)off, off += matched;
    q.off_mi = (uint32_t)off, off += matched;
    q.off_cid = (uint32_t)off, off += ncand;
    q.off_cd = (uint32_t)off, off += ncand;
    q.off_ca = (uint32_t)off, off += ncand;
    q.off_beam = (uint32_t)off, off += round_up((size_t)beam * 4, 16);
    return round_up(off, 128);
}

int filtered_check_smem(const dab_index* idx, const char* api, uint32_t l_search, uint32_t best_max, uint32_t beam, int store) {
    const size_t smem = filtered_warp_smem(idx, l_search, best_max, beam, store, nullptr) * kFiltWarps;
    if (smem > kFilteredMaxSmem)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: L=%u, longest list %u, beam_width=%u, dim=%u, max_degree=%u need %zu B shared memory per CTA (> %zu)",
                    api, l_search, best_max, beam, idx->dim, idx->max_degree, smem, kFilteredMaxSmem);
    return DAB_OK;
}

int filtered_plan(const dab_index* idx, uint32_t l_search, uint32_t best_max, uint32_t beam, int store, SearchParamsFiltered& p,
                  WarpPlan<SearchParamsFiltered>& plan) {
    p.warp_smem = (uint32_t)filtered_warp_smem(idx, l_search, best_max, beam, store, &p);
    int rc;
    if ((rc = traversal_kernel(idx, store, [](auto m) { return filtered_kernel_quant<decltype(m)::value>; },
                               [](auto sc) { return filtered_kernel_of<decltype(sc)>(); }, plan.kern)))
        return rc;
    if (!plan_warps(idx, store, kFiltWarps, p.warp_smem, kFilteredMaxSmem, plan))
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_search_batch_filtered: L=%u, beam_width=%u, dim=%u need %zu B shared memory per CTA",
                    l_search, beam, idx->dim, plan.smem_block);
    return DAB_OK;
}

int filtered_range_plan(const dab_index* idx, uint32_t l_search, uint32_t beam, int store, FilteredRangeParams& p,
                        WarpPlan<FilteredRangeParams>& plan) {
    p.f.warp_smem = (uint32_t)filtered_warp_smem(idx, l_search, l_search + idx->n_start, beam, store, &p.f);
    int rc;
    if ((rc = traversal_kernel(idx, store, [](auto m) { return filtered_range_kernel_quant<decltype(m)::value>; },
                               [](auto sc) {
                                   using S = decltype(sc);
                                   return filtered_range_kernel<typename S::TD, S::KIND, S::POST, S::NA>;
                               },
                               plan.kern)))
        return rc;
    plan_warps(idx, store, kFiltWarps, p.f.warp_smem, SIZE_MAX, plan);
    return DAB_OK;
}

// ---- the label table ---------------------------------------------------------------------------------------------
void labels_release(dab_index* idx) {
    cudaFree(idx->d_labels);
    idx->d_labels = nullptr;
}

}  // namespace dab

using namespace dab;

extern "C" {

int dab_upload_labels(dab_index* idx, const uint64_t* labels, uint64_t first, uint64_t count) {
    if (!idx || (count && !labels)) return fail(DAB_ERR_INVALID_ARGUMENT, "dab_upload_labels: NULL argument");
    if (first > idx->n_total() || count > idx->n_total() - first)
        return fail(DAB_ERR_INVALID_ARGUMENT, "dab_upload_labels: ids [%llu, %llu) out of range (%llu ids)", (unsigned long long)first,
                    (unsigned long long)(first + count), (unsigned long long)idx->n_total());
    DAB_CUDA(cudaSetDevice(idx->device));
    if (!idx->d_labels) {
        // the table is published only once it exists and is cleared
        DevBuf table;
        int rc;
        if ((rc = table.alloc(idx->n_total() * 8, "dab_upload_labels"))) return rc;
        DAB_CUDA(cudaMemsetAsync(table.p, 0, idx->n_total() * 8, idx->stream));
        DAB_CUDA(cudaStreamSynchronize(idx->stream));
        idx->d_labels = (uint64_t*)table.p;
        table.p = nullptr;
    }
    if (count == 0) return DAB_OK;
    DAB_CUDA(cudaMemcpyAsync(idx->d_labels + first, labels, count * 8, cudaMemcpyHostToDevice, idx->stream));
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    return DAB_OK;
}

}  // extern "C"
