// search_kernel_v3.cu — batched greedy search with the visited set in SHARED memory.
//
// Same semantics and bit-identical results as search_kernel_v2.cu
// (DiskANNIndex::search_internal, index.rs:1933-2000; NeighborPriorityQueue, queue.rs:130-318;
// expand_beam, provider.rs:436-479, 620-690).  What changes against v2 is the number of
// dependent GLOBAL-memory round trips a hop costs — v2 has three (bucket probe, CAS, row
// copy), and its per-warp tables (tens of MB for a few thousand resident warps) do not stay in
// L2, so a large share of the bytes a launch moves is random 32-byte table sectors:
//
//   * the visited set of a query is an exact open-addressed table of 16-bit quotient tags in
//     the warp's own shared memory (id -> (bucket, tag) is a bijection for ids < 2^K, so only
//     the tag is stored: 16 entries per 32-byte bucket, displacement <= 2 buckets recorded in
//     the tag's top two bits).  A probe is two LDS.128, an insert one 32-bit shared-memory CAS;
//     a query that outgrows its table is handed to search_kernel_v2 (exactness is kept,
//     only speed is lost);
//   * the only HBM round trip left on a hop's critical path is the row gather itself: rows are
//     read straight into registers with 16-byte loads, 8 (f32) / 4 (f16) lanes per row and up
//     to 16 rows in flight per warp, each lane running the FMA chains of the SIMD slots it
//     loaded (the lane mapping of frontier_wide_kernel) — no staging buffer, which is what makes
//     room for the table;
//   * i8 / u8 rows use the same structure with exact i32 dot products (dp4a);
//   * the adjacency row of the predicted next node is copied into shared memory while the
//     current hop runs (as in v2), so a hop normally starts without a global round trip.
#include "dab_common.cuh"
#include "distance_device.cuh"
#include "search_common.cuh"
#include "search_host.cuh"
#include "search_smem.cuh"
#include "search_v3.cuh"

#include <algorithm>
#include <cstdlib>
#include <type_traits>

namespace dab {

namespace {

template <typename T>
struct IsInt {
    static constexpr bool value = std::is_same<T, int8_t>::value || std::is_same<T, uint8_t>::value;
};

constexpr int kV3MinCtas = 4;
constexpr int kV3PassesF32 = 2;  // f32 rows: passes (of 4 rows, 4 x 16-byte loads per lane each) in flight
constexpr int kV3PassesF16 = 2;  // f16 rows: passes (of 8 rows) in flight
constexpr int kV3LoadsF16 = 4;   // f16 rows: 16-byte loads per lane per pass in flight
constexpr int kV3PassesInt = 4;  // i8 / u8 rows: passes (of 4 rows, one 16-byte load per lane each) in flight

}  // namespace

template <typename TD, int KIND, int POST, int QT, bool FAST>
__global__ void __launch_bounds__(kV3Warps * 32, kV3MinCtas) search_kernel_v3(const SearchParamsV3 p) {
    extern __shared__ __align__(128) uint8_t smem[];
    constexpr bool kInt = IsInt<TD>::value;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    uint8_t* base = smem + (size_t)wib * p.warp_smem;
    float* qf = reinterpret_cast<float*>(base + p.off_q);
    float* qd = reinterpret_cast<float*>(base + p.off_qd);
    uint32_t* qi = reinterpret_cast<uint32_t*>(base + p.off_qi);
    uint32_t* cid = reinterpret_cast<uint32_t*>(base + p.off_cid);
    float* cd = reinterpret_cast<float*>(base + p.off_cd);
    uint32_t* beam_ids = reinterpret_cast<uint32_t*>(base + p.off_beam);
    uint32_t* adjbuf = reinterpret_cast<uint32_t*>(base + p.off_adj);
    const uint32_t adjbuf_a = smem_addr(adjbuf);
    uint32_t* table = reinterpret_cast<uint32_t*>(base + p.off_table);
    const uint32_t nbk = p.n_buckets;
    const Tag16Map tmap{p.tag_kmask, nbk, p.tag_magic, p.tag_shift};
    auto visit = [&](uint32_t id, bool& ovf) -> bool {
        uint32_t bk, tg;
        tag16_of(id, tmap, bk, tg);
        return smem16_insert(table, nbk, bk, tg, ovf);
    };
    const uint64_t n_total = p.n_points + p.n_start;
    const int dim = (int)p.dim;

    for (uint32_t qidx; next_query(p.counters, p.n_work, p.query_list, lane, qidx);) {
        __syncwarp();
        {
            const TD* s = p.query_rows ? reinterpret_cast<const TD*>(p.vectors + (size_t)p.query_rows[qidx] * p.row_stride)
                                       : reinterpret_cast<const TD*>(p.queries) + (size_t)qidx * dim;
            load_query(s, dim, 16, qf, lane);
            const uint4 e4 = make_uint4(kEmptyV2, kEmptyV2, kEmptyV2, kEmptyV2);
            for (uint32_t i = lane; i < nbk * 2; i += 32) reinterpret_cast<uint4*>(table)[i] = e4;
        }
        __syncwarp();
        int qq = 0;  // sum x^2 of an integer query (unused by inner product)
        if constexpr (kInt) {
            if (KIND != KIND_IP) qq = warp_int_self<std::is_same<TD, int8_t>::value>(reinterpret_cast<const uint8_t*>(qf), dim, lane);
        }
        (void)qq;
        // fast f32 path: the 16 query elements this lane multiplies, as packed pairs
        uint64_t q2[8] = {0ull, 0ull, 0ull, 0ull, 0ull, 0ull, 0ull, 0ull};
        if constexpr (FAST) {
            {
#pragma unroll
                for (int m = 0; m < 4; ++m) {
                    if (m < (int)p.fast_nm) {
                        const float4 x = *reinterpret_cast<const float4*>(qf + 32 * m + 4 * (lane & 7));
                        q2[2 * m] = pack2(x.x, x.y);
                        q2[2 * m + 1] = pack2(x.z, x.w);
                    }
                }
            }
        }

        uint32_t size = 0, cursor_lo = 0, cmps = 0, hops = 0, nvisited = 0, nrec = 0;
        uint32_t pred = kEmptyV2;  // node whose adjacency row sits in adjbuf
        bool overflow = false;

        auto distances = [&](uint32_t c0, uint32_t n) {
            if constexpr (kInt) {
                wide_distances_int<std::is_same<TD, int8_t>::value, KIND, POST, kV3PassesInt>(reinterpret_cast<const uint8_t*>(qf), qq, p.vectors,
                                                                                 p.row_stride, cid + c0, n, cd + c0, dim, lane);
            } else if constexpr (sizeof(TD) == 2) {
                wide_distances<TD, KIND, POST, kV3PassesF16, kV3LoadsF16>(qf, p.vectors, p.row_stride, cid + c0, n, cd + c0, dim, lane);
            } else if constexpr (FAST) {
                wide_distances_f32_fast<KIND, POST>(q2, (int)p.fast_nm, p.vectors, p.row_stride, cid + c0, n, cd + c0, lane);
            } else {
                wide_distances<TD, KIND, POST, kV3PassesF32, 4>(qf, p.vectors, p.row_stride, cid + c0, n, cd + c0, dim, lane);
            }
            __syncwarp();
        };

        // ---- start points (SearchAccessor::start_point_distances, provider.rs:406-433)
        for (uint32_t s0 = 0; s0 < p.n_start; s0 += 32) {
            const uint32_t n = min(32u, p.n_start - s0);
            bool ovf = false;
            if ((uint32_t)lane < n) {
                const uint32_t id = (uint32_t)p.n_points + s0 + lane;
                cid[lane] = id;
                visit(id, ovf);
            }
            if (__any_sync(kFull, ovf)) overflow = true;
            __syncwarp();
            distances(0, n);
            merge_round<QT>(qd, qi, p.cap, size, cursor_lo, cid, cd, 0, n, lane);
            nvisited += n;
            cmps += n;
        }
        if (nvisited > p.visited_limit) overflow = true;

        // ---- greedy loop (index.rs:1961-1992)
        while (!overflow) {
            const uint32_t lim = min(p.cap, size);
            // the build records every expanded node and its distance, in expansion order
            const uint32_t nb = pick_beam(qi, lim, p.beam, cursor_lo, beam_ids, lane, [&](uint32_t b, uint32_t idx, uint32_t id) {
                if (p.rec_ids && nrec + b < p.rec_cap) {
                    p.rec_ids[(size_t)qidx * p.rec_cap + nrec + b] = id;
                    p.rec_dists[(size_t)qidx * p.rec_cap + nrec + b] = qd[idx];
                }
            });
            if (nb == 0) break;
            nrec += nb;

            uint32_t ncand = 0;
            for (uint32_t b = 0; b < nb; ++b) {
                const uint32_t node = beam_ids[b];
                const uint32_t* row = p.adj + (size_t)node * p.adj_stride;
                uint32_t wd[3];
                if (b == 0 && p.adj_words) {
                    // the speculative copy of the previous hop must be drained before the buffer
                    // is read or re-targeted
                    asm volatile("cp.async.wait_group 0;" ::: "memory");
                    __syncwarp();
                }
                if (b == 0 && node == pred) {
                    wd[0] = adjbuf[lane];
                    wd[1] = 32 + lane < p.adj_words ? adjbuf[32 + lane] : kEmptyV2;
                    wd[2] = 64 + lane < p.adj_words ? adjbuf[64 + lane] : kEmptyV2;
                    __syncwarp();
                } else {
                    wd[0] = __ldg(row + lane);
                    wd[1] = 32 + lane < p.adj_stride ? __ldg(row + 32 + lane) : kEmptyV2;
                    wd[2] = 64 + lane < p.adj_stride ? __ldg(row + 64 + lane) : kEmptyV2;
                }
                if (b == 0) {
                    // speculative: the next hop most likely expands the now-first unvisited entry
                    const uint32_t nxt = first_unvisited(qi, cursor_lo, lim, lane);
                    pred = kEmptyV2;
                    if (nxt < lim && p.adj_words) {
                        const uint32_t nid = qi[nxt] & ~kFlagV2;
                        const uint32_t* nrow = p.adj + (size_t)nid * p.adj_stride;
                        pred = nid;
                        if ((uint32_t)lane * 4 < p.adj_words)
                            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(adjbuf_a + lane * 16), "l"(nrow + lane * 4) : "memory");
                        asm volatile("cp.async.commit_group;" ::: "memory");
                    }
                }
                const uint32_t deg = min(__shfl_sync(kFull, wd[0], 0), p.max_degree);
                if (nvisited + deg > p.visited_limit) {  // the table could pass its load limit: global-table kernel
                    overflow = true;
                    break;
                }
                bool ovf = false;
                auto filter = [&](uint32_t word, uint32_t j) {
                    bool inserted = false;
                    // ids beyond 2^K cannot be in bounds and never reach the outputs: not tracked
                    if (j >= 1 && j <= deg && word <= tmap.kmask) inserted = visit(word, ovf);
                    push_new(inserted, inserted && word < n_total, word, cid, ncand, nvisited, lane);  // is_in_bounds
                };
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    if ((uint32_t)c * 32 <= deg) filter(wd[c], c * 32 + lane);
                // adjacency rows longer than 95 neighbours: remaining chunks
                for (uint32_t c0 = 96; c0 < deg + 1; c0 += 32) {
                    const uint32_t j = c0 + lane;
                    filter(j < p.adj_stride ? __ldg(row + j) : kEmptyV2, j);
                }
                if (__any_sync(kFull, ovf)) {
                    overflow = true;
                    break;
                }
            }
            if (overflow) break;
            __syncwarp();

            distances(0, ncand);

            // best.insert for every neighbour in adjacency order (index.rs:1986-1988)
            for (uint32_t c0 = 0; c0 < ncand; c0 += 32)
                merge_round<QT>(qd, qi, p.cap, size, cursor_lo, cid, cd, c0, min(32u, ncand - c0), lane);
            cmps += ncand;
            hops += nb;
        }

        if (overflow) {
            if (p.adj_words) asm volatile("cp.async.wait_group 0;" ::: "memory");
            report_overflow(p.counters, p.overflow_list, qidx, lane);
            continue;
        }

        // ---- post-process: drop start points, first k (provider.rs:907-950)
        {
            const uint32_t count = write_results(qi, qd, min(p.cap, size), p.result_bound, p.k, p.out_ids, p.out_dists, qidx, lane);
            write_stats(p.counters, nvisited, p.out_counts, p.out_cmps, p.out_hops, qidx, count, cmps, hops, lane);
            if (lane == 0 && p.rec_counts) {
                p.rec_counts[qidx] = min(nrec, p.rec_cap);
                if (nrec > p.rec_cap) atomicAdd(p.counters + 3, 1u);  // expanded nodes beyond the record: reported by dab_build
            }
        }
    }
}

// ------------------------------------------------------------------ host side
// v3_prepare for the index's distance schema S (visit_schema)
template <typename S>
static int v3_prepare_schema(const dab_index* idx, uint32_t l_search, uint32_t beam, uint32_t visited_need, SearchParamsV3& p,
                             V3Launch& out) {
    // v3 is for short candidate lists (L + start points <= 24), whose visited sets are small.  At the headline L = 100
    // its whole-set tag table (~11.5 KB per warp) leaves 16 warps per SM, while v2's 4 KB level 1 with the global
    // table behind it leaves 28 (f32 rows in registers) or 20 (staged rows), so v2 is faster there
    if (l_search + idx->n_start > 24) return 1;
    const uint32_t cap = l_search + idx->n_start;
    if (idx->max_degree > 1000) return 1;
    if ((idx->row_stride & 15) != 0) return 1;
    // quotient tags: ids < 2^K, tag = h / n_buckets must fit 14 bits
    const uint32_t K = tag_id_bits(idx->n_total());
    if (K > 30) return 1;
    const uint64_t min_buckets = std::max<uint64_t>(16, (((uint64_t)1 << K) + 16383) >> 14);

    size_t off = 0;
    p.off_q = (uint32_t)off;
    off += S::IS_INT ? round_up((size_t)idx->dim, 16) : round_up((size_t)idx->dim * 4, 16);
    const size_t ncand_max = std::max<size_t>((size_t)beam * idx->max_degree, std::min<uint32_t>(32, idx->n_start));
    p.off_cid = (uint32_t)off;
    off += round_up(ncand_max * 4, 16);
    p.off_cd = (uint32_t)off;
    off += round_up(ncand_max * 4, 16);
    p.off_beam = (uint32_t)off;
    off += round_up((size_t)beam * 4, 16);
    p.adj_words = idx->adj_stride % 4 == 0 ? (uint32_t)std::min<size_t>(idx->adj_stride, 96) : 0;
    p.off_adj = (uint32_t)off;
    off += (size_t)p.adj_words * 4;
    const size_t cap_pad = round_up(cap, 4);
    p.off_qd = (uint32_t)off;
    off += cap_pad * 4;
    p.off_qi = (uint32_t)off;
    off += cap_pad * 4;
    off = round_up(off, 32);
    p.off_table = (uint32_t)off;
    const size_t fixed = off;

    const size_t smem_sm = 227 * 1024;  // per SM, 1 KB per CTA is reserved by the system
    auto table_bytes_at = [&](int ctas) -> long long {
        const long long per_cta = (long long)(smem_sm / ctas) - 1024;
        return (per_cta / kV3Warps - (long long)fixed) / 32 * 32;
    };
    // registers bound the residency (kV3MinCtas CTAs per SM), so the table takes all the shared
    // memory that residency leaves: a smaller table would only overflow more often
    long long tbytes = table_bytes_at(kV3MinCtas);
    if (idx->tune.test_visited_log2 && visited_need)  // tests: a table small enough to overflow
        tbytes = (long long)round_up((size_t)((visited_need + idx->max_degree) / 0.875) * 2 + 32, 32);
    if (tbytes < (long long)min_buckets * 32) tbytes = (long long)min_buckets * 32;
    if (tbytes > table_bytes_at(1)) return 1;
    const uint64_t nbk = (uint64_t)tbytes / 32;
    if (!set_tag_map(idx, nbk, p)) return 1;
    p.n_buckets = (uint32_t)nbk;
    p.visited_limit = (uint32_t)(nbk * 14);  // 87.5 % of 16 tags per bucket
    p.fast_nm = (idx->dtype == DAB_F32 && idx->dim % 32 == 0 && idx->dim <= 128) ? idx->dim / 32 : 0;
    out.capacity = p.visited_limit > idx->max_degree ? p.visited_limit - idx->max_degree : 0;
    if (out.capacity < 4 * idx->max_degree) return 1;
    p.warp_smem = (uint32_t)round_up(fixed + (size_t)tbytes, 128);
    out.smem_block = (size_t)p.warp_smem * kV3Warps;

    // cap <= 24: the list fits one register tile of the merge (QT = 4, up to 128 entries)
    using TD = typename S::TD;
    out.kern = search_kernel_v3<TD, S::KIND, S::POST, 4, false>;
    if constexpr (std::is_same<TD, float>::value) {
        if (p.fast_nm) out.kern = search_kernel_v3<TD, S::KIND, S::POST, 4, true>;
    }
    const int per_sm = ctas_per_sm(out.kern, kV3Warps * 32, out.smem_block);
    if (per_sm < 1) return 1;
    out.grid = per_sm * idx->sm_count;
    return 0;
}

int v3_prepare(const dab_index* idx, uint32_t l_search, uint32_t beam, uint32_t visited_need, SearchParamsV3& p, V3Launch& out) {
    return visit_schema<OPS_QUERY>(idx->dtype, idx->metric, [&](auto s) -> int {
        using S = decltype(s);
        if constexpr (S::NA == 2) return 1;  // float cosine: the two-accumulator schema, search_kernel_v2
        else return v3_prepare_schema<S>(idx, l_search, beam, visited_need, p, out);
    });
}

}  // namespace dab
