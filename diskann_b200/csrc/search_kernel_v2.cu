// search_kernel_v2.cu — batched greedy (beam) search kept entirely on the device, one warp per query, for
// every row type (f32, f32-widened x f16, i8, u8), metric and list length.
//
// Restates DiskANNIndex::search_internal (index.rs:1933-2000) with the reference's NeighborPriorityQueue
// semantics (queue.rs:130-318) and the inmem expand_beam (provider.rs:436-479, 620-690), bit-identical
// results; the sorted candidate list (capacity L + #start, scratch.rs:195-208) lives in shared memory, the
// visited set (a HashSet in the reference) is exact, and a query whose global table would pass its load
// limit is re-run with a larger one.  The kernel is built to keep the dependent memory round trips of a hop few:
//
//   * f32 rows of 32..128 elements with level 1 of the visited set on (REG): every surviving row of a hop
//     gets one bulk L2 prefetch, then the rows are read straight into registers, 8 lanes per row and
//     4 rows per pass (wide_distances_f32_fast, the lane mapping of search_kernel_v3); prefetches and
//     loads both carry the evict_first policy of the staged copies, unless the row store is small enough for L2 to hold;
//   * all other rows are staged in shared memory with cp.async (16 B per lane, eight lanes per row:
//     one warp instruction moves 128 B of four rows and no lane needs another lane's address; no
//     registers tied up), a stage of rows in flight at once (a TMA bulk-copy variant was measured
//     slower: UBLKCP takes warp-uniform operands, so per-row copies serialise); their distances
//     are computed from shared memory (lane s <-> SIMD slot s, conflict-free) for 8 rows per pass
//     and reduced with a transpose-butterfly in the reference's association (xor 8, 16,
//     [remainder], 4, 2, 1) — 9 shuffles per 8 rows;
//   * lists of any length (QT = 0: L + #start > 256), the two-accumulator float cosine schema (NA = 2) and rows
//     too wide to stage eight of them are read straight from global memory into the FMA chains of
//     distance_device.cuh, kRowsInFlight rows per team and pass;
//   * a whole round of candidates is merged into the list at once by rank (search_common.cuh),
//     equivalent to the reference's sequential inserts;
//   * all visited-set probes of an adjacency row are issued together (two 128-bit evict_last
//     loads per 8-id bucket); the adjacency row of the next-best unvisited candidate is copied
//     into shared memory while the current hop runs, so the next hop usually starts without a
//     global round trip;
//   * the distance arithmetic is scalar f32, one row at a time (sm_90 has no packed f32x2 FADD2 / FFMA2).
#include "dab_common.cuh"
#include "distance_device.cuh"
#include "search_common.cuh"
#include "search_host.cuh"
#include "search_smem.cuh"
#include "search_v2.cuh"

#include <algorithm>
#include <cstdlib>
#include <type_traits>

namespace dab {

constexpr int kGroup = 8;  // rows reduced together
constexpr int kRowsInFlight = 4;  // QT = 0: rows per team per pass
constexpr int kV2MinCtas = 21;  // staged rows: shared memory binds residency first
constexpr int kV2MinCtasAny = 20;  // QT = 0: 96 registers, what its merge tiles and row gathers need without a spill
// rows in registers (REG): registers bind residency.  A warp scheduler holds 16K registers, so 28 one-warp CTAs per
// SM (7 per scheduler) leave 72 per thread.
constexpr int kV2MinCtasReg = 28;

__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// transpose-butterfly stage over M live values (see flat_kernels.cu)
template <int M>
__device__ __forceinline__ void bfly8(float (&v)[kGroup], int lane, int bit) {
    const bool up = (lane & bit) != 0;
#pragma unroll
    for (int i = 0; i < M / 2; ++i) {
        const float keep = up ? v[M / 2 + i] : v[i];
        const float send = up ? v[i] : v[M / 2 + i];
        v[i] = __fadd_rn(keep, __shfl_xor_sync(kFull, send, bit));
    }
}

// distances of 8 staged rows (shared memory) against the query (shared memory, f32); returns on
// every lane the value of row u = ((lane>>3)&1)<<2 | ((lane>>4)&1)<<1 | ((lane>>2)&1)
template <typename TD, int KIND>
__device__ __forceinline__ float group_distance(const float* __restrict__ q, const uint8_t* __restrict__ rows,
                                                uint32_t row_slot, int dim, int lane) {
    const int full8 = dim & ~7, rem = dim & 7;
    float v[kGroup];
#pragma unroll
    for (int g = 0; g < kGroup; ++g) v[g] = 0.0f;
    for (int e = lane; e < full8; e += 32) {
        const float x = q[e];
#pragma unroll
        for (int g = 0; g < kGroup; ++g) {
            const float y = to_f32(reinterpret_cast<const TD*>(rows + (size_t)g * row_slot)[e]);
            if (KIND == KIND_L2) {
                const float c = __fsub_rn(x, y);
                v[g] = __fmaf_rn(c, c, v[g]);
            } else {
                v[g] = __fmaf_rn(x, y, v[g]);
            }
        }
    }
    bfly8<8>(v, lane, 8);
    bfly8<4>(v, lane, 16);
    if (rem) {
        // two live values: index i | b4 << 1 | b3 << 2 (b3 = lane bit 3, b4 = lane bit 4)
        const int hi = (((lane >> 4) & 1) << 1) | (((lane >> 3) & 1) << 2);
        const int l = lane & 7;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int g = i | hi;
            const float x = l < rem ? q[full8 + l] : 0.0f;
            const float y = l < rem ? to_f32(reinterpret_cast<const TD*>(rows + (size_t)g * row_slot)[full8 + l]) : 0.0f;
            if (KIND == KIND_L2) {
                const float c = __fsub_rn(x, y);
                v[i] = __fmaf_rn(c, c, v[i]);
            } else {
                v[i] = __fmaf_rn(x, y, v[i]);
            }
        }
    }
    bfly8<2>(v, lane, 4);
    float a = v[0];
    a = __fadd_rn(a, __shfl_xor_sync(kFull, a, 2));
    a = __fadd_rn(a, __shfl_xor_sync(kFull, a, 1));
    return a;
}

// i8 / u8 rows through the same hop structure.  Integer distances are exact in i32
// (Sum(x-y)^2 = Sum x^2 + Sum y^2 - 2 Sum xy in wrapping arithmetic, as warp_int_multi), so any
// summation order gives the reference's value: lane w owns 4-byte word w of all 8 staged rows.
template <typename T>
struct V2Int {
    static constexpr bool value = false, is_signed = false;
};
template <>
struct V2Int<int8_t> {
    static constexpr bool value = true, is_signed = true;
};
template <>
struct V2Int<uint8_t> {
    static constexpr bool value = true, is_signed = false;
};

// value (before the post-op) of staged row u on every lane, for u = 0..7
template <bool SIGNED, int KIND>
__device__ __forceinline__ void group_distance_int(const uint8_t* __restrict__ q, const uint8_t* __restrict__ rows, uint32_t row_slot, int dim,
                                                   int lane, int qq, float (&out)[kGroup]) {
    int xy[kGroup], yy[kGroup];
#pragma unroll
    for (int g = 0; g < kGroup; ++g) xy[g] = yy[g] = 0;
    const int nwords = dim >> 2;
    for (int w = lane; w < nwords; w += 32) {
        const int x = reinterpret_cast<const int*>(q)[w];
#pragma unroll
        for (int g = 0; g < kGroup; ++g) {
            const int y = reinterpret_cast<const int*>(rows + (size_t)g * row_slot)[w];
            xy[g] = dp4<SIGNED>(x, y, xy[g]);
            if (KIND != KIND_IP) yy[g] = dp4<SIGNED>(y, y, yy[g]);
        }
    }
    const int tail = dim & 3;
    if (lane < tail) {
        const int i = (nwords << 2) + lane;
        const int x = byte_at<SIGNED>(q, i);
#pragma unroll
        for (int g = 0; g < kGroup; ++g) {
            const int y = byte_at<SIGNED>(rows + (size_t)g * row_slot, i);
            xy[g] += x * y;
            if (KIND != KIND_IP) yy[g] += y * y;
        }
    }
#pragma unroll
    for (int g = 0; g < kGroup; ++g) {
        const int sxy = __reduce_add_sync(kFull, xy[g]);
        if (KIND == KIND_IP) {
            out[g] = (float)sxy;
        } else {
            const int syy = __reduce_add_sync(kFull, yy[g]);
            if (KIND == KIND_L2) out[g] = (float)(int)((unsigned)qq + (unsigned)syy - 2u * (unsigned)sxy);
            else out[g] = cosine_finish((float)qq, (float)syy, (float)sxy);
        }
    }
}

// Rare path of the two-level visited set: clearing the warp's global table when its first id arrives (the atomic
// insert is visit_global).  (The kernel is sensitive to its code size — at ~100 KB of SASS every phase ran ~20 % slower than at
// 60 KB — so the hot loop is kept compact: one rolled loop over a row's chunks, no unrolled copies of these.)
__device__ __forceinline__ void clear_global_table(uint32_t* table, uint32_t nbk, int lane) {
#pragma unroll 1
    for (uint32_t i = lane; i < nbk; i += 32) store_empty_bucket(table + (size_t)i * 8);
    __syncwarp();
}

// L1 = true: two-level visited set.  Level 1 is a table of 16-bit quotient tags in the warp's own shared memory
// (tag16_probe, search_common.cuh); an id lives in exactly one level: level 1 while it has room for it (its three
// buckets not full, table not closed at 87.5 % load), otherwise level 2, this warp's global table.  A probe asks level 1
// first and only an id that is neither found nor placed there goes on to the global table — for most queries never,
// so their visited set costs no global traffic at all; the global table is cleared when its first id arrives.
// L1 = false: the global table alone (ids too wide for 14-bit tags at the table size, or level 1 disabled).
// REG = true (f32 rows of 32, 64, 96 or 128 elements, L1 on): a hop's candidate rows are read straight into registers
// after one bulk L2 prefetch per row (wide_distances_f32_fast, search_smem.cuh), so all of them are on their way from
// HBM at once and no shared memory is spent on staging them.  REG = false: rows staged in shared memory.
// QT = 4 / 8: the list is one register tile of up to 128 / 256 entries in a merge.  QT = 0: lists of any length,
// with the global table alone and the rows read straight from global memory.
template <typename TD, int KIND, int POST, int QT, bool L1, bool REG>
__global__ void __launch_bounds__(kV2Warps * 32, REG ? kV2MinCtasReg : QT == 0 ? kV2MinCtasAny : kV2MinCtas) search_kernel_v2(const SearchParamsV2 p) {
    static_assert(!REG || (std::is_same<TD, float>::value && L1), "the register row path reads f32 rows, with level 1 on");
    static_assert(QT != 0 || !L1, "lists of any length run the global table alone");
    static_assert(QT == 0 || KIND != KIND_COS || V2Int<TD>::value, "float cosine reads its rows from global memory");
    extern __shared__ __align__(128) uint8_t smem[];
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

    uint32_t* t1 = reinterpret_cast<uint32_t*>(base + p.off_t1);
    const uint32_t nb1 = p.t1_buckets;
    const Tag16Map tmap{p.tag_kmask, nb1, p.tag_magic, p.tag_shift};

    const uint32_t warp_slot = blockIdx.x * kV2Warps + wib;
    const uint32_t nbk = p.n_buckets;
    uint32_t* table = p.tables + (size_t)warp_slot * nbk * 8;
    const uint32_t hlimit = nbk * 7;  // 87.5 % load: 8-way buckets stay short
    const uint64_t n_total = p.n_points + p.n_start;
    const int dim = (int)p.dim;
    // vector rows stream through L2 (a row is read once per query): evict them first so the
    // visited tables, which are re-probed every hop, stay resident.  REG: a row store that L2 can hold is re-read from L2
    // by the other queries of the batch, so its rows keep the normal priority
    uint64_t row_policy;
    if (REG && !p.rows_evict_first) asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(row_policy));
    else asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(row_policy));

    for (uint32_t qidx; next_query(p.counters, p.n_work, p.query_list, lane, qidx);) {
        __syncwarp();
        {
            const TD* s = p.query_rows ? reinterpret_cast<const TD*>(p.vectors + (size_t)p.query_rows[qidx] * p.row_stride)
                                       : reinterpret_cast<const TD*>(p.queries) + (size_t)qidx * dim;
            load_query(s, dim, 4, qf, lane);
            if constexpr (L1) {
                const uint4 e4 = make_uint4(kEmptyV2, kEmptyV2, kEmptyV2, kEmptyV2);
                for (uint32_t i = lane; i < nb1 * 2; i += 32) reinterpret_cast<uint4*>(t1)[i] = e4;
            } else {
                for (uint32_t i = lane; i < nbk; i += 32) store_empty_bucket(table + (size_t)i * 8);
            }
        }
        __syncwarp();
        int qq = 0;  // Sum x^2 of the query (unused by inner product)
        if constexpr (V2Int<TD>::value) {
            if (KIND != KIND_IP) qq = warp_int_self<V2Int<TD>::is_signed>(reinterpret_cast<const uint8_t*>(qf), dim, lane);
        }

        uint32_t size = 0, cursor_lo = 0, cmps = 0, nvisited = 0, nrec = 0;  // nrec: expanded nodes, i.e. hops
        uint32_t n1 = 0;          // ids held by level 1 (nvisited counts those of the global table when L1 is on)
        bool closed = false;      // level 1 takes no more ids
        bool l2_used = false;     // the global table has been cleared for this query and may hold ids
        uint32_t pred = kEmptyV2;  // node whose adjacency row sits in adjbuf
        bool overflow = false;

        // HashSet::insert of one id per lane through both levels (`ok`: this lane has an id); whole warp calls
        auto visit_l1 = [&](uint32_t id, bool ok) -> bool {
            bool ins = false, need = false;
            if (ok) {
                uint32_t b1, tg;
                tag16_of(id, tmap, b1, tg);
                const int r = tag16_probe(t1, nb1, b1, tg, !closed);
                ins = r == 1;
                need = r == 2;
            }
            n1 += __popc(__ballot_sync(kFull, ins));
            if (__any_sync(kFull, need)) {  // rare
                if (!l2_used) {
                    clear_global_table(table, nbk, lane);
                    l2_used = true;
                }
                bool ins2 = false;
                if (need) ins2 = visit_global(table, nbk, id);
                nvisited += __popc(__ballot_sync(kFull, ins2));
                ins |= ins2;
            }
            return ins;
        };


        // stage `n` candidate rows (ids cid[c0..)) with per-lane 16 B async copies and compute
        // their distances into cd[]
        auto stage = [&](uint32_t c0, uint32_t n) {
            uint8_t* rows = base + p.off_rows;
            const uint32_t rows_a = smem_addr(rows);
            // eight lanes per row, 16 B each: one warp instruction moves 128 B of four different
            // rows, and every lane forms its own source address (no cross-lane traffic)
            const uint32_t sub = (uint32_t)lane >> 3, nsub = 4, off0 = ((uint32_t)lane & 7u) * 16u, offs = 128;
            auto copy16 = [&](uint32_t dst, const uint8_t* src) {
                asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "l"(row_policy) : "memory");
            };
            // copies of rows [lo, hi) as one cp.async group
            auto issue = [&](uint32_t lo, uint32_t hi) {
                if (p.row_bytes == 4 * offs) {  // 128-d f32 / 256-d f16 rows: fixed trip count, immediate offsets
                    for (uint32_t j = lo + sub; j < hi; j += nsub) {
                        const uint8_t* src = p.vectors + (size_t)cid[c0 + j] * p.row_stride + off0;
                        const uint32_t dst = rows_a + j * p.row_slot + off0;
#pragma unroll
                        for (uint32_t k = 0; k < 4; ++k) copy16(dst + k * offs, src + k * offs);
                    }
                } else {
                    for (uint32_t j = lo + sub; j < hi; j += nsub) {
                        const uint8_t* src = p.vectors + (size_t)cid[c0 + j] * p.row_stride;
                        const uint32_t dst = rows_a + j * p.row_slot;
                        for (uint32_t off = off0; off < p.row_bytes; off += offs) copy16(dst + off, src + off);
                    }
                }
                asm volatile("cp.async.commit_group;" ::: "memory");
            };
            auto compute = [&](uint32_t g0) {
                if constexpr (V2Int<TD>::value) {
                    float vals[kGroup];
                    group_distance_int<V2Int<TD>::is_signed, KIND>(reinterpret_cast<const uint8_t*>(qf), rows + (size_t)g0 * p.row_slot,
                                                                  p.row_slot, dim, lane, qq, vals);
#pragma unroll
                    for (int u = 0; u < kGroup; ++u)
                        if (lane == u && g0 + u < n) cd[c0 + g0 + u] = post_op<POST>(vals[u]);
                } else {
                    const float r = group_distance<TD, KIND>(qf, rows + (size_t)g0 * p.row_slot, p.row_slot, dim, lane);
                    const uint32_t u = (((lane >> 3) & 1) << 2) | (((lane >> 4) & 1) << 1) | ((lane >> 2) & 1);
                    if ((lane & 3) == 0 && g0 + u < n) cd[c0 + g0 + u] = post_op<POST>(r);
                }
            };
            issue(0, n);
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            __syncwarp();
            for (uint32_t g0 = 0; g0 < n; g0 += kGroup) compute(g0);
            __syncwarp();
        };

        // distances of the candidates cid[0..n) into cd[0..n)
        auto distances = [&](uint32_t n) {
            if constexpr (REG) {
                // the 16 query elements this lane multiplies, as packed pairs (re-read from shared memory per call so
                // that they do not hold registers across the hop)
                const int nm = dim >> 5;
                uint64_t q2[8] = {0ull, 0ull, 0ull, 0ull, 0ull, 0ull, 0ull, 0ull};
#pragma unroll
                for (int m = 0; m < 4; ++m) {
                    if (m < nm) {
                        const float4 x = *reinterpret_cast<const float4*>(qf + 32 * m + 4 * (lane & 7));
                        q2[2 * m] = pack2(x.x, x.y);
                        q2[2 * m + 1] = pack2(x.z, x.w);
                    }
                }
                wide_distances_f32_fast<KIND, POST, true>(q2, nm, p.vectors, p.row_stride, cid, n, cd, lane, row_policy);
                __syncwarp();
            } else if constexpr (QT == 0) {
                // a team per row, kRowsInFlight rows per team and pass: the whole warp (integers, NA = 4 float
                // schemas) or 16 lanes (float cosine, NA = 2)
                constexpr bool INT = V2Int<TD>::value;
                constexpr int S = KIND == KIND_COS && !INT ? 16 : 32, TEAMS = 32 / S, U = kRowsInFlight;
                using Row = typename std::conditional<INT, uint8_t, TD>::type;
                const int team = lane / S, slot = lane % S;
                for (uint32_t c0 = 0; c0 < n; c0 += TEAMS * U) {
                    float r[U];
                    uint32_t cc[U];
                    const Row* rows[U];
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        cc[u] = c0 + u * TEAMS + team;
                        rows[u] = reinterpret_cast<const Row*>(p.vectors + (size_t)cid[min(cc[u], n - 1)] * p.row_stride);
                    }
                    if constexpr (INT) warp_int_multi<V2Int<TD>::is_signed, KIND, U>(reinterpret_cast<const uint8_t*>(qf), rows, dim, lane, qq, r);
                    else team_float_multi<S / 8, KIND, U>(qf, rows, dim, slot, r);
#pragma unroll
                    for (int u = 0; u < U; ++u)
                        if (slot == 0 && cc[u] < n) cd[cc[u]] = post_op<POST>(r[u]);
                }
                __syncwarp();
            } else {
                for (uint32_t c0 = 0; c0 < n; c0 += p.stage_rows) stage(c0, min(p.stage_rows, n - c0));
            }
        };

        // ---- start points (SearchAccessor::start_point_distances, provider.rs:406-433)
        for (uint32_t s0 = 0; s0 < p.n_start; s0 += 32) {
            const uint32_t n = min(32u, p.n_start - s0);
            if constexpr (L1) {
                const uint32_t id = (uint32_t)p.n_points + s0 + lane;
                if ((uint32_t)lane < n) cid[lane] = id;
                visit_l1(id, (uint32_t)lane < n);
            } else if ((uint32_t)lane < n) {
                const uint32_t id = (uint32_t)p.n_points + s0 + lane;
                cid[lane] = id;
                visit_global(table, nbk, id);
            }
            __syncwarp();
            distances(n);
            merge_any<QT>(qd, qi, p.cap, size, cursor_lo, cid, cd, 0, n, lane);
            if constexpr (!L1) nvisited += n;
            cmps += n;
        }

        // ---- greedy loop (index.rs:1961-1992)
        for (;;) {
            const uint32_t lim = min(p.cap, size);
            // closest_notvisited x beam_width (queue.rs:297-313) with the build's record of expanded nodes.  The statements
            // of pick_beam (search_common.cuh), kept here: through the helper and its callback ptxas spills 4 to 20 bytes
            // more in most instantiations of this kernel, which is at its register bound
            uint32_t nb = 0;
            while (nb < p.beam) {
                const uint32_t idx = first_unvisited(qi, cursor_lo, lim, lane);
                if (idx >= lim) break;
                const uint32_t id = qi[idx];
                __syncwarp();
                if (lane == 0) {
                    qi[idx] = id | kFlagV2;
                    beam_ids[nb] = id;
                    if (p.rec_ids && nrec < p.rec_cap) {
                        p.rec_ids[(size_t)qidx * p.rec_cap + nrec] = id;
                        p.rec_dists[(size_t)qidx * p.rec_cap + nrec] = qd[idx];
                    }
                }
                cursor_lo = idx + 1;
                ++nrec;
                ++nb;
                __syncwarp();
            }
            if (nb == 0) break;

            uint32_t ncand = 0;
            for (uint32_t b = 0; b < nb; ++b) {
                const uint32_t node = beam_ids[b];
                const uint32_t* row = p.adj + (size_t)node * p.adj_stride;
                uint32_t wd[3];
                if (b == 0 && p.adj_words) {
                    // the speculative copy of the previous hop has long landed; it must be
                    // drained before the buffer is read or re-targeted
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
                    // speculative: the next hop most likely expands the now-first unvisited entry;
                    // fetch its adjacency row into shared memory (or at least into L2) while
                    // this hop runs
                    const uint32_t nxt = first_unvisited(qi, cursor_lo, lim, lane);
                    pred = kEmptyV2;
                    if (nxt < lim) {
                        const uint32_t nid = qi[nxt] & ~kFlagV2;
                        const uint32_t* nrow = p.adj + (size_t)nid * p.adj_stride;
                        if (p.adj_words) {
                            pred = nid;
                            if ((uint32_t)lane * 4 < p.adj_words)
                                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(adjbuf_a + lane * 16), "l"(nrow + lane * 4)
                                             : "memory");
                            asm volatile("cp.async.commit_group;" ::: "memory");
                        } else if (lane < 3) {
                            prefetch_l2(nrow + lane * 32);
                        }
                    }
                }
                const uint32_t deg = min(__shfl_sync(kFull, wd[0], 0), p.max_degree);
                if constexpr (L1) {
                    // one compact loop over the row's chunks of 32 neighbours (the first three sit in registers)
#pragma unroll 1
                    for (uint32_t c0 = 0; c0 <= deg; c0 += 32) {
                        const uint32_t j = c0 + lane;
                        uint32_t word = c0 == 0 ? wd[0] : (c0 == 32 ? wd[1] : wd[2]);
                        if (c0 >= 96) word = j < p.adj_stride ? __ldg(row + j) : kEmptyV2;
                        // ids beyond 2^K cannot be in bounds and would share the tag of id mod 2^K: not tracked
                        const bool ins = visit_l1(word, j >= 1 && j <= deg && word <= tmap.kmask);
                        push_new(ins && word < n_total, word, cid, ncand, lane);  // is_in_bounds; visit_l1 has counted the insert
                    }
                    if (!closed && n1 + p.max_degree > p.t1_limit) closed = true;
                } else {
                // bucket probes of all three chunks in flight together
                    bool valid[3];
                    uint32_t bk[3];
                    uint32_t bs[3][8];
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const uint32_t j = c * 32 + lane;
                        valid[c] = j >= 1 && j <= deg;
                        bk[c] = bucket_of(wd[c], nbk);
                        if (valid[c]) load_bucket(table + (size_t)bk[c] * 8, bs[c]);
                    }
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        bool inserted = false;
                        if (valid[c]) inserted = bucket_insert(table, nbk, bk[c], bs[c], wd[c]);
                        push_new(inserted, inserted && wd[c] < n_total, wd[c], cid, ncand, nvisited, lane);  // is_in_bounds
                    }
                    // adjacency rows longer than 95 neighbours: remaining chunks
                    for (uint32_t c0 = 96; c0 < deg + 1; c0 += 32) {
                        const uint32_t j = c0 + lane;
                        const uint32_t word = j < p.adj_stride ? __ldg(row + j) : kEmptyV2;
                        const bool inserted = j <= deg && visit_global(table, nbk, word);
                        push_new(inserted, inserted && word < n_total, word, cid, ncand, nvisited, lane);
                    }
                }
                if (nvisited + p.max_degree > hlimit) {  // the next node could pass the load limit: stop expanding now
                    overflow = true;
                    break;
                }
            }
            if (overflow) break;
            __syncwarp();

            distances(ncand);

            // best.insert for every neighbour in adjacency order (index.rs:1986-1988)
            for (uint32_t c0 = 0; c0 < ncand; c0 += 32)
                merge_any<QT>(qd, qi, p.cap, size, cursor_lo, cid, cd, c0, min(32u, ncand - c0), lane);
            cmps += ncand;
        }

        if (overflow) {
            report_overflow(p.counters, p.overflow_list, qidx, lane);
            continue;
        }

        // ---- post-process: drop start points, first k (provider.rs:907-950)
        {
            const uint32_t count = write_results(qi, qd, min(p.cap, size), p.result_bound, p.k, p.out_ids, p.out_dists, qidx, lane);
            // the visited set is level 1's ids plus the global table's (nvisited counts only those when level 1 is on);
            // every expanded node is a hop, so nrec is the hop count
            write_stats(p.counters, n1 + nvisited, p.out_counts, p.out_cmps, p.out_hops, qidx, count, cmps, nrec, lane);
            if (lane == 0 && p.rec_counts) {
                p.rec_counts[qidx] = min(nrec, p.rec_cap);
                if (nrec > p.rec_cap) atomicAdd(p.counters + 3, 1u);  // expanded nodes beyond the record: reported by dab_build
            }
        }
    }
    // without row staging nothing else drains the last speculative adjacency copy
    if constexpr (REG) asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// ------------------------------------------------------------------ host side
// the instantiation for a level-1 choice and row path (only f32 rows with level 1 on have the register path)
template <typename TD, int K, int P, int Q>
static void (*pick_v2(bool l1, bool reg))(const SearchParamsV2) {
    if constexpr (std::is_same<TD, float>::value) {
        if (reg) return search_kernel_v2<TD, K, P, Q, true, true>;
    }
    return l1 ? search_kernel_v2<TD, K, P, Q, true, false> : search_kernel_v2<TD, K, P, Q, false, false>;
}

// v2_prepare for the index's distance schema S (visit_schema)
template <typename S>
static int v2_prepare_schema(const dab_index* idx, uint32_t l_search, uint32_t beam, bool level1, SearchParamsV2& p, V2Launch& out) {
    const uint32_t cap = l_search + idx->n_start;
    const uint32_t row_bytes = (uint32_t)round_up((size_t)idx->dim * elem_size(idx->dtype), 16);
    auto too_big = [&] {
        return fail(DAB_ERR_INVALID_ARGUMENT, "search: L=%u, beam=%u, dim=%u need %zu B shared memory per CTA (> 200 KB)", l_search,
                    beam, idx->dim, out.smem_block);
    };
    size_t off = 0;
    p.off_q = (uint32_t)off;
    off += S::IS_INT ? round_up(round_up((size_t)idx->dim, 4), 16) : round_up((size_t)idx->dim * 4, 16);
    const size_t ncand_max = (size_t)beam * idx->max_degree;
    p.off_cid = (uint32_t)off;
    off += round_up(std::max<size_t>(ncand_max, idx->n_start) * 4, 16);
    p.off_cd = (uint32_t)off;
    off += round_up(std::max<size_t>(ncand_max, idx->n_start) * 4, 16);
    p.off_beam = (uint32_t)off;
    off += round_up((size_t)beam * 4, 16);
    // speculative adjacency buffer: the first <= 96 words of a row, 16-byte granules
    p.adj_words = idx->adj_stride % 4 == 0 ? (uint32_t)std::min<size_t>(idx->adj_stride, 96) : 0;
    p.off_adj = (uint32_t)off;
    off += (size_t)p.adj_words * 4;
    const size_t cap_pad = round_up(cap, 4);
    p.off_qd = (uint32_t)off;
    off += cap_pad * 4;
    p.off_qi = (uint32_t)off;
    off += cap_pad * 4;
    p.row_bytes = row_bytes;
    // register rows that stream through L2 are evicted first; a store of at most twice the L2 size (100K x 128 f32:
    // 51 MB on the H100's 50 MB L2) is largely re-read from L2 and keeps the normal priority (staged rows are always
    // evicted first: at 100K, one batch at a time measured 12 % slower with the normal priority)
    p.rows_evict_first = idx->n_total() * idx->row_stride > 2 * (uint64_t)idx->l2_bytes;
    // rows staged per round: as many as fit ~6 KB per warp, a multiple of the reduce group
    const size_t stage_bytes = 6144;
    const uint32_t stage = std::min<uint32_t>(32, (uint32_t)std::max<size_t>(kGroup, (stage_bytes / row_bytes) / kGroup * kGroup));
    // QT = 0 where one register tile does not hold the list, for the float cosine schema (NA = 2), and for rows so wide
    // that a stage of them does not fit: rows read straight from global memory, the global table alone
    const bool any_len = cap > 256 || S::NA == 2 || round_up(off, 128) + (size_t)stage * row_bytes > 200 * 1024;
    // level-1 visited table: 4 KB of 16-bit tags per warp (2048 slots; the mean visited set of the headline
    // workload is ~1200 ids) when the ids fit 14-bit quotient tags, i.e. n_total <= 16384 * buckets
    size_t t1_bytes = idx->tune.test_visited_log2 ? 512 : 4096;  // tests: a level 1 that fills at once
    p.t1_buckets = 0;
    const uint64_t nb1 = t1_bytes / 32;
    if (set_tag_map(idx, nb1, p)) {
        p.t1_buckets = (uint32_t)nb1;
        p.t1_limit = (uint32_t)(nb1 * 14);
    }
    // level 1 pays for itself only while enough warps stay resident: at C2 (24 -> 20 one-warp CTAs per SM) it removes
    // the table traffic (8.8 -> 5.3 GB of DRAM traffic per 10K queries) and is 2 % faster, at C3 (12 -> 10) it is 11 % slower
    // ... and while batches overlap: one batch at a time is dominated by its tail, where the 4 resident warps fewer
    // cost more (2.96 vs 2.67 ms) than the traffic saves
    if (!level1 || any_len) p.t1_buckets = 0;
    auto resident_warps = [&](size_t t1_at) {
        return (227 * 1024) / (round_up(round_up(t1_at, 32) + t1_bytes, 128) * kV2Warps + 1024) * kV2Warps;
    };
    // f32 rows of 32, 64, 96 or 128 elements (C2, the C5 shape) with level 1 on are read into registers: without the
    // staging buffer registers bind residency (28 warps per SM at C2 instead of 20).  Everything else stages its rows:
    // with the global table alone the register path does not raise residency (registers bind both at 80), and one
    // batch at a time at C2 measured 3.6 % slower on it.
    const bool reg = idx->dtype == DAB_F32 && idx->dim % 32 == 0 && idx->dim <= 128 && p.t1_buckets && resident_warps(off) >= 16;
    if (!reg && !any_len) {
        off = round_up(off, 128);
        p.off_rows = (uint32_t)off;
        p.stage_rows = stage;
        p.row_slot = row_bytes;
        off += (size_t)stage * row_bytes;
    }
    p.off_t1 = (uint32_t)round_up(off, 32);
    if (p.t1_buckets && resident_warps(off) < 16) p.t1_buckets = 0;
    if (!p.t1_buckets) t1_bytes = 0;
    p.warp_smem = (uint32_t)round_up((size_t)p.off_t1 + t1_bytes, 128);
    out.smem_block = (size_t)p.warp_smem * kV2Warps;
    if (out.smem_block > 200 * 1024) return too_big();

    using TD = typename S::TD;
    const bool l1 = p.t1_buckets != 0;
    // the float cosine schema (NA = 2) always runs with any_len: it has no tiled instantiations
    if (any_len) out.kern = search_kernel_v2<TD, S::KIND, S::POST, 0, false, false>;
    else if constexpr (S::NA == 4)
        out.kern = cap <= 128 ? pick_v2<TD, S::KIND, S::POST, 4>(l1, reg) : pick_v2<TD, S::KIND, S::POST, 8>(l1, reg);
    const int per_sm = ctas_per_sm(out.kern, kV2Warps * 32, out.smem_block);
    if (per_sm < 1) return too_big();
    out.grid = per_sm * idx->sm_count;
    return 0;
}

int v2_prepare(const dab_index* idx, uint32_t l_search, uint32_t beam, bool level1, SearchParamsV2& p, V2Launch& out) {
    return visit_schema<OPS_QUERY>(idx->dtype, idx->metric, [&](auto s) {
        return v2_prepare_schema<decltype(s)>(idx, l_search, beam, level1, p, out);
    });
}

}  // namespace dab
