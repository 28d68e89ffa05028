// search_source.cuh — the distance sources of the paged, diverse, filtered and range traversals (search_paged.cu,
// search_diverse.cu, search_filtered.cu, search_range.cu) and the store fields of their parameter blocks.
//
// Each of those searches is one device function over a distance source (paged_queries, diverse_queries,
// filtered_queries, range_queries).  A source has load(q), which brings query q into the front of the warp's shared
// memory; prepare(), which runs once the query's list or visited table is in place (what the distances need of the
// loaded query); and distances(cid, cd, n), which writes the distances of cid[0..n) into cd[0..n) and ends with the warp
// converged.  FullRowSource reads full-precision rows, StoreSource a quantized store; both read whichever parameter
// block P is.
#pragma once

#include "dab_common.cuh"
#include "quant_device.cuh"
#include "search_common.cuh"

#include <type_traits>

namespace dab {

// The quantized store a traversal reads (set_store_params), named as in SearchParamsPq for the per-candidate code
// (quant_device.cuh).  Every parameter block keeps it after the fields of its full-precision kernel, so that their
// offsets stay as they were.
struct StoreParams {
    int dtype;
    const float* pivots;  // PQ: the table, [n_centers][dim]
    const uint32_t* offsets;
    const uint8_t* codes;  // [n_total][n_chunks]
    uint32_t n_chunks, n_centers;
    int ip_table, direct_cosine;
    float* luts;  // PQ tables (TableL2 / TableIP): n_chunks x n_centers f32 for every warp of the grid
    const uint8_t* row_codes;  // SQ / MinMax: the store's rows and the batch's staged queries
    const float* row_meta;
    uint32_t code_stride, code_dim;
    int code_nbits, code_metric;
    float sq_scale_squared, sq_shift_square_norm;
    const uint8_t* query_codes;  // [nq][code_stride]
    const float4* query_meta;    // [nq]
};

// Full precision: rows from global memory with the shared distance schemas (distance_device.cuh), a team of lanes per
// row and kRows rows in flight per team.  Reads p.queries, p.vectors, p.row_stride and p.dim.
template <typename TD, int KIND, int POST, int NA, class P>
struct FullRowSource {
    static constexpr bool INT = std::is_same<TD, int8_t>::value || std::is_same<TD, uint8_t>::value;
    static constexpr int kRows = 4;
    const P& p;
    float* qf;
    int lane, dim, qq;  // qq, integer rows: Sum x^2 of the query (unused by inner product)

    __device__ __forceinline__ FullRowSource(const P& p_, uint8_t* base, int lane_)
        : p(p_), qf(reinterpret_cast<float*>(base)), lane(lane_), dim((int)p_.dim), qq(0) {}
    __device__ __forceinline__ void load(uint32_t q) { load_query(reinterpret_cast<const TD*>(p.queries) + (size_t)q * dim, dim, 4, qf, lane); }
    __device__ __forceinline__ void prepare() {
        if constexpr (INT) {
            if (KIND != KIND_IP) qq = warp_int_self<std::is_same<TD, int8_t>::value>(reinterpret_cast<const uint8_t*>(qf), dim, lane);
        }
    }
    __device__ __forceinline__ void distances(const uint32_t* cid, float* cd, uint32_t n) {
        constexpr int S = INT ? 32 : 8 * NA, TEAMS = 32 / S, U = kRows;
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
            if constexpr (INT) warp_int_multi<std::is_same<TD, int8_t>::value, KIND, U>(reinterpret_cast<const uint8_t*>(qf), rows, dim, lane, qq, r);
            else team_float_multi<NA, KIND, U>(qf, rows, dim, slot, r);
#pragma unroll
            for (int u = 0; u < U; ++u)
                if (slot == 0 && cc[u] < n) cd[cc[u]] = post_op<POST>(r[u]);
        }
        __syncwarp();
    }
};

// A quantized store (MODE as search_kernel_pq: 0 PQ, 1 SQ, 2 MinMax): per candidate the code of quant_device.cuh, one
// lane per candidate, so a traversal gets the distances of dab_search_batch_{pq,sq,minmax}.  Reads p.queries and p.store.
//   PQ: the query (index dtype, T: Into<f32>) in f32 at the front of the warp's shared memory.  TableL2 / TableIP build
//     the query's table once per query into the warp's own slice of p.store.luts (global memory, read through L2: the
//     table does not fit next to the lists in shared memory); `warp` is the warp's index in the grid.  DirectCosine
//     reads the pivots directly.
//   SQ / MinMax: the query's code words (and MinMax its four compensations), staged before the launch, copied to the
//     front of the warp's shared memory; the SQ compensation stays in a register.
template <int MODE, class P>
struct StoreSource {
    const P& p;
    float* qf;     // PQ: the f32 query
    uint32_t* qc;  // SQ / MinMax: the query's code words, then (MinMax) {b, n, a, norm_squared}
    float* lut;    // PQ tables: this warp's table
    int lane, dim;
    uint32_t entries;
    float q_comp;

    __device__ __forceinline__ StoreSource(const P& p_, uint8_t* base, int lane_, uint32_t warp)
        : p(p_), qf(reinterpret_cast<float*>(base)), qc(reinterpret_cast<uint32_t*>(base)),
          lut(p_.store.luts + (size_t)warp * (p_.store.n_chunks * p_.store.n_centers)), lane(lane_), dim((int)p_.dim),
          entries(p_.store.n_chunks * p_.store.n_centers), q_comp(0.0f) {}
    __device__ __forceinline__ void load(uint32_t q) {
        if (MODE == 0) widen_query(p.store.dtype, p.queries, q, dim, qf, lane);
        else load_query_codes<MODE>(p.store.query_codes + (size_t)q * p.store.code_stride, p.store.query_meta + q, p.store.code_stride >> 2, qc, q_comp, lane);
    }
    __device__ __forceinline__ void prepare() {
        if (MODE == 0 && !p.store.direct_cosine) {
            for (uint32_t t = lane; t < entries; t += 32) __stcg(lut + t, pq_table_entry(p.store, qf, dim, t));
            __syncwarp();
        }
    }
    __device__ __forceinline__ void distances(const uint32_t* cid, float* cd, uint32_t n) {
        for (uint32_t c = lane; c < n; c += 32) {
            if (MODE != 0) cd[c] = packed_code_distance<MODE>(p.store, qc, q_comp, cid[c]);
            else if (p.store.direct_cosine) cd[c] = pq_direct_cosine(p.store, qf, dim, cid[c]);
            else cd[c] = pq_table_distance(p.store, lut, cid[c]);
        }
        __syncwarp();
    }
};

}  // namespace dab
