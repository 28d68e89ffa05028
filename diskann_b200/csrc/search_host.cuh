// search_host.cuh — the host protocol of full-precision and quantized graph search (defined in search_kernel.cu): argument
// checks, the size of the per-warp visited tables in global memory, re-runs of the queries that outgrow them, host buffers.
#pragma once

#include "dab_common.cuh"

#include <functional>

namespace dab {

// k, L and beam of a search call; `need_vectors`: the search reads the full-precision rows (the quantized traversal
// reads only the graph and its codes)
int check_search_args(const dab_index* idx, uint32_t k, uint32_t l_search, uint32_t beam, bool need_vectors = true);

// Ids a warp's visited table holds in the first global-table pass at (L, beam, mode): the reference's estimate, or less
// where `hint` has seen the visited sets of this (or a larger) L and beam.  A default VisitedHint is no hint.
uint64_t table_slots(const dab_index* idx, const VisitedHint& hint, uint32_t l_search, uint32_t beam, int mode);
// `hint` takes in the largest visited set of a pass at (L, beam, mode)
void learn_visited(VisitedHint& hint, uint32_t l_search, uint32_t beam, int mode, uint32_t visited);
// After a global-table pass `pass` that overflowed: the table of the next one, or DAB_ERR_VISITED_OVERFLOW after six
int grow_visited_tables(const dab_index* idx, int& pass, uint64_t& slots);
// The `n_over` query ids a pass reported at `d_overflow` become the work list of the next pass, in `retry`
int take_overflow_list(cudaStream_t stream, const uint32_t* d_overflow, uint32_t n_over, Scratch& retry);

// Where a batch's results go: ids and dists [nq][k]; counts, cmps and hops [nq], optional
struct SearchOut {
    uint32_t* ids;
    float* dists;
    uint32_t *counts, *cmps, *hops;
};

// The synchronous host-buffer calls: checks the buffers, copies the queries to the handle's scratch, runs `run` on them
// with device result buffers, copies the results to `out` and waits.  `api` names the entry point in error messages.
int search_host_buffers(dab_index* idx, const char* api, const void* queries, uint32_t nq, uint32_t k, const SearchOut& out,
                        const std::function<int(const void* d_queries, const SearchOut& d_out)>& run);

}  // namespace dab
