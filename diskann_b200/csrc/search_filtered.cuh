// search_filtered.cuh — parameter block and host entry points of the label-filtered traversal (search_filtered.cu), run
// as one kind of the search job (SlotJob, search_kernel.cu).
#pragma once

#include "dab_common.cuh"
#include "search_host.cuh"
#include "search_source.cuh"

#include <vector>

namespace dab {

constexpr int kFiltWarps = 4;
// the longest list a filtered search keeps: L + #start, and floor(L * scale) once adaptive L has grown it
constexpr uint32_t kFilteredMaxL = 1024;
// a CTA's shared memory may not pass this: kFiltWarps x (the query, 2 x the longest list, 2 x L matched entries,
// 3 x beam_width x max_degree candidate words, the beam)
constexpr size_t kFilteredMaxSmem = 200 * 1024;

struct SearchParamsFiltered {
    const uint32_t* adj;
    uint32_t adj_stride;
    uint64_t n_points;
    uint32_t n_start;
    uint32_t dim;
    uint32_t max_degree;
    const uint8_t* vectors;
    size_t row_stride;
    const void* queries;
    const uint32_t* query_list;
    uint32_t n_work;
    uint32_t k, cap, beam;  // cap: L, the matched entries kept
    uint32_t* out_ids;
    float* out_dists;
    uint32_t *out_counts, *out_cmps, *out_hops;
    uint32_t* tables;
    uint32_t n_buckets;
    uint32_t* counters;
    uint32_t* overflow_list;
    const uint64_t* labels;  // [n_total] (dab_upload_labels)
    const uint64_t* masks;   // [nq]
    uint32_t match_all;      // 0: ANY (labels & mask != 0), else ALL (labels & mask == mask)
    uint32_t best_cap;       // the list's first capacity, L + #start
    // adaptive L: samples == 0 is off.  Once `samples` neighbours were evaluated, the hop's (visited, matched) picks
    // the new L in adapt[(visited - samples) * (samples + span) + matched], span = beam * max_degree
    uint32_t samples, span;
    const uint16_t* adapt;
    uint32_t warp_smem, off_bd, off_bi, off_md, off_mi, off_cid, off_cd, off_ca, off_beam;
    StoreParams store;  // the quantized traversals (filtered_kernel_quant)
    // with rerank: the matched list of every query (at most L ids, start points included) for launch_rerank
    uint32_t* list_ids;     // [nq][list_cap]
    uint32_t* list_counts;  // [nq]
    uint32_t list_cap;
};

// What a filtered batch adds to a k-NN batch: the device masks, the mode and adaptive L's table on the device (`adapt`,
// NULL when adaptive L is off or its sample is never reached); best_max: the longest the list can become
struct FilterSpec {
    const uint64_t* masks;
    uint32_t match_all;
    uint32_t samples;
    const uint16_t* adapt;
    uint32_t best_max;
};

// compute_adaptive_l (inline_filter_search.rs:294-310) in the same f64 expression
uint32_t adaptive_l(uint32_t base_l, uint64_t visited, uint64_t matched, double scale);
// The table of new L values for every (visited, matched) pair a query can reach when the sample fires: `span` rows
// (visited = samples .. samples + span - 1) of samples + span entries (matched = 0 ..)
std::vector<uint16_t> adaptive_table(uint32_t l_search, uint32_t samples, uint32_t span, double scale);

// "<api>: ... need N B shared memory per CTA" unless a list of best_max entries, L matched entries and beam_width fit
// kFilteredMaxSmem on this index for a traversal over `store` (-1: full precision, else a QuantStore); no device work
int filtered_check_smem(const dab_index* idx, const char* api, uint32_t l_search, uint32_t best_max, uint32_t beam, int store = -1);

// The kernel of this index's schema (store -1) or of `store`, and its shape in CTAs of kFiltWarps warps; fills p's
// shared-memory offsets
int filtered_plan(const dab_index* idx, uint32_t l_search, uint32_t best_max, uint32_t beam, int store, SearchParamsFiltered& p,
                  WarpPlan<SearchParamsFiltered>& plan);

}  // namespace dab
