// dab_common.cuh — shared host-side plumbing for libdiskann_b200.so (index handle, error
// reporting, launch accounting).  Compiled for sm_90a (H100) only.
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>

#include "../../include/diskann_b200.h"

struct dab_index;

namespace dab {

constexpr uint32_t kNoId = 0xFFFFFFFFu;

// the quantized stores of an index, numbered as the MODE of the quantized traversals (search_kernel_pq.cu)
enum QuantStore { STORE_PQ = 0, STORE_SQ = 1, STORE_MINMAX = 2 };

// thread-local error message (dab_last_error)
char* error_buffer();
int fail(int code, const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;
void comm_release(struct ::dab_index* idx);  // replicate.cu
void tc_release(struct ::dab_index* idx);    // flat_tc.cu
void search_slots_release(struct ::dab_index* idx);  // search_kernel.cu
// search_kernel.cu: called by every call that frees or reallocates a quantized store (PQ table and codes, SQ or MinMax
// rows), before it frees anything: waits for every slot's stream and bumps dab_index::stores_version, so that a batch in
// flight whose overflowed queries still need a pass fails in dab_wait instead of launching on the freed buffers
int retire_quantized_stores(struct ::dab_index* idx);
void minmax_release(struct ::dab_index* idx);        // minmax_index.cu: the store's transform
void paged_release(struct ::dab_index* idx);         // search_paged.cu: every paged search session still open
void attributes_release(struct ::dab_index* idx);    // search_diverse.cu: the attribute table
void labels_release(struct ::dab_index* idx);        // search_filtered.cu: the label table
void range_release(struct ::dab_index* idx);         // search_range.cu: every range search result set still open
// delete_kernels.cu: the deletion table.  deleted_assign replaces it with `words` ((n_total + 31) / 32 of them, bit i of
// word i / 32 for id i) holding n_deleted set bits; n_deleted == 0 clears it (words may then be NULL).
int deleted_assign(struct ::dab_index* idx, const uint32_t* words, uint64_t n_deleted);
int deleted_alloc(struct ::dab_index* idx);  // both copies of the table, every bit clear (nothing when they exist)
void deleted_release(struct ::dab_index* idx);
// the device bitmap the searches filter with while some id is deleted, else NULL
const uint32_t* deleted_filter(const struct ::dab_index* idx);
// marks the n ids (data points) deleted in both copies of the table (dab_delete without its checks)
int deleted_mark(struct ::dab_index* idx, const uint32_t* ids, uint64_t n);
// adj[ids[i]] <- the empty list, for the n device ids, queued on the index stream
int clear_rows(const struct ::dab_index* idx, const uint32_t* d_ids, uint64_t n);
// The calls that change the deletion table or consolidate wait for no batch: "<api>: slot i holds a batch in flight"
// while one does
int refuse_in_flight(const struct ::dab_index* idx, const char* api);

#define DAB_CUDA(expr)                                                                        \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess)                                                                \
            return ::dab::fail(_e == cudaErrorMemoryAllocation ? DAB_ERR_OUT_OF_MEMORY         \
                                                               : DAB_ERR_CUDA,               \
                               "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),        \
                               __FILE__, __LINE__);                                           \
    } while (0)

#define DAB_LAUNCHED() (::dab::g_launches.fetch_add(1, std::memory_order_relaxed))

inline size_t elem_size(int dtype) {
    switch (dtype) {
        case DAB_F32: return 4;
        case DAB_F16: return 2;
        default: return 1;
    }
}
inline size_t round_up(size_t x, size_t m) { return (x + m - 1) / m * m; }

// CTAs of `threads` threads with `smem` B of dynamic shared memory (the kernel's attribute is set to it) that one SM holds
// at once; 0 when the kernel does not fit, with the CUDA error cleared so that the caller reports its own
template <class P>
int ctas_per_sm(void (*kern)(P), int threads, size_t smem) {
    int per_sm = 0;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return per_sm;
}

// A device buffer owned by one call, freed when it goes out of scope (cudaFree waits for the whole device).  alloc()
// frees what it held and allocates n bytes; on failure "<who>: cudaMalloc(n) failed".
struct DevBuf {
    void* p = nullptr;
    ~DevBuf() { cudaFree(p); }
    int alloc(size_t n, const char* who = "build") {
        cudaFree(p);
        p = nullptr;
        cudaError_t e = cudaMalloc(&p, n ? n : 1);
        if (e != cudaSuccess) return fail(DAB_ERR_OUT_OF_MEMORY, "%s: cudaMalloc(%zu) failed: %s", who, n, cudaGetErrorString(e));
        return DAB_OK;
    }
};

// code_store.cu: blocks of 256 threads for `work` threads, at most 16 per SM (grid-stride kernels)
int grid_for(const struct ::dab_index* idx, uint64_t work);

// A grow-only device (or pinned host) scratch buffer.
struct Scratch {
    void* p = nullptr;
    size_t bytes = 0;
    bool pinned_host = false;
    int reserve(size_t n);
    void release();
};

// Test hooks, read from the environment ONCE at dab_create: they let tests reach paths the default inputs do not
// (neither changes results).
struct Tuning {
    int test_visited_log2 = 0;        // DAB_TEST_VISITED_LOG2: tests force the overflow / retry path
    bool test_pq_global_lut = false;  // DAB_TEST_PQ_GLOBAL_LUT: PQ kernels with the per-warp table in global memory also where the pivots fit shared memory
    uint32_t test_diverse_pool = 0;   // DAB_TEST_DIVERSE_POOL: local-queue entries of a diverse search's first pass (tests force its re-runs)
    uint32_t test_range_list = 0;     // DAB_TEST_RANGE_LIST: in_range entries per warp in a range search's first pass (tests force its re-runs)
    uint64_t test_range_arena = 0;    // DAB_TEST_RANGE_ARENA: entries of a range search's first result arena (tests force its extension)
    uint64_t test_range_limit = 0;    // DAB_TEST_RANGE_LIMIT: most entries a range search may hold (tests reach its out-of-memory failure)
    void load();
};

// The largest visited set the searches at (l, beam, mode) have seen; later calls size their visited tables from it
// (search_kernel.cu).  `mode`: which quantized store the traversal reads (full precision shares STORE_PQ: the two keep separate
// hints, dab_index::hint and pq_hint).
struct VisitedHint {
    uint32_t l = 0, beam = 0, visited = 0;
    QuantStore mode = STORE_PQ;
};

// A store of dense N-bit code rows, one per point (the SQ and MinMax stores of an index).  Host-facing rows use the
// reference's canonical-front layout (meta/vector.rs): a header — an optional u32 dim word, then meta_words f32 — and
// ceil(dim * nbits / 8) bytes of dense codes, value i at bit i * nbits (bits/slice.rs:261-323).  On the device the codes
// are 16 B-aligned rows, zero padded (the integer cores read whole words), and the header's floats a separate
// [n_total][meta_words] array; the dim word is checked on upload and not stored.  code_store.cu moves rows between the
// two layouts.
struct CodeStore {
    int nbits = 0;                // 0: not set up
    uint32_t dim = 0;             // codes per row
    bool dim_word = false;        // the header starts with a u32 dim word
    uint32_t meta_words = 0;      // f32 per row after it
    uint32_t row_bytes = 0;       // canonical row: header + codes
    uint32_t stride = 0;          // device code row
    uint8_t* d_codes = nullptr;   // [n_total][stride]
    float* d_meta = nullptr;      // [n_total][meta_words]
    bool ready = false;           // rows uploaded or encoded
    __host__ __device__ uint32_t header_bytes() const { return (dim_word ? 4u : 0u) + meta_words * 4u; }
};

// code_store.cu
// Releases `s`, then allocates it for n_total rows of `dim` codes of `nbits`, zeroed and not ready.
int store_alloc(struct ::dab_index* idx, CodeStore& s, int nbits, uint32_t dim, bool dim_word, uint32_t meta_words);
void store_release(CodeStore& s);
// "<who>: idx is NULL", or "<who>: <upload> has not been called" while the store is not set up
int store_require(const struct ::dab_index* idx, CodeStore dab_index::*store, const char* upload, const char* who);
// n canonical rows (device memory) -> codes [n][s.stride] and meta [n][s.meta_words], queued on `stream`.  The bits
// past dim * nbits in a row's last code byte are cleared.  first_bad (device, may be NULL) takes the first row whose dim
// word is not s.dim.
int store_split(const struct ::dab_index* idx, cudaStream_t stream, const CodeStore& s, const uint8_t* rows, uint64_t n, uint8_t* codes,
                float* meta, unsigned long long* first_bad);
// every row from host canonical rows, staged in slabs; fails naming the first row whose dim word is not s.dim
int store_upload(struct ::dab_index* idx, CodeStore& s, const uint8_t* rows, const char* who);
// every row back to host canonical rows, byte for byte what the store holds
int store_download(struct ::dab_index* idx, const CodeStore& s, uint8_t* rows);
// The staging scratch `stage` of a packed-code search batch: `work` bytes for the quantizer, then the compressed queries,
// codes [nq][s.stride] and one float4 per query.
int stage_query_buffers(const CodeStore& s, Scratch& stage, uint32_t nq, size_t work, uint8_t** codes, float4** meta);
// the bytes stage_query_buffers reserves
size_t stage_query_bytes(const CodeStore& s, uint32_t nq, size_t work);
// T::as_f32 of n rows of the index dtype, src_stride bytes apart -> dst [n][dim], queued on `stream`
int widen_rows(const struct ::dab_index* idx, cudaStream_t stream, const void* src, size_t src_stride, uint64_t n, float* dst);

// The store encoders over n rows of the index dtype, src_stride bytes apart, into any codes / meta arrays ([n] rows at
// the store's device layout), queued on `stream`.
// quant_kernels.cu: BasicTable::compress_into of n f32 rows on the idx stream (synchronizes); fails naming the first row
// infinitely far from every centre, numbered from first_row
int pq_encode_device(struct ::dab_index* idx, const float* d_vectors, uint64_t n, uint8_t* d_codes_out, uint64_t first_row);
// sq_index.cu: SQStore::set_vector
int sq_encode_rows(const struct ::dab_index* idx, cudaStream_t stream, const uint8_t* src, size_t src_stride, uint64_t n, uint8_t* codes,
                   float* comp);
// minmax_index.cu: as_f32 -> transform -> compress, in `work` (minmax_encode_bytes(idx, n) bytes); *h_first_nan (host,
// valid once the stream is synchronized) takes the first row whose transformed vector holds a NaN, else ~0
size_t minmax_encode_bytes(const struct ::dab_index* idx, uint64_t n);
int minmax_encode_rows(const struct ::dab_index* idx, cudaStream_t stream, uint8_t* work, const void* src, size_t src_stride, uint64_t n,
                       uint8_t* codes, float* meta, unsigned long long* h_first_nan);

// insert_rows.cu, for dab_insert: "<who>: ..." naming the first id that is not a data point, repeats or is deleted
int insert_check_ids(const struct ::dab_index* idx, const uint32_t* ids, uint64_t n, const char* who);
// rows[i] -> row ids[i] of the index and of every quantized store that holds rows, encoded as the encode-all calls
// encode; every encoder check runs before anything is written
int insert_rows(struct ::dab_index* idx, const uint32_t* ids, const void* rows, uint64_t n, const char* who);

}  // namespace dab

struct dab_index {
    int dtype = 0, metric = 0;
    uint32_t dim = 0;
    uint64_t n_points = 0;
    uint32_t n_start = 0;
    uint32_t max_degree = 0;
    int device = 0;
    int sm_count = 132;
    int l2_bytes = 50 << 20;  // the device's L2 cache

    cudaStream_t stream = nullptr;      // stream in use
    cudaStream_t own_stream = nullptr;  // library-created

    // HBM-resident snapshot
    uint8_t* d_vectors = nullptr;  // (n_points + n_start) rows, row_stride bytes apart
    size_t row_stride = 0;         // round_up(dim * sizeof(T), 32): rows start on sector bounds
    uint32_t* d_adj = nullptr;     // (n_points + n_start) rows of adj_stride words: [len, ids...]
    uint32_t adj_stride = 0;       // round_up(max_degree + 1, 8) words (32 B multiple)
    bool vectors_ready = false, graph_ready = false;

    // product quantization
    float* d_pivots = nullptr;     // [n_centers][dim]
    uint32_t* d_offsets = nullptr; // [n_chunks + 1]
    uint8_t* d_codes = nullptr;    // [n_total][n_chunks]
    uint32_t pq_chunks = 0, pq_centers = 0;
    uint32_t pq_uniform_len = 0;   // every chunk has this many dimensions (0: lengths differ)
    bool pq_codes_ready = false;   // codes uploaded (dab_upload_pq) or produced (dab_pq_encode_all)
    // packed-code stores: scalar-quantized (sq_index.cu; providers inmem/scalar.rs SQStore<NBITS>), rows of index dim
    // codes with one f32 compensation (only the inner-product epilogue reads it); MinMax (minmax_index.cu; providers
    // common/minmax_repr.rs MinMaxElement<NBITS>), rows of the transform's output dim with {b, n, a, norm_squared}
    dab::CodeStore sq, mm;
    // the scalar quantizer
    float sq_scale = 0.0f, sq_shift_square_norm = 0.0f, sq_mean_norm = 0.0f;
    float* d_sq_shift = nullptr;  // [dim]
    // the MinMax quantizer: grid scale, its own copy of the transform with the tables on the device
    float mm_grid_scale = 0.0f;
    dab_transform* mm_transform = nullptr;  // NULL: Transform::Null
    uint32_t* d_mm_tables = nullptr;        // transform_tables(mm_transform)

    // scratch (grow-only)
    dab::Scratch s_queries, s_ids, s_out, s_out2, s_tables, s_counters, s_stats;
    dab::Scratch s_stage;  // packed-code store upload / encode / download staging, and the SQ and MinMax searches' compressed queries
    dab::Scratch s_pools;  // the local queues of diverse search (search_diverse.cu), or a filtered search's masks and adaptive-L table
    dab::Scratch h_stage;  // pinned host staging
    dab::Scratch h_counters;  // pinned: the four counters a search pass reports
    void* slots[DAB_MAX_SLOTS] = {};  // batches in flight (dab_search_batch_async), search_kernel.cu

    // search-side state learned across calls
    dab::VisitedHint hint, pq_hint;  // full precision; PQ / SQ / MinMax traversal (visits other nodes: kept apart)
    uint32_t v3_overflow_l = 0, v3_overflow_beam = 0;      // share of queries that outgrew the shared-memory
    float v3_overflow_frac = 0.0f;                         // tables at (L, beam): search_kernel_v3 is skipped when large

    uint64_t stores_version = 0;  // bumped whenever a quantized store is freed or reallocated (retire_quantized_stores)
    // bumped by every upload of rows or adjacency, dab_build and the broadcasts: a paged search session that began under
    // another generation fails its next page (search_paged.cu)
    uint64_t generation = 0;
    // one write counter per quantized store, indexed by dab::QuantStore: bumped by every call that writes the store
    // (upload, encode-all, PQ training, broadcast).  Only paged search sessions over that store read it.
    uint64_t store_writes[3] = {};
    void* paged = nullptr;  // the open paged search sessions (a list, search_paged.cu)
    dab_range* ranges = nullptr;  // the open range search result sets (a list, search_range.cu)
    // the deletion table (delete_kernels.cu; providers TableDeleteProviderAsync): one bit per id, kept on the host and
    // copied to the device after every change.  Both are allocated by the first dab_delete; n_deleted counts set bits.
    uint32_t* h_deleted = nullptr;  // (n_total + 31) / 32 words
    uint32_t* d_deleted = nullptr;
    uint64_t n_deleted = 0;
    uint64_t rec_truncated = 0;  // build: searches whose expanded-node record was cut at its capacity
    // the attribute table of diverse search (search_diverse.cu): one value and one presence bit per id, allocated by the
    // first dab_upload_attributes (nothing present).  Independent of the graph: inserts, deletes and releases leave it.
    uint32_t* d_attr_values = nullptr;   // [n_total]
    uint32_t* d_attr_present = nullptr;  // (n_total + 31) / 32 words
    uint32_t* h_attr_present = nullptr;  // the host copy of the presence bits
    // the label table of filtered search (search_filtered.cu): one 64-bit label set per id, allocated by the first
    // dab_upload_labels (every set empty).  Independent of the graph, as the attribute table is.
    uint64_t* d_labels = nullptr;  // [n_total]
    dab::Tuning tune;

    // tensor-core exhaustive scan (flat_tc.cu): bf16 operand copy of the rows + score coefficients
    void* d_tc_base = nullptr;
    void* d_tc_coef = nullptr;
    uint64_t tc_version = 0, vectors_version = 1;  // the copy is rebuilt when rows were uploaded since

    // replication (replicate.cu): NCCL communicator of a one-process-per-GPU host
    void* nccl_comm = nullptr;
    int nccl_rank = 0, nccl_ranks = 0;

    uint64_t n_total() const { return n_points + n_start; }
    uint64_t deleted_words() const { return (n_total() + 31) / 32; }
};
