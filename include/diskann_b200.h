/*
 * diskann_b200.h — C ABI of the H100-native distance hot path for microsoft/DiskANN (DiskANN3).
 *
 * This is the drop-in boundary (SURVEY.md §8b): a plain-C shared library
 * (libdiskann_b200.so, sm_90a CUDA inside) whose entry points are what a Rust `-sys` crate
 * for this path binds.  Conventions mirror the reference's only FFI precedent,
 * diskann-garnet/src/lib.rs:262-630: opaque handle, (pointer, length) pairs, integer status,
 * no unwinding across the boundary, caller owns every host buffer, the library owns device
 * memory.  INTEGRATION.md shows the reference-side binding.
 *
 * Each entry point cites the reference interface it replaces (paths relative to the
 * reference checkout).
 *
 * Value conventions are the reference's (diskann-vector/src/distance/distance_provider.rs:
 * 30-43, implementations.rs:217-404): L2 -> sum (x-y)^2 (no sqrt); InnerProduct -> -sum xy;
 * Cosine -> 1 - cos (clamped); CosineNormalized -> 1 - sum xy (== Cosine for i8/u8).
 * Float results are bit-identical to the reference's x86-64-v3 SIMD order; integer and PQ
 * results are exact.
 */
#ifndef DISKANN_B200_H
#define DISKANN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* element types: diskann/src/utils/vector_repr.rs:117-190 (f32, f16, i8, u8) */
enum { DAB_F32 = 0, DAB_F16 = 1, DAB_I8 = 2, DAB_U8 = 3 };

/* diskann-vector/src/distance/metric.rs:8-20, #[repr(C)] values */
enum { DAB_COSINE = 0, DAB_INNER_PRODUCT = 1, DAB_L2 = 2, DAB_COSINE_NORMALIZED = 3 };

/* status codes (0 == ok); dab_last_error() has the message (maps to ANNError::message) */
enum {
    DAB_OK = 0,
    DAB_ERR_INVALID_ARGUMENT = 1, /* bad dtype/metric/length: layers/full.rs:203-213, 306-314 */
    DAB_ERR_CUDA = 2,
    DAB_ERR_OUT_OF_MEMORY = 3,
    DAB_ERR_VISITED_OVERFLOW = 4, /* per-query visited set exceeded its capacity (retried internally) */
    DAB_ERR_NOT_READY = 5,        /* e.g. search before vectors/graph were uploaded */
    DAB_ERR_NO_DEVICE = 6
};

typedef struct dab_index dab_index; /* opaque */

/* ------------------------------------------------------------------ lifecycle */

/* Replaces diskann_inmem::Provider::new(layer, config, start_points)
 * (diskann-inmem/src/provider.rs:71-131) + layers::Full::<T>::new(dim, metric)
 * (diskann-inmem/src/layers/full.rs:368-504) for the device-resident snapshot:
 * n_points data rows (ids [0, n_points)) + n_start frozen start rows
 * (ids [n_points, n_points + n_start)), adjacency rows of max_degree + 1 words. */
int dab_create(dab_index** out, int dtype, int metric, uint32_t dim, uint64_t n_points,
               uint32_t n_start, uint32_t max_degree, int device);
void dab_destroy(dab_index* idx);

/* thread-local message of the last failing call on this thread */
const char* dab_last_error(void);

/* Launch on the caller's CUDA stream (cudaStream_t passed as void*); NULL restores the
 * library's own stream. */
int dab_set_stream(dab_index* idx, void* cuda_stream);

/* number of kernels this library has launched in this process (bench.py "gpu_launches") */
uint64_t dab_launch_count(void);

/* ------------------------------------------------------------------ data upload */

/* layers::Set<T>::set(element, bytes) (diskann-inmem/src/layers/mod.rs:79-96) /
 * Provider::set_element (provider.rs:341-372): dense row-major rows of dim elements, no
 * tags.  `first` may address start rows (first >= n_points).  Host or device source. */
int dab_upload_vectors(dab_index* idx, const void* rows, uint64_t first, uint64_t count);
int dab_upload_vectors_device(dab_index* idx, const void* d_rows, uint64_t first, uint64_t count);

/* Neighbors buffer (diskann-inmem/src/neighbors.rs:69-163): row = [len, id_0 .. id_{len-1}],
 * src_stride words between source rows (>= max_degree + 1). */
int dab_upload_graph(dab_index* idx, const uint32_t* adj, uint32_t src_stride, uint64_t first,
                     uint64_t count);
int dab_upload_graph_device(dab_index* idx, const uint32_t* d_adj, uint32_t src_stride,
                            uint64_t first, uint64_t count);
int dab_download_graph(dab_index* idx, uint32_t* adj, uint32_t dst_stride, uint64_t first,
                       uint64_t count);

/* FixedChunkPQTable::new(dim, pq_table, chunk_offsets)
 * (diskann-providers/src/model/pq/fixed_chunk_pq_table.rs:104-135) + the compressed
 * vectors of the quant store: pivots [n_centers][dim] f32, offsets [n_chunks + 1],
 * codes [(n_points + n_start)][n_chunks] (may be NULL, then call dab_pq_encode_all; a PQ
 * traversal before that returns DAB_ERR_NOT_READY). */
int dab_upload_pq(dab_index* idx, const float* pivots, uint32_t n_centers,
                  const uint64_t* offsets, uint32_t n_chunks, const uint8_t* codes);

/* train_pq (diskann-providers/src/index/diskann_async.rs:61-89 -> model/pq/pq_construction.rs:163-243
 * -> diskann-quantization/src/product/train.rs): per chunk k-means++ seeding
 * (algorithms/kmeans/plusplus.rs:381-498) and `lloyds_reps` Lloyd iterations (lloyds.rs:372-426; the
 * benchmark uses 5) over n host training rows [n][dim] f32, entirely on the device, arithmetic in the
 * reference's order.  Chunk offsets are ChunkOffsets::partition (quantization/src/views.rs:226-243).
 * The random draws come from SplitMix64(seed + chunk) (the reference's StdRng is not reproduced).
 * Replaces the resident table; codes are cleared until dab_pq_encode_all. */
int dab_pq_train(dab_index* idx, const float* train, uint64_t n, uint32_t n_chunks, uint32_t n_centers,
                 uint32_t lloyds_reps, uint64_t seed);
/* BasicTable::compress_into (product/tables/basic.rs:161-194) for every uploaded row (converted to
 * f32, T: Into<f32>) into the resident codes — the quant store of a quantized build. */
int dab_pq_encode_all(dab_index* idx);
/* copies the resident table back: pivots [n_centers][dim], offsets [n_chunks + 1], codes
 * [(n_points + n_start)][n_chunks]; any pointer may be NULL. */
int dab_pq_download(dab_index* idx, float* pivots, uint64_t* offsets, uint8_t* codes);

/* ------------------------------------------------------------------ replication across GPUs */

/* The index is replicated, the query batch is sharded, the search path has no collective
 * (benchmark-core/src/search/api.rs:410-419 partitions queries over tasks the same way; SURVEY.md §8e).
 * One NCCL broadcast per resident buffer (vectors, adjacency, PQ table and codes) at load.  NCCL is
 * resolved with dlopen("libnccl.so.2") at first use; DAB_ERR_NOT_READY if it cannot be loaded.
 * One process per GPU: rank 0 calls dab_comm_unique_id and ships the 128 bytes to the other ranks,
 * every rank calls dab_comm_init on its own handle (created with the same shape), then
 * dab_broadcast_index(idx, root).  dab_destroy releases the communicator. */
int dab_comm_unique_id(char* out_id128);
int dab_comm_init(dab_index* idx, const char* id128, int n_ranks, int rank);
int dab_broadcast_index(dab_index* idx, int root);
int dab_comm_destroy(dab_index* idx);
/* One process driving several GPUs: per_gpu[0] is the root, per_gpu[i] lives on its own device. */
int dab_broadcast(dab_index* const* per_gpu, int n_gpus);

/* ------------------------------------------------------------------ (1) per-pair / per-query distances */

/* DistanceProvider::distance_comparer(metric, dim) -> Distance<T,U>::call
 * (diskann-vector/src/distance/distance_provider.rs:44-46, 86) and
 * layers::Distance::evaluate(x, y) (diskann-inmem/src/layers/mod.rs:68-77): n independent
 * pairs x[i] . y[i], host buffers, dense rows.  Supported (dtype_x, dtype_y): (f32,f32)
 * (f16,f16) (f32,f16) (i8,i8) (u8,u8).  Stateless: no index needed. */
int dab_pair_distances(int dtype_x, int dtype_y, int metric, uint32_t dim, const void* x,
                       const void* y, uint64_t n, float* out, int device);

/* SearchAccessor::expand_beam's distance stage batched over queries
 * (diskann-inmem/src/provider.rs:436-479, 620-690; glue.rs:210-219):
 * out[q][j] = QueryDistance(query q).evaluate(row ids[q][j]); ids == UINT32_MAX are skipped
 * (out = NaN).  Queries have the index dtype (f16 queries are widened once,
 * layers/full.rs:421-423). */
int dab_distances(dab_index* idx, const void* queries, uint32_t nq, const uint32_t* ids,
                  uint32_t c, float* out);
int dab_distances_device(dab_index* idx, const void* d_queries, uint32_t nq,
                         const uint32_t* d_ids, uint32_t c, float* d_out);

/* PruneAccessor::fill + Distance: DistanceFunction<ElementRef, ElementRef>
 * (diskann/src/graph/glue.rs:855-906; index.rs:2623-2625): data x data distances.
 * out[i] = Distance<T,T>(row a[i], row b[i]). */
int dab_row_pair_distances(dab_index* idx, const uint32_t* a, const uint32_t* b, uint64_t n,
                           float* out);
/* candidate x candidate block for robust_prune: out[i][j] = Distance<T,T>(ids[i], ids[j]) */
int dab_pairwise(dab_index* idx, const uint32_t* ids, uint32_t n, float* out);

/* ------------------------------------------------------------------ (3') batched greedy search */

/* DiskANNIndex::search_internal + Knn::search + post-process for a whole query batch
 * (diskann/src/graph/index.rs:1933-2000; graph/search/knn_search.rs:170-190;
 * diskann-inmem/src/provider.rs:907-950), i.e. benchmark_core::search::graph::KNN::search
 * (diskann-benchmark-core/src/search/graph/knn.rs:208-238) for every query at once.
 * Results exclude start points; rows are padded with id UINT32_MAX / distance +inf;
 * out_counts/out_cmps/out_hops may be NULL.  cmps/hops follow SearchStats
 * (index.rs:1990-1991). */
int dab_search_batch(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                     uint32_t beam_width, uint32_t* out_ids, float* out_dists,
                     uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops);
int dab_search_batch_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k,
                            uint32_t l_search, uint32_t beam_width, uint32_t* d_out_ids,
                            float* d_out_dists, uint32_t* d_out_counts, uint32_t* d_out_cmps,
                            uint32_t* d_out_hops);

/* ------------------------------------------------------------------ (3''') diverse search */

/* The attribute table of diverse search: AttributeValueProvider::get
 * (diskann/src/neighbor/diverse_priority_queue.rs:265-279) as one u32 value and one presence
 * bit per id, over every id of the index (start points included).  Ids [first, first + count)
 * take values[i]; present[i] != 0 marks id first + i as having an attribute (present NULL: all
 * of them), present[i] == 0 as having none.  first + count <= n_points + n_start.  The first
 * call allocates the table with no id present.  The table is independent of the graph: inserts,
 * deletes and releases neither read nor clear it (an inserted point has what was uploaded for
 * its id). */
int dab_upload_attributes(dab_index* idx, const uint32_t* values, const uint8_t* present,
                          uint64_t first, uint64_t count);

/* Diverse::search (diskann/src/graph/search/diverse_search.rs:189-234) for a whole query batch:
 * search_internal with a DiverseNeighborQueue (neighbor/diverse_priority_queue.rs:90-220) of L
 * entries and one local queue of diverse_k * L / k entries per attribute value, then its
 * post_process (at most diverse_k entries per attribute value stay in the list) and the k-NN
 * post-processing of the first L entries (start points and deleted ids dropped, the first k kept).
 * Ids without an attribute never enter the list; they are still visited and counted in cmps.
 * Full-precision rows of every dtype and metric; k >= 1, diverse_k >= 1 (diverse_k > k is
 * accepted, as in the reference), k <= l_search <= 1024, 1 <= beam_width <= 64, a CTA's shared
 * memory fits 200 KB: 4 x (query row (f32 for float rows, the bytes for i8 / u8) + 12 * l_search
 * + 8 * beam_width * max_degree + 4 * beam_width bytes, each part rounded up to 16, the whole to
 * 128), and an attribute table must have been uploaded: each is checked before any device work
 * and fails with DAB_ERR_INVALID_ARGUMENT and a message.  Outputs as dab_search_batch. */
int dab_search_batch_diverse(dab_index* idx, const void* queries, uint32_t nq, uint32_t k,
                             uint32_t l_search, uint32_t beam_width, uint32_t diverse_k,
                             uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                             uint32_t* out_cmps, uint32_t* out_hops);
/* the same with device buffers; returns with the outputs complete */
int dab_search_batch_diverse_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k,
                                    uint32_t l_search, uint32_t beam_width, uint32_t diverse_k,
                                    uint32_t* d_out_ids, float* d_out_dists,
                                    uint32_t* d_out_counts, uint32_t* d_out_cmps,
                                    uint32_t* d_out_hops);

/* Diverse::search over a quantized store (diverse_search.rs:189-234 with the quantized strategy):
 * the traversal distances are those of dab_search_batch_pq / _sq / _minmax on the same store (PQ:
 * TableL2 / TableIP, DirectCosine for Metric::Cosine; SQ and MinMax: the queries compressed by the
 * store's quantizer), the list and the local queues run as in dab_search_batch_diverse, and
 * best.post_process() keeps at most diverse_k entries per attribute value.
 *   rerank == 0: the default post-processing of the first L entries (start points and deleted ids
 *     dropped, the first k kept) with their quantized distances;
 *   rerank != 0: Pipeline<FilterStartPoints, Rerank> over the post-processed list (providers
 *     inmem/product.rs:391-400, full_precision.rs:356-399): each remaining entry that is not
 *     deleted gets its full-precision distance, the list is sorted by it (ties keep list order)
 *     and the first k are kept.  The diverse limit holds: the rerank reorders a subset of the list.
 * cmps / hops follow SearchStats as in dab_search_batch_diverse.  Checked before any device work:
 * the arguments of dab_search_batch_diverse (the shared memory with the query area the f32 query
 * for PQ, the store's code row + 16 bytes for SQ and MinMax), then the store checks of the
 * synchronous quantized call (store uploaded with rows, no Metric::Cosine on the SQ store, rerank
 * only with the full-precision vectors uploaded); a MinMax query that holds a NaN after the
 * transform fails the call.  Outputs as dab_search_batch; the _device forms return with the
 * outputs complete. */
int dab_search_batch_diverse_pq(dab_index* idx, const void* queries, uint32_t nq, uint32_t k,
                                uint32_t l_search, uint32_t beam_width, uint32_t diverse_k,
                                int rerank, uint32_t* out_ids, float* out_dists,
                                uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops);
int dab_search_batch_diverse_sq(dab_index* idx, const void* queries, uint32_t nq, uint32_t k,
                                uint32_t l_search, uint32_t beam_width, uint32_t diverse_k,
                                int rerank, uint32_t* out_ids, float* out_dists,
                                uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops);
int dab_search_batch_diverse_minmax(dab_index* idx, const void* queries, uint32_t nq, uint32_t k,
                                    uint32_t l_search, uint32_t beam_width, uint32_t diverse_k,
                                    int rerank, uint32_t* out_ids, float* out_dists,
                                    uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops);
int dab_search_batch_diverse_pq_device(dab_index* idx, const void* d_queries, uint32_t nq,
                                       uint32_t k, uint32_t l_search, uint32_t beam_width,
                                       uint32_t diverse_k, int rerank, uint32_t* d_out_ids,
                                       float* d_out_dists, uint32_t* d_out_counts,
                                       uint32_t* d_out_cmps, uint32_t* d_out_hops);
int dab_search_batch_diverse_sq_device(dab_index* idx, const void* d_queries, uint32_t nq,
                                       uint32_t k, uint32_t l_search, uint32_t beam_width,
                                       uint32_t diverse_k, int rerank, uint32_t* d_out_ids,
                                       float* d_out_dists, uint32_t* d_out_counts,
                                       uint32_t* d_out_cmps, uint32_t* d_out_hops);
int dab_search_batch_diverse_minmax_device(dab_index* idx, const void* d_queries, uint32_t nq,
                                           uint32_t k, uint32_t l_search, uint32_t beam_width,
                                           uint32_t diverse_k, int rerank, uint32_t* d_out_ids,
                                           float* d_out_dists, uint32_t* d_out_counts,
                                           uint32_t* d_out_cmps, uint32_t* d_out_hops);

/* ------------------------------------------------------------------ (3''''') filtered search */

/* The label table of filtered search: one 64-bit label set per id, over every id of the index
 * (start points included).  Ids [first, first + count) take labels[i];
 * first + count <= n_points + n_start.  The first call allocates the table with every set empty
 * (8 bytes per id).  The table is independent of the graph: inserts, deletes and releases neither
 * read nor clear it. */
int dab_upload_labels(dab_index* idx, const uint64_t* labels, uint64_t first, uint64_t count);

/* InlineFilterSearch::search (diskann/src/graph/search/inline_filter_search.rs:89-160) for a whole
 * query batch over full-precision rows of every dtype and metric.  Query q accepts id i when
 *   match_all == 0 (ANY): labels[i] & query_masks[q] != 0;
 *   match_all != 0 (ALL): labels[i] & query_masks[q] == query_masks[q] (an empty mask accepts all).
 * The traversal is the k-NN traversal of dab_search_batch (inline_filter_search_internal,
 * :166-282): every evaluated neighbour enters the list of L + n_start entries, accepted or not;
 * the accepted start points and neighbours are also kept as matches.  Results: the first L
 * matches by distance, start points and deleted ids dropped, the first k kept; a query can
 * return fewer than k.  Among matches at exactly equal distances an earlier match comes first
 * (the reference's sort_unstable leaves that order open), and NaN distances come last.  cmps
 * counts the evaluated neighbours (start points are not counted, as in the reference), hops the
 * expanded nodes.
 * adaptive_samples == 0: no AdaptiveL.  Otherwise AdaptiveL(adaptive_samples, adaptive_scale):
 * after the hop in which the evaluated neighbours reach adaptive_samples, L' =
 * compute_adaptive_l(L, evaluated, accepted, adaptive_scale) (:294-310), computed on the host in
 * the reference's f64 expression; when L' > L the list's capacity becomes L' and a longer list is
 * cut to L' (NeighborPriorityQueue::reconfigure, neighbor/queue.rs:339-353).
 * Checked before any device work, each failing with DAB_ERR_INVALID_ARGUMENT and a message: k >= 1,
 * k <= l_search, 1 <= beam_width <= 64, adaptive_scale >= 1.0 (when adaptive), a label table was
 * uploaded, l_search + n_start <= 1024 and floor(l_search * adaptive_scale) <= 1024 (when
 * adaptive), and a CTA's shared memory fits 200 KB: 4 x (query row (f32 for float rows, the bytes
 * for i8 / u8) + 8 * the longest list + 8 * l_search + 12 * max(beam_width * max_degree, 32) +
 * 4 * beam_width bytes, each part rounded up to 16, the whole to 128).  Outputs as
 * dab_search_batch; query_masks holds nq host words. */
int dab_search_batch_filtered(dab_index* idx, const void* queries, uint32_t nq, uint32_t k,
                              uint32_t l_search, uint32_t beam_width, const uint64_t* query_masks,
                              uint32_t match_all, uint32_t adaptive_samples, double adaptive_scale,
                              uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                              uint32_t* out_cmps, uint32_t* out_hops);
/* the same with device buffers, d_query_masks included; returns with the outputs complete */
int dab_search_batch_filtered_device(dab_index* idx, const void* d_queries, uint32_t nq,
                                     uint32_t k, uint32_t l_search, uint32_t beam_width,
                                     const uint64_t* d_query_masks, uint32_t match_all,
                                     uint32_t adaptive_samples, double adaptive_scale,
                                     uint32_t* d_out_ids, float* d_out_dists,
                                     uint32_t* d_out_counts, uint32_t* d_out_cmps,
                                     uint32_t* d_out_hops);

/* InlineFilterSearch::search over a quantized store (inline_filter_search.rs:89-160 with the
 * quantized strategy behind graph::ext::labeled::Filtered, labeled.rs:96-129): the traversal, the
 * matches and adaptive L are those of dab_search_batch_filtered, and the traversal distances are
 * those of dab_search_batch_pq / _sq / _minmax on the same store (PQ: TableL2 / TableIP,
 * DirectCosine for Metric::Cosine; SQ and MinMax: the queries compressed by the store's
 * quantizer).
 *   rerank == 0: the first L matches by store distance, start points and deleted ids dropped, the
 *     first k kept, with their store distances;
 *   rerank != 0: Pipeline<FilterStartPoints, Rerank> over the first L matches (providers
 *     inmem/product.rs:391-400, full_precision.rs:356-399): each match that is neither a start
 *     point nor deleted gets its full-precision distance, the matches are sorted by it (ties keep
 *     matched-list order) and the first k are kept with their full-precision distances.
 * A query can return fewer than k.  cmps / hops as in dab_search_batch_filtered.  Checked before
 * any device work: the arguments of dab_search_batch_filtered (the shared memory with the query
 * area the f32 query for PQ, the store's code row + 16 bytes for SQ and MinMax), then the store
 * checks of the synchronous quantized call (store uploaded with rows, no Metric::Cosine on the SQ
 * store, rerank only with the full-precision vectors uploaded); a MinMax query that holds a NaN
 * after the transform fails the call.  Outputs as dab_search_batch; the _device forms take
 * d_query_masks on the device and return with the outputs complete. */
int dab_search_batch_filtered_pq(dab_index* idx, const void* queries, uint32_t nq, uint32_t k,
                                 uint32_t l_search, uint32_t beam_width,
                                 const uint64_t* query_masks, uint32_t match_all,
                                 uint32_t adaptive_samples, double adaptive_scale, int rerank,
                                 uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                                 uint32_t* out_cmps, uint32_t* out_hops);
int dab_search_batch_filtered_sq(dab_index* idx, const void* queries, uint32_t nq, uint32_t k,
                                 uint32_t l_search, uint32_t beam_width,
                                 const uint64_t* query_masks, uint32_t match_all,
                                 uint32_t adaptive_samples, double adaptive_scale, int rerank,
                                 uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                                 uint32_t* out_cmps, uint32_t* out_hops);
int dab_search_batch_filtered_minmax(dab_index* idx, const void* queries, uint32_t nq, uint32_t k,
                                     uint32_t l_search, uint32_t beam_width,
                                     const uint64_t* query_masks, uint32_t match_all,
                                     uint32_t adaptive_samples, double adaptive_scale, int rerank,
                                     uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                                     uint32_t* out_cmps, uint32_t* out_hops);
int dab_search_batch_filtered_pq_device(dab_index* idx, const void* d_queries, uint32_t nq,
                                        uint32_t k, uint32_t l_search, uint32_t beam_width,
                                        const uint64_t* d_query_masks, uint32_t match_all,
                                        uint32_t adaptive_samples, double adaptive_scale,
                                        int rerank, uint32_t* d_out_ids, float* d_out_dists,
                                        uint32_t* d_out_counts, uint32_t* d_out_cmps,
                                        uint32_t* d_out_hops);
int dab_search_batch_filtered_sq_device(dab_index* idx, const void* d_queries, uint32_t nq,
                                        uint32_t k, uint32_t l_search, uint32_t beam_width,
                                        const uint64_t* d_query_masks, uint32_t match_all,
                                        uint32_t adaptive_samples, double adaptive_scale,
                                        int rerank, uint32_t* d_out_ids, float* d_out_dists,
                                        uint32_t* d_out_counts, uint32_t* d_out_cmps,
                                        uint32_t* d_out_hops);
int dab_search_batch_filtered_minmax_device(dab_index* idx, const void* d_queries, uint32_t nq,
                                            uint32_t k, uint32_t l_search, uint32_t beam_width,
                                            const uint64_t* d_query_masks, uint32_t match_all,
                                            uint32_t adaptive_samples, double adaptive_scale,
                                            int rerank, uint32_t* d_out_ids, float* d_out_dists,
                                            uint32_t* d_out_counts, uint32_t* d_out_cmps,
                                            uint32_t* d_out_hops);

/* ------------------------------------------------------------------ (3'''') range search */

/* Range::search (diskann/src/graph/search/range_search.rs:255-469) for a whole query batch over
 * full-precision rows of every dtype and metric: every point within `radius` of each query.
 *   phase 1: the k-NN traversal of dab_search_batch with a list of l_search + n_start entries;
 *     in_range is its first l_search entries with distance <= radius, in list order.
 *   second round iff |in_range| >= (size_t)((float)l_search * initial_slack) and
 *     |in_range| < max_returned: the visited set is re-seeded with the in_range ids and the
 *     graph is walked breadth-first from them, beam_width ids at a time; each new neighbour with
 *     distance <= radius * range_slack (an f32 product) is appended while |in_range| < max_returned.
 *   results: in_range in insertion order (not sorted) without start points, deleted ids, ids
 *     with distance <= inner_radius (when has_inner_radius) and ids with distance > radius.
 * Deleted ids and start points are walked and count toward max_returned; they are never returned.
 * Per query: cmps are phase 1's comparisons; hops are phase 1's, or phase1 + (phase1 + phase2)
 * when the second round ran (the reference adds its cumulative hop count to phase 1's);
 * second_round says whether it ran.  max_returned == 0 means no limit (the reference rejects
 * every limit below l_search).  Queries [nq][dim] have the index dtype (f16 queries are widened).
 * Checked before any device work, each failing with DAB_ERR_INVALID_ARGUMENT and a message, in
 * the reference's order: beam_width == 0, l_search == 0, max_returned < l_search,
 * initial_slack outside [0, 1] (NaN included), range_slack < 1, inner_radius > radius; then
 * beam_width > 64 and a CTA's shared memory above 200 KB (4 x (the query row + 8 * max(max_degree,
 * 32) bytes)).  DAB_ERR_NOT_READY without vectors and graph.  A batch whose results cannot be held
 * in device memory fails with DAB_ERR_OUT_OF_MEMORY naming the entries it needs; nothing stays
 * allocated and the index stays usable.
 * On success *out is a result set resident on the device: a snapshot that later uploads, inserts
 * and deletes do not change.  dab_destroy releases every result set still open; their handles
 * are invalid after it. */
typedef struct dab_range dab_range; /* opaque: one batch's results, resident on the device */
int dab_range_search(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search,
                     uint32_t beam_width, float radius, int has_inner_radius, float inner_radius,
                     float initial_slack, float range_slack, uint64_t max_returned, dab_range** out);
/* the same with the queries in device memory */
int dab_range_search_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t l_search,
                            uint32_t beam_width, float radius, int has_inner_radius,
                            float inner_radius, float initial_slack, float range_slack,
                            uint64_t max_returned, dab_range** out);
/* Range::search over the PQ, SQ or MinMax store: the arguments and result set of dab_range_search,
 * plus `rerank`.  Every distance of both phases is the store's, those of
 * dab_search_batch_{pq,sq,minmax} on the same index: PQ TableL2 for L2 and CosineNormalized,
 * TableIP for InnerProduct, DirectCosine for Cosine; SQ compensated distances (Cosine refused);
 * MinMax every metric behind the store's transform (a query holding a NaN after the transform fails
 * the call, naming it).  SQ and MinMax compress the queries once, before the launch.
 *   rerank == 0: the results of dab_range_search with the store's distances (in insertion order,
 *     the radius and inner radius compared with the store's distances).
 *   rerank != 0: in_range (decided on the store's distances) without start points and deleted ids;
 *     each id's full-precision distance to the query; the ids with inner_radius < d <= radius of
 *     that distance, sorted by it (stable: ties in in_range order, -0.0 equal to +0.0).  The result
 *     set holds the full-precision distances.
 * cmps, hops and second_round are those of the traversal, with or without rerank.  Checked before
 * any device work: every check of dab_range_search (the shared-memory bound with the query area of
 * the store: the f32 query for PQ, the code row + 16 B for SQ and MinMax; the graph must be
 * uploaded), then the store's (its rows uploaded, SQ not under Cosine, l_search + n_start <= 1024)
 * and, with rerank, the full-precision vectors (DAB_ERR_NOT_READY), which are not needed without
 * it.  DAB_ERR_OUT_OF_MEMORY as dab_range_search, the rerank's sort included. */
int dab_range_search_pq(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search,
                        uint32_t beam_width, float radius, int has_inner_radius, float inner_radius,
                        float initial_slack, float range_slack, uint64_t max_returned, int rerank,
                        dab_range** out);
int dab_range_search_pq_device(dab_index* idx, const void* d_queries, uint32_t nq,
                               uint32_t l_search, uint32_t beam_width, float radius,
                               int has_inner_radius, float inner_radius, float initial_slack,
                               float range_slack, uint64_t max_returned, int rerank,
                               dab_range** out);
int dab_range_search_sq(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search,
                        uint32_t beam_width, float radius, int has_inner_radius, float inner_radius,
                        float initial_slack, float range_slack, uint64_t max_returned, int rerank,
                        dab_range** out);
int dab_range_search_sq_device(dab_index* idx, const void* d_queries, uint32_t nq,
                               uint32_t l_search, uint32_t beam_width, float radius,
                               int has_inner_radius, float inner_radius, float initial_slack,
                               float range_slack, uint64_t max_returned, int rerank,
                               dab_range** out);
int dab_range_search_minmax(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search,
                            uint32_t beam_width, float radius, int has_inner_radius,
                            float inner_radius, float initial_slack, float range_slack,
                            uint64_t max_returned, int rerank, dab_range** out);
int dab_range_search_minmax_device(dab_index* idx, const void* d_queries, uint32_t nq,
                                   uint32_t l_search, uint32_t beam_width, float radius,
                                   int has_inner_radius, float inner_radius, float initial_slack,
                                   float range_slack, uint64_t max_returned, int rerank,
                                   dab_range** out);
/* FilteredRange::search (diskann/src/graph/search/filtered_range_search.rs:119-248) over
 * full-precision rows of every dtype and metric: every point within `radius` of each query that
 * its mask accepts, with the arguments of dab_range_search plus the masks and mode of
 * dab_search_batch_filtered (ANY: labels & mask != 0; ALL: labels & mask == mask).
 *   phase 1: the filtered traversal of dab_search_batch_filtered (inline_filter_search_internal,
 *     without adaptive L) with a list of l_search + n_start entries.  matched: every accepted start
 *     point and evaluated neighbour with distance <= radius, sorted by distance (stable: among
 *     exactly equal distances the earlier match first, the order InlineFilterSearch fixes too;
 *     -0.0 equal to +0.0).  It is not cut to l_search.
 *   in_range: the list's first l_search entries and matched, those with distance <= radius,
 *     sorted by (distance, id) and each id once (:162-172).
 *   second round iff |in_range| >= (size_t)((float)l_search * initial_slack) and
 *     |matched| < max_returned (:182-185): the visited set is re-seeded with the in_range ids,
 *     which also form a FIFO frontier; while it is not empty and |matched| < max_returned, up to
 *     beam_width ids are popped and their unvisited neighbours evaluated, accepted or not
 *     (filtered_range_search_internal, :259-322).  Every neighbour with distance <= radius *
 *     range_slack (an f32 product) is pushed onto the frontier; an accepted one with distance
 *     <= radius is appended to matched while |matched| < max_returned.  The cap does not cut a hop
 *     short: the rest of the hop is still evaluated, pushed and counted.
 *   results: matched.take(max_returned) in order (phase 1's sorted matches, then the second
 *     round's in the order found; not sorted) without ids with distance <= inner_radius (when
 *     has_inner_radius), start points and deleted ids.  Start points and deleted ids are walked and
 *     count toward max_returned; they are never returned.
 * Per query: cmps and hops are both phases' totals when the second round ran (one scratch counts
 * both), else phase 1's; cmps do not count start points; second_round says whether it ran.
 * max_returned == 0 means no limit.  query_masks: one u64 per query (host memory, device memory for
 * the _device form).  Checked before any device work, each failing with DAB_ERR_INVALID_ARGUMENT
 * and a message: the checks of dab_range_search in its order up to beam_width > 64, then a label
 * table uploaded (dab_upload_labels), l_search + n_start <= 1024 and the shared memory of the
 * filtered kernel (that of dab_search_batch_filtered with a list of l_search + n_start).
 * DAB_ERR_NOT_READY without vectors and graph.  DAB_ERR_OUT_OF_MEMORY, the result set and
 * dab_destroy as dab_range_search. */
int dab_range_search_filtered(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search,
                              uint32_t beam_width, float radius, int has_inner_radius,
                              float inner_radius, float initial_slack, float range_slack,
                              uint64_t max_returned, const uint64_t* query_masks,
                              uint32_t match_all, dab_range** out);
int dab_range_search_filtered_device(dab_index* idx, const void* d_queries, uint32_t nq,
                                     uint32_t l_search, uint32_t beam_width, float radius,
                                     int has_inner_radius, float inner_radius,
                                     float initial_slack, float range_slack,
                                     uint64_t max_returned, const uint64_t* d_query_masks,
                                     uint32_t match_all, dab_range** out);
/* FilteredRange::search over the PQ, SQ or MinMax store (graph::ext::labeled::Filtered over the
 * quantized strategies): the arguments and result set of dab_range_search_filtered, plus `rerank`.
 * Both phases are those of dab_range_search_filtered, and every distance of both is the store's,
 * as in dab_range_search_{pq,sq,minmax} (SQ and MinMax compress the queries once, before the
 * launch; a MinMax query holding a NaN after the transform fails the call, naming it).
 *   rerank == 0: the results of dab_range_search_filtered with the store's distances.
 *   rerank != 0: matched.take(max_returned) without start points and deleted ids; each id's
 *     full-precision distance to the query; sorted by it (stable: ties in matched order, -0.0
 *     equal to +0.0, NaN after every number: the reference leaves the order of NaN open); the ids
 *     with d <= inner_radius of it (when has_inner_radius) dropped.  There is no outer-radius
 *     filter, unlike dab_range_search_pq: FilteredRange::search checks only the inner radius, so the
 *     results may hold ids whose full-precision distance is above radius, or NaN.  The result set
 *     holds the full-precision distances.
 * cmps, hops and second_round are those of the traversal, with or without rerank.  Checked before
 * any device work, in this order: every check of dab_range_search_filtered (the shared-memory
 * bound with the store's query area; the graph must be uploaded), then the store's (its rows
 * uploaded, SQ not under Cosine, l_search + n_start <= 1024) and, with rerank, the full-precision
 * vectors (DAB_ERR_NOT_READY) and the rerank's shared memory.  Without rerank only the graph, the
 * store and the label table are needed.  DAB_ERR_OUT_OF_MEMORY as dab_range_search, the rerank's
 * sort included. */
int dab_range_search_filtered_pq(dab_index* idx, const void* queries, uint32_t nq,
                                 uint32_t l_search, uint32_t beam_width, float radius,
                                 int has_inner_radius, float inner_radius, float initial_slack,
                                 float range_slack, uint64_t max_returned,
                                 const uint64_t* query_masks, uint32_t match_all, int rerank,
                                 dab_range** out);
int dab_range_search_filtered_pq_device(dab_index* idx, const void* d_queries, uint32_t nq,
                                        uint32_t l_search, uint32_t beam_width, float radius,
                                        int has_inner_radius, float inner_radius,
                                        float initial_slack, float range_slack,
                                        uint64_t max_returned, const uint64_t* d_query_masks,
                                        uint32_t match_all, int rerank, dab_range** out);
int dab_range_search_filtered_sq(dab_index* idx, const void* queries, uint32_t nq,
                                 uint32_t l_search, uint32_t beam_width, float radius,
                                 int has_inner_radius, float inner_radius, float initial_slack,
                                 float range_slack, uint64_t max_returned,
                                 const uint64_t* query_masks, uint32_t match_all, int rerank,
                                 dab_range** out);
int dab_range_search_filtered_sq_device(dab_index* idx, const void* d_queries, uint32_t nq,
                                        uint32_t l_search, uint32_t beam_width, float radius,
                                        int has_inner_radius, float inner_radius,
                                        float initial_slack, float range_slack,
                                        uint64_t max_returned, const uint64_t* d_query_masks,
                                        uint32_t match_all, int rerank, dab_range** out);
int dab_range_search_filtered_minmax(dab_index* idx, const void* queries, uint32_t nq,
                                     uint32_t l_search, uint32_t beam_width, float radius,
                                     int has_inner_radius, float inner_radius,
                                     float initial_slack, float range_slack,
                                     uint64_t max_returned, const uint64_t* query_masks,
                                     uint32_t match_all, int rerank, dab_range** out);
int dab_range_search_filtered_minmax_device(dab_index* idx, const void* d_queries, uint32_t nq,
                                            uint32_t l_search, uint32_t beam_width, float radius,
                                            int has_inner_radius, float inner_radius,
                                            float initial_slack, float range_slack,
                                            uint64_t max_returned,
                                            const uint64_t* d_query_masks, uint32_t match_all,
                                            int rerank, dab_range** out);
/* offsets [nq + 1]: query q's results are entries offsets[q] .. offsets[q + 1] - 1; cmps, hops
 * [nq] u32 and second_round [nq] (0 / 1) may be NULL.  Host buffers. */
int dab_range_offsets(const dab_range* r, uint64_t* offsets, uint32_t* cmps, uint32_t* hops,
                      uint8_t* second_round);
/* the offsets[nq] results: ids and distances, host buffers / device buffers */
int dab_range_results(const dab_range* r, uint32_t* ids, float* dists);
int dab_range_results_device(const dab_range* r, uint32_t* d_ids, float* d_dists);
void dab_range_free(dab_range* r);

/* ------------------------------------------------------------------ (3'') paged search */

/* DiskANNIndex::paged_search (diskann/src/graph/index.rs:2075-2155) and PagedSearch::next_page
 * (graph/search/paged.rs:53-149) for a whole query batch: successive, non-overlapping pages of one
 * resumable search per query, each query's candidate list and visited set kept on the device
 * between pages (only the pages cross PCIe).
 *   begin: queries [nq][dim] of the index dtype (f16 queries are widened as in dab_search_batch);
 *     l_search + n_start <= 1024.  The start points are expanded once; nothing is counted yet.
 *   next:  the next page of at most k results per query, 0 < k <= l_search: rows [nq][k] of ids and
 *     distances, padded with UINT32_MAX / +inf, ordered by non-decreasing distance within a page.
 *     out_counts[q] == 0 means query q is exhausted (and stays so).  out_cmps / out_hops are the
 *     session's cumulative comparisons and hops, counted as SearchStats counts them.  The counts,
 *     cmps and hops pointers may be NULL.  Host buffers only.
 *   end:   releases the session.
 * Several sessions may be open on one index.  Any upload of rows or adjacency, dab_build or a
 * broadcast after a session began makes its next page fail with DAB_ERR_INVALID_ARGUMENT.
 * dab_destroy releases every session still open; their handles are invalid after it. */
typedef struct dab_paged dab_paged; /* opaque */
int dab_paged_search_begin(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search,
                           dab_paged** out);
/* The same sessions over the quantized stores: traversal distances from the PQ table and codes (TableL2 / TableIP,
 * DirectCosine for Metric::Cosine), the scalar-quantized store or the MinMax store, as dab_search_batch_pq /
 * dab_search_batch_sq / dab_search_batch_minmax compute them (the PQ table of a query is rebuilt at every call; SQ and
 * MinMax queries are compressed once, at begin).  Pages return those quantized distances: the reference's paged search
 * applies no post-processing, so there is no rerank.  begin makes the store checks of the synchronous call (a store
 * never uploaded: "... has not been called"; rows not ready; Metric::Cosine on the SQ store) and fails on a MinMax
 * query holding a NaN after the transform, naming it; nothing stays allocated after a failed begin.  next and end are
 * the calls above.  Besides what invalidates every session, any later write to the session's own store (its upload,
 * encode-all, dab_pq_train or a broadcast) makes its next page fail with DAB_ERR_INVALID_ARGUMENT; writes to another
 * store do not, and no store write invalidates a full-precision session. */
int dab_paged_search_begin_pq(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search,
                              dab_paged** out);
int dab_paged_search_begin_sq(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search,
                              dab_paged** out);
int dab_paged_search_begin_minmax(dab_index* idx, const void* queries, uint32_t nq, uint32_t l_search,
                                  dab_paged** out);
int dab_paged_search_next(dab_paged* s, uint32_t k, uint32_t* out_ids, float* out_dists,
                          uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops);
void dab_paged_search_end(dab_paged* s);

/* Batches in flight.  The reference keeps every core busy by handing each query to a task of a
 * thread pool (diskann-benchmark-core/src/search/api.rs:410-419: `search_all` spawns one task per
 * query partition and joins them); the device equivalent is to keep more than one BATCH in flight:
 * `dab_search_batch_async` queues the copy of the queries, the search and the copy of the results
 * on a stream owned by `slot` (0 <= slot < DAB_MAX_SLOTS) and returns without waiting, `dab_wait`
 * joins the slot.  Batches on different slots overlap: the host<->device copies of one run under
 * the kernel of another, and the CTAs of the next batch fill the SMs that the draining tail of the
 * previous one leaves idle.  Results, statistics and error behaviour are those of dab_search_batch;
 * the host buffers (pinned memory makes the copies asynchronous) and the device buffers of the
 * `_device_` flavour must stay valid and untouched until `dab_wait(slot)` returns.  A slot holds
 * one batch at a time (DAB_ERR_INVALID_ARGUMENT otherwise); waiting on an idle slot is a no-op. */
#define DAB_MAX_SLOTS 4
int dab_search_batch_async(dab_index* idx, uint32_t slot, const void* queries, uint32_t nq, uint32_t k,
                           uint32_t l_search, uint32_t beam_width, uint32_t* out_ids, float* out_dists,
                           uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops);
int dab_search_batch_device_async(dab_index* idx, uint32_t slot, const void* d_queries, uint32_t nq, uint32_t k,
                                  uint32_t l_search, uint32_t beam_width, uint32_t* d_out_ids,
                                  float* d_out_dists, uint32_t* d_out_counts, uint32_t* d_out_cmps,
                                  uint32_t* d_out_hops);
int dab_wait(dab_index* idx, uint32_t slot);

/* The PQ, SQ and MinMax traversals (below) as batches in flight: each call takes the arguments
 * of its synchronous twin plus `slot`, queues the whole batch on the slot's stream (the copy of the queries, their
 * compression by the store's quantizer for SQ and MinMax, the traversal, the rerank when `rerank` is set, the copies of
 * the results) and returns without waiting; dab_wait(slot) joins a batch of any kind.
 *   Results: ids, distance bits, counts, cmps and hops are bit-identical to the synchronous call with the same
 *     arguments — dab_search_batch_pq (or dab_search_batch_pq_rerank when rerank is set), dab_search_batch_sq,
 *     dab_search_batch_minmax — including when queries outgrow their visited tables: dab_wait re-runs them, then runs
 *     the rerank over the whole batch again and repeats the copies of the host-buffer flavour.
 *   Launch-time errors: every error the synchronous call reports before it launches anything (a store that is not
 *     ready, Metric::Cosine on the SQ store, L + #start > 1024, NULL buffers, rerank without the full-precision rows)
 *     is reported by the launching call, and nothing is queued; so are a slot out of range and a slot that still holds
 *     a batch of any kind (full precision included).
 *   MinMax NaN query: the launching call does not wait for the query compression.  dab_wait returns
 *     DAB_ERR_INVALID_ARGUMENT with the synchronous call's message ("query %llu contains NaN after the transform");
 *     the outputs are then unspecified and the slot is idle.  (The synchronous call still fails before any traversal.)
 *   The launching calls never wait on the device; the only waits are dab_wait's.
 *   Buffers: as dab_search_batch_async — the host buffers (pinned memory makes the copies asynchronous) and the device
 *     buffers of the `_device_` flavour stay valid and untouched until dab_wait(slot) returns, and the graph and the
 *     stores must not change while a batch is in flight.  dab_upload_pq, dab_pq_train, dab_upload_sq,
 *     dab_upload_minmax and dab_broadcast_index wait for every slot before they free a store, and a batch launched on
 *     the replaced store never runs again: if some of its queries still need a re-run, dab_wait returns
 *     DAB_ERR_INVALID_ARGUMENT instead.  So a caller who breaks that rule gets unspecified results or that error,
 *     never a freed buffer under a running kernel. */
int dab_search_batch_pq_async(dab_index* idx, uint32_t slot, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                              uint32_t beam_width, int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                              uint32_t* out_cmps, uint32_t* out_hops);
int dab_search_batch_pq_device_async(dab_index* idx, uint32_t slot, const void* d_queries, uint32_t nq, uint32_t k,
                                     uint32_t l_search, uint32_t beam_width, int rerank, uint32_t* d_out_ids,
                                     float* d_out_dists, uint32_t* d_out_counts, uint32_t* d_out_cmps, uint32_t* d_out_hops);
int dab_search_batch_sq_async(dab_index* idx, uint32_t slot, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                              uint32_t beam_width, int rerank, uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                              uint32_t* out_cmps, uint32_t* out_hops);
int dab_search_batch_sq_device_async(dab_index* idx, uint32_t slot, const void* d_queries, uint32_t nq, uint32_t k,
                                     uint32_t l_search, uint32_t beam_width, int rerank, uint32_t* d_out_ids,
                                     float* d_out_dists, uint32_t* d_out_counts, uint32_t* d_out_cmps, uint32_t* d_out_hops);
int dab_search_batch_minmax_async(dab_index* idx, uint32_t slot, const void* queries, uint32_t nq, uint32_t k,
                                  uint32_t l_search, uint32_t beam_width, int rerank, uint32_t* out_ids, float* out_dists,
                                  uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops);
int dab_search_batch_minmax_device_async(dab_index* idx, uint32_t slot, const void* d_queries, uint32_t nq, uint32_t k,
                                         uint32_t l_search, uint32_t beam_width, int rerank, uint32_t* d_out_ids,
                                         float* d_out_dists, uint32_t* d_out_counts, uint32_t* d_out_cmps,
                                         uint32_t* d_out_hops);

/* ------------------------------------------------------------------ product quantization */

/* FixedChunkPQTable::populate_chunk_distances / populate_chunk_inner_products
 * (fixed_chunk_pq_table.rs:152-218): lut[q][chunk][center]; metric L2 or InnerProduct. */
int dab_pq_populate_lut(dab_index* idx, const float* queries, uint32_t nq, int metric, float* out_lut);

/* QueryComputer::evaluate_similarity over gathered codes
 * (pq/distance/dynamic.rs:63-103; pq_dist_lookup_single, fixed_chunk_pq_table.rs:82-98;
 * compute_pq_distance :617-670): out[q][j] for ids[q][j].  Queries are f32. */
int dab_pq_distances(dab_index* idx, const float* queries, uint32_t nq, const uint32_t* ids,
                     uint32_t c, float* out);

/* DistanceComputer::evaluate_similarity(code, code) (pq/distance/dynamic.rs:101-140; the PQ prune path):
 * FixedChunkPQTable::{qq_l2_distance, qq_inner_product, qq_cosine_distance}
 * (fixed_chunk_pq_table.rs:285-361) between the stored codes of rows a[i] and b[i] under the index
 * metric (CosineNormalized -> cosine, VTable dynamic.rs:126-131).  Resumable accumulation across chunks. */
int dab_pq_self_distances(dab_index* idx, const uint32_t* ids_a, const uint32_t* ids_b, uint64_t n, float* out);

/* The providers' PQ traversal: QuantAccessor::expand_beam with
 * `computer.evaluate_similarity(aux_vectors[i])`
 * (diskann-providers/src/model/graph/provider/async_/inmem/product.rs:311-340) inside
 * search_internal — dab_search_batch with every traversal distance an ADC lookup over the
 * uploaded codes (start points included).  Queries have the index dtype and are converted to
 * f32 (T: Into<f32>); L2 / CosineNormalized use TableL2, InnerProduct TableIP; Metric::Cosine
 * runs QueryComputer::DirectCosine (pq/distance/cosine.rs:16-70: no table, the resumable cosine
 * over the pivot chunks a code selects).  No rerank: distances returned are the traversal values. */
int dab_search_batch_pq(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                        uint32_t beam_width, uint32_t* out_ids, float* out_dists,
                        uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops);

/* The same followed by the quantized providers' default post-processing
 * Pipeline<FilterStartPoints, Rerank> (inmem/product.rs:391-400; full_precision.rs:356-399): every
 * entry of the candidate list that is not a start point is re-scored with the full-precision
 * Distance<T, T> over the uploaded rows, the list is ordered by that distance (ties keep their
 * traversal order; the reference leaves them unspecified) and the first k are returned — what
 * `use_fp_for_search: false` runs in diskann-benchmark (src/index/inmem/product.rs:233-239).
 * Every row type and metric of the index: f32 / f16 / i8 / u8 (f16 x f16 and Metric::Cosine over float rows use the
 * schemas with two accumulators, simd.rs:424-483). */
int dab_search_batch_pq_rerank(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                               uint32_t beam_width, uint32_t* out_ids, float* out_dists,
                               uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops);
/* device-pointer variant of both (rerank = 0 / 1); results stay in HBM */
int dab_search_batch_pq_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                               uint32_t beam_width, int rerank, uint32_t* d_out_ids, float* d_out_dists,
                               uint32_t* d_out_counts, uint32_t* d_out_cmps, uint32_t* d_out_hops);

/* BasicTable::compress_into (diskann-quantization/src/product/tables/basic.rs:161-194) for n
 * host vectors (f32): codes [n][n_chunks].  Returns DAB_ERR_INVALID_ARGUMENT if a chunk's
 * minimum distance is infinite/NaN (first offending row/chunk in the message). */
int dab_pq_encode(dab_index* idx, const float* vectors, uint64_t n, uint8_t* out_codes);

/* ------------------------------------------------------------------ scalar quantization */

/* ScalarQuantizer::compress_into (diskann-quantization/src/scalar/quantizer.rs:190-239,
 * 407-430): codes one per byte in [0, 2^nbits), compensation per vector. */
int dab_sq_compress(int device, const float* shift, float scale, uint32_t dim, int nbits,
                    const float* vectors, uint64_t n, uint8_t* out_codes, float* out_comp);

/* CompensatedSquaredL2 / CompensatedIP / CompensatedCosineNormalized
 * (scalar/vectors.rs:206-237, 310-376, 380-460) for n code pairs. */
int dab_sq_distances(int device, int metric, int nbits, float scale_squared, float shift_square_norm,
                     uint32_t dim, const uint8_t* x, const float* comp_x, const uint8_t* y,
                     const float* comp_y, uint64_t n, float* out);

/* The scalar-quantized store of an index (diskann-providers/src/model/graph/provider/async_/inmem/
 * scalar.rs:60-258, SQStore<NBITS>): the quantizer (ScalarQuantizer: shift[dim], scale, and the two
 * derived fields quantizer.shift_square_norm() and quantizer.mean_norm(), 0 when None) and one row
 * per point (data + start points) in the reference's canonical-front layout (diskann-quantization/
 * src/meta/vector.rs:478-507): 4 bytes f32 compensation, then ceil(dim * nbits / 8) bytes of
 * Dense-packed codes (bits/slice.rs:261-323) — what set_quant_vector (:193-212) stores.  rows may
 * be NULL when dab_sq_encode_all follows.  Bits past dim * nbits in a row's last code byte are
 * ignored, as the reference's BitSlice never reads them.  nbits in {1, 2, 4, 8}. */
int dab_upload_sq(dab_index* idx, int nbits, const float* shift, float scale, float shift_square_norm,
                  float mean_norm, const uint8_t* rows);
/* SQStore::set_vector (scalar.rs:150-175) for every resident row (any dtype, as_f32 first). */
int dab_sq_encode_all(dab_index* idx);
/* rows back in the canonical-front layout, (n_points + n_start) x (4 + ceil(dim * nbits / 8)): byte
 * for byte what the store holds, the padding bits of the last code byte cleared */
int dab_sq_download(dab_index* idx, uint8_t* rows);

/* KNN::search through the scalar-quantized accessor (scalar.rs:449-570): the query is compressed
 * with the store's quantizer (query_computer, :227-253; rescaled to mean_norm for InnerProduct) and
 * every traversal distance is Compensated{SquaredL2, IP, CosineNormalized} over the packed codes
 * (scalar/vectors.rs:206-460; integer cores bits/distances.rs:397, 979).  rerank = 0: the
 * quant-only strategy (RemoveDeletedIdsAndCopy: first k of the candidate list with their quantized
 * distances, scalar.rs:640-670); rerank = 1: Pipeline<FilterStartPoints, Rerank> with the
 * full-precision rows (:596-610).  Metric::Cosine is rejected like SQStore::distance_computer
 * (:214-226).  Outputs as dab_search_batch. */
int dab_search_batch_sq(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                        uint32_t beam_width, int rerank, uint32_t* out_ids, float* out_dists,
                        uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops);
int dab_search_batch_sq_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                               uint32_t beam_width, int rerank, uint32_t* d_out_ids, float* d_out_dists,
                               uint32_t* d_out_counts, uint32_t* d_out_cmps, uint32_t* d_out_hops);

/* ------------------------------------------------------------------ MinMax quantization */

/* The per-vector N-bit quantizer of diskann-quantization/src/minmax (NBITS = 1, 2, 4, 8; Transform::Null).  Rows use the
 * reference's canonical-front layout of minmax::Data<NBITS> (meta/vector.rs:377-392): MinMaxCompensation
 * {dim: u32, b, n, a, norm_squared} (vectors.rs:43-52, 20 bytes) followed by ceil(dim * NBITS / 8) bytes of dense codes,
 * value i at bit i * NBITS — so rows written here can be handed to DataRef::from_canonical_front and back. */
uint32_t dab_minmax_row_bytes(uint32_t dim, int nbits);  /* Data::<NBITS>::canonical_bytes(dim); 0 for an unsupported width */

/* MinMaxQuantizer::new(Transform::Null(dim), grid_scale) + CompressInto<&[f32], DataMutRef<NBITS>> for n vectors
 * (quantizer.rs:153-228, get_range :117-151): out_rows [n][dab_minmax_row_bytes], out_loss [n] (L2Loss, may be NULL).
 * An input vector containing NaN makes the call fail (InputContainsNaN, naming the first such vector) after every row
 * has been written, the way the reference sets the meta before returning the error. */
int dab_minmax_compress(int device, float grid_scale, uint32_t dim, int nbits, const float* vectors, uint64_t n,
                        uint8_t* out_rows, float* out_loss);

/* PureDistanceFunction<DataRef<NBITS>, DataRef<MBITS>, distances::Result<f32>> for MinMaxL2Squared / MinMaxIP (negated) /
 * MinMaxCosine / MinMaxCosineNormalized (vectors.rs:206-455), selected by `metric` (Metric repr): out[i] = d(x_rows[i],
 * y_rows[i]).  Widths: N x N, and 8 x N (the pairings the reference instantiates).  Rows whose stored dimension differs
 * from `dim` give NaN (UnequalLengths). */
int dab_minmax_distances(int device, int metric, int nbits_x, int nbits_y, uint32_t dim, const uint8_t* x_rows,
                         const uint8_t* y_rows, uint64_t n, float* out);

/* The query side of the minmax-exhaustive-search benchmark (diskann-benchmark/src/exhaustive/minmax.rs): queries stay
 * full precision — CompressInto<&[f32], FullQueryMut> (quantizer.rs:369-417: FullQueryMeta {sum, norm_squared}) — and
 * PureDistanceFunction<FullQueryRef, DataRef<NBITS>, distances::Result<f32>> for the four MinMax distances
 * (vectors.rs:272-305, 347-392, 417-476) is evaluated for every (query, row) pair: out [nq][n].  The f32 x N-bit inner
 * product follows the reference's x86-64-v3 kernels lane for lane (bits/distances.rs:2295-2725).  A query containing NaN
 * fails the call (InputContainsNaN). */
int dab_minmax_query_distances(int device, int metric, int nbits, uint32_t dim, const float* queries, uint32_t nq,
                               const uint8_t* rows, uint64_t n, float* out);

/* ------------------------------------------------------------------ Hadamard transforms in front of MinMax */

/* The Hadamard transforms of diskann-quantization/src/algorithms/transforms, the counterpart of Transform::PaddingHadamard
 * and Transform::DoubleHadamard (RandomRotation is not offered: its transform_into is a faer sgemm whose summation
 * order is not restated).  A dab_transform is a host-side object; only the calls that take a device touch one. */
typedef struct dab_transform dab_transform; /* opaque */
enum {
    DAB_TRANSFORM_PADDING_HADAMARD = 1, /* padding_hadamard.rs */
    DAB_TRANSFORM_DOUBLE_HADAMARD = 2   /* double_hadamard.rs */
};

/* PaddingHadamard::try_from_parts (padding_hadamard.rs:137-173) / DoubleHadamard::try_from_parts (double_hadamard.rs:
 * 146-206) from the parts the reference serializes.  Signs are 0 / 1 bytes (the flatbuffer's bool form): signs0 has
 * input_dim of them; signs1 (DoubleHadamard only, NULL otherwise) has inner_dim.  inner_dim is padded_dim for
 * PaddingHadamard and len(signs1) for DoubleHadamard.  subsample == NULL: none; otherwise n_subsample sorted indices
 * into the inner vector.  The output dimension is n_subsample, or inner_dim without a subsample.  Every error of
 * try_from_parts fails with its own message, in the reference's order; inner_dim > 32768 (one vector has to fit a
 * warp's shared memory) fails with DAB_ERR_INVALID_ARGUMENT.  No device is touched. */
int dab_transform_create(dab_transform** out, int kind, uint32_t input_dim, uint32_t inner_dim, const uint8_t* signs0,
                         const uint8_t* signs1, const uint32_t* subsample, uint32_t n_subsample);
void dab_transform_destroy(dab_transform* t);
uint32_t dab_transform_input_dim(const dab_transform* t);   /* 0 for NULL */
uint32_t dab_transform_output_dim(const dab_transform* t);  /* 0 for NULL */

/* transform_into (padding_hadamard.rs:227-273, double_hadamard.rs:238-287) for n rows: src [n][input_dim] ->
 * dst [n][output_dim], bit-identical to hadamard_transform's x86-64-v3 order (hadamard.rs:194-371). */
int dab_transform_apply(const dab_transform* t, int device, const float* src, uint64_t n, float* dst);

/* MinMaxQuantizer::new(transform, grid_scale) + CompressInto<&[f32], DataMutRef<NBITS>> (quantizer.rs:153-228) for n
 * rows of input_dim values: the rows are transformed, then compressed like dab_minmax_compress with dim = output_dim.
 * out_rows [n][dab_minmax_row_bytes(output_dim, nbits)], out_loss [n] (may be NULL).  The NaN check runs on the
 * transformed vectors, as in the reference: the call fails naming the first row whose transformed vector holds a NaN
 * (an input with two infinities of opposite sign does), after every row has been written. */
int dab_minmax_compress_transformed(const dab_transform* t, int device, float grid_scale, int nbits, const float* vectors,
                                    uint64_t n, uint8_t* out_rows, float* out_loss);

/* dab_minmax_query_distances behind a transform: CompressInto<&[f32], FullQueryMut> (quantizer.rs:393-415) checks the
 * *untransformed* query for NaN, transforms it and takes FullQueryMeta of the transformed vector; then the four MinMax
 * distances against rows compressed at output_dim.  queries [nq][input_dim], out [nq][n]. */
int dab_minmax_query_distances_transformed(const dab_transform* t, int device, int metric, int nbits, const float* queries,
                                           uint32_t nq, const uint8_t* rows, uint64_t n, float* out);

/* ------------------------------------------------------------------ MinMax store of an index */

/* MinMaxElement<NBITS> as the VectorRepr of an index (diskann-providers/src/common/minmax_repr.rs:167-336), the traversal
 * store diskann-garnet runs (quantization.rs:229-362, MinMax8Bit; provider.rs:1170-1358): MinMaxQuantizer::new(t, or
 * Transform::Null(dim) when t is NULL, grid_scale) and one row per point (data + start points).  rows are
 * (n_points + n_start) x dab_minmax_row_bytes(out_dim, nbits) in the canonical-front Data<NBITS> layout, out_dim =
 * t ? output_dim(t) : dim; NULL when dab_minmax_encode_all follows.  Bits past dim * nbits in a row's last code byte are
 * ignored, as the reference's BitSlice never reads them.  Fails naming the entry point for nbits not in {1, 2, 4, 8},
 * grid_scale <= 0, input_dim(t) != dim, and a row whose stored dim is not out_dim (the first such row).  The store keeps
 * its own copy of t: the caller may destroy t after the call. */
int dab_upload_minmax(dab_index* idx, int nbits, float grid_scale, const dab_transform* t, const uint8_t* rows);
/* For every resident row: T::as_f32, the transform, CompressInto<&[f32], DataMutRef<NBITS>> (quantizer.rs:153-228) — what
 * garnet's backfill stores.  A transformed row holding a NaN fails the call, naming the first such row; the store then
 * has no rows until the next successful upload or encode. */
int dab_minmax_encode_all(dab_index* idx);
/* the rows back in the canonical-front layout, byte for byte what the store holds, the padding bits of the last code
 * byte cleared */
int dab_minmax_download(dab_index* idx, uint8_t* rows);

/* KNN::search through the MinMax store (garnet DynamicAccessor, provider.rs:1170-1358: as_f32, then
 * quantizer.query_computer): queries have the index dtype and go through as_f32, the store's transform and its
 * compressor at the store's NBITS and grid scale (the query is &[MinMaxElement<N>]); every traversal distance, start
 * points included, is MinMax{Cosine, IP, L2Squared, CosineNormalized} of the index metric between the compressed query
 * and the row (vectors.rs:206-455; all four metrics).  rerank = 0: the first k non-start entries of the candidate list
 * with their MinMax distances; rerank = 1: Pipeline<FilterStartPoints, Rerank> over the full-precision rows (garnet
 * Rerank, provider.rs:1457-1530), as dab_search_batch_sq.  A query whose transformed vector holds a NaN fails the call,
 * naming the first such query.  L + #start <= 1024.  Outputs as dab_search_batch. */
int dab_search_batch_minmax(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t l_search,
                            uint32_t beam_width, int rerank, uint32_t* out_ids, float* out_dists,
                            uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops);
int dab_search_batch_minmax_device(dab_index* idx, const void* d_queries, uint32_t nq, uint32_t k, uint32_t l_search,
                                   uint32_t beam_width, int rerank, uint32_t* d_out_ids, float* d_out_dists,
                                   uint32_t* d_out_counts, uint32_t* d_out_cmps, uint32_t* d_out_hops);

/* ------------------------------------------------------------------ build-side reuse */

/* PruneAccessor::fill + robust_prune (diskann/src/graph/index.rs:2349-2380, 2565-2650;
 * graph/internal/prune.rs:106-259; PruneKind graph/config/mod.rs:80-103) for n_pools
 * independent candidate pools: pool p has pool_lens[p] (id, source distance) entries in
 * pool_ids/pool_dists[p * pool_cap ...] (any order; sorted by distance then arrival order and
 * truncated to max_occlusion_size = 750 like SortedNeighbors::new), locations[p] is the node
 * being pruned (excluded from its own pool).  Candidate x candidate distances are
 * Distance<T,T> over the uploaded rows.  out_ids [n_pools][degree] (padded UINT32_MAX).
 * pool_cap must be in [1, 2048] (a whole pool is held in shared memory) and degree > 0;
 * otherwise DAB_ERR_INVALID_ARGUMENT and nothing is written. */
int dab_robust_prune(dab_index* idx, const uint32_t* pool_ids, const float* pool_dists,
                     const uint32_t* pool_lens, const uint32_t* locations, uint32_t n_pools,
                     uint32_t pool_cap, uint32_t degree, float alpha, uint32_t* out_ids,
                     uint32_t* out_counts);

/* Batched Vamana construction on the device (the rows SURVEY.md §8f.2 marks "next"):
 * DiskANNIndex::multi_insert semantics (diskann/src/graph/index.rs:815) — batches of inserts
 * searched with the same search kernel, pruned with robust_prune
 * (graph/internal/prune.rs:106-259) and back-edges merged per destination (aggregate_backedges :123, one
 * add_edge_and_prune per target: extend with every source, prune once).  intra_batch_candidates = None; the
 * bootstrap routine (index.rs:589-747, run by the reference while a batch's back-edges reach <= 8 x batch distinct
 * targets) is NOT run: batch_size = 1 is DiskANNIndex::insert point by point, larger batches grow as inserted / 8 up
 * to batch_size (0: a default from the index size) so that no point is inserted blind.  Uses the uploaded vectors
 * (including start rows) and overwrites the adjacency.  A target's back-edges are not limited in number.  An insert
 * search keeps a record of min(2048, 4 * l_build + 64) expanded nodes; when a search expands more, its prune pool is
 * cut, the build still completes with a valid graph, and the call returns DAB_ERR_INVALID_ARGUMENT saying "their prune
 * pools were cut" (the graph is then usable but not the reference's). */
int dab_build(dab_index* idx, uint32_t pruned_degree, uint32_t l_build, float alpha,
              uint32_t batch_size);

/* Inserts points into the index as it stands: DiskANNIndex::insert (diskann/src/graph/index.rs:226-341) and multi_insert
 * (:815-1030).  rows holds [n][dim] values of the index dtype, dense, on the host (as dab_upload_vectors); ids[i] takes
 * rows[i].
 *   set_element: every row is written into the index and into each quantized store that holds rows (the PQ codes when
 *     codes were uploaded or encoded, the SQ and MinMax stores when they hold rows), the aux stores before the base
 *     store as the inmem providers do (diskann-providers/.../async_/inmem/provider.rs:695-725).  The codes are
 *     byte-identical to what dab_pq_encode_all, dab_sq_encode_all and dab_minmax_encode_all write for those rows; a store
 *     without rows stays without rows.  The encoders' checks (a PQ row infinitely far from every centre, a MinMax row
 *     with a NaN after the transform) run before anything is written and fail naming the caller's row index, leaving the
 *     rows, every store and the adjacency as they were.
 *   linking: the ids are cut into consecutive chunks of batch_size in the caller's order (0: 65536, the cap of
 *     dab_build's default batch size), and each chunk is one multi_insert on the graph the previous chunk left, with
 *     dab_build's semantics: every member searched against the graph as it was before the chunk (beam 1, l_build, a
 *     visited record, the deletion table ignored), pruned to pruned_degree and its out-list written, then one
 *     add_edge_and_prune per back-edge target with its sources sorted; max_backedges = pruned_degree,
 *     intra_batch_candidates = None, no bootstrap.  batch_size = 1 is DiskANNIndex::insert point by point.  A graph that
 *     was never uploaded or built starts empty, so an index can be grown from its start points by inserts alone.
 * Any id in [0, n_points) that is not deleted may be inserted: a row no list reaches, a released slot, or a live point,
 * whose vector and out-list are then replaced.  DAB_ERR_INVALID_ARGUMENT, changing nothing and naming the first
 * offending id: an id >= n_points (start points are frozen), a repeated id, a deleted id (dab_release it first); also
 * NULL pointers with n > 0, pruned_degree outside [1, max_degree], l_build == 0, alpha < 1, or any slot holding a batch
 * in flight.  DAB_ERR_NOT_READY when no vectors were uploaded.  n == 0 returns DAB_OK after these checks.  Visited
 * records cut are reported as dab_build reports them (the graph is then usable but not the reference's).  Open paged sessions fail their next page; the tensor-core scan rebuilds its operand on its next use;
 * dab_flat_knn* still scan every row. */
int dab_insert(dab_index* idx, const uint32_t* ids, const void* rows, uint64_t n, uint32_t pruned_degree, uint32_t l_build,
               float alpha, uint32_t batch_size);

/* ------------------------------------------------------------------ deletion */

/* Delete::delete / release / status_by_internal_id of the providers' TableDeleteProviderAsync
 * (diskann-providers/src/model/graph/provider/async_/table_delete_provider.rs; inmem/provider.rs:596-655): one bit per id.
 *   dab_delete: marks ids deleted; deleting an id twice is a no-op.  An id >= n_points (a start point, which is frozen,
 *     or an id out of range) fails the call with DAB_ERR_INVALID_ARGUMENT naming the first such id, and nothing changes.
 *   dab_release: clears the mark and empties the node's adjacency row.  An id that is not deleted fails the call,
 *     naming the first such id, and nothing changes (the reference would silently clear a live node's list).
 *   dab_delete_status: out_deleted[i] = 1 when ids[i] is deleted, else 0; ids must be < n_points + n_start.
 * Every k-NN search (dab_search_batch*, dab_search_batch_pq*, _sq*, _minmax*; host, _device and _async) then applies
 * the reference's post-processing over the same traversal: without rerank the first k entries of the final candidate
 * list that are neither start points nor deleted (Pipeline<FilterStartPoints, RemoveDeletedIdsAndCopy>, async_/
 * postprocess.rs:35-61); with rerank deleted entries are dropped before they are scored.  out_counts is the number of
 * live results, which can be below k (the rest is padded UINT32_MAX / +inf); cmps and hops are the traversal's, which
 * still expands deleted nodes.  While nothing is deleted a search launches exactly what it launches without a table.
 * Paged search applies no post-processing (paged.rs:122), so its pages keep deleted ids; the exhaustive scans
 * (dab_flat_knn*) stay ground truth over every row, and dab_build ignores the table, as the reference's insert does.
 * The table travels with dab_broadcast_index and dab_broadcast.  dab_delete, dab_release and dab_consolidate fail with
 * DAB_ERR_INVALID_ARGUMENT, changing nothing, while any slot holds a batch in flight (join it with dab_wait first).
 * dab_release, and dab_consolidate when it rewrites a list, make open paged sessions fail their next page; dab_delete
 * does not. */
int dab_delete(dab_index* idx, const uint32_t* ids, uint64_t n);
int dab_release(dab_index* idx, const uint32_t* ids, uint64_t n);
int dab_delete_status(dab_index* idx, const uint32_t* ids, uint64_t n, uint8_t* out_deleted);
/* DiskANNIndex::consolidate_vector (diskann/src/graph/index.rs:1819-1931) for every id in [0, n_points + n_start), in
 * one device pass, which equals the reference's sequential loop in any order: a deleted node is left alone; a node with
 * no deleted neighbour (an id >= n_points + n_start counts as one, with no neighbours) and at most pruned_degree
 * distinct live neighbours is left alone; otherwise its pool is the set of its live neighbours and of the live
 * neighbours of its deleted ones, itself removed, and becomes the new list as it is when it has fewer than
 * pruned_degree ids, else goes through robust_prune_list (index.rs:2397-2454: Distance<T,T> from the node, sorted, cut to
 * 750, occlude_list without saturation; the prune kind from the metric, as dab_robust_prune).  Where the reference's
 * HashSet leaves an order unspecified the pool's order is fixed: the node's live neighbours in list order, then each
 * deleted neighbour's live neighbours, deleted neighbours in list order, first occurrence kept; exact distance ties
 * keep that order.  List lengths above max_degree are read as max_degree.  With nothing deleted it still prunes the
 * lists longer than pruned_degree.  Needs the vectors and the graph; pruned_degree in [1, max_degree]; alpha >= 1.
 * out_rewritten (may be NULL): the number of lists written. */
int dab_consolidate(dab_index* idx, uint32_t pruned_degree, float alpha, uint64_t* out_rewritten);

/* The three ways DiskANNIndex::inplace_delete finds the lists to repair (diskann/src/graph/misc.rs:28) */
enum { DAB_INPLACE_VISITED_AND_TOPK = 0, DAB_INPLACE_TWO_HOP_AND_ONE_HOP = 1, DAB_INPLACE_ONE_HOP = 2 };

/* DiskANNIndex::multi_inplace_delete (diskann/src/graph/index.rs:1338-1520): deletes ids and repairs only the lists
 * around each of them, so the cost follows n, not the size of the index.  The ids are cut into consecutive chunks of
 * batch_size (max_minibatch_par) in the caller's order, members kept in that order; batch_size = 1 is inplace_delete
 * called id by id (the reference's default), 0 is one chunk of all n.  Each chunk, on the graph the previous one left:
 *   1. work lists (inplace_delete_inner, index.rs:1585-1749).  Every member of the chunk is marked deleted before any
 *      list is read: of the schedules the reference's parallel tasks allow (each marks its member, then reads the graph),
 *      the device takes this one, which is also the only one in which step 2 never adds an edge to a chunk-mate.  Then,
 *      per member m, with live meaning neither deleted nor an id >= n_points + n_start:
 *        OneHop: replace candidates = m's live neighbours in list order; in-neighbours = those of them whose list holds m.
 *        TwoHopAndOneHop: the same replace candidates; in-neighbours = the live ids of {m's live neighbours and their
 *          neighbours} whose list holds m.
 *        VisitedAndTopK{k_value, l_value}: search_internal with m's own row as the query (beam 1, L = l_value, the
 *          deletion table ignored during the traversal); deleted ids are dropped from the whole best list, start points
 *          kept (RemoveDeletedIdsAndCopy), and the first l_value taken; in-neighbours = those whose list holds m,
 *          replace candidates = the first k_value (k_value may exceed l_value).
 *      With Distance<T,T>, each in-neighbour c gets edges[c] = the num_to_replace replace candidates nearest to c,
 *      c excluded (a later entry for the same c replaces an earlier one, and an empty one still counts); then each
 *      live neighbour a of m is appended to edges[r] for each of the num_to_replace replace candidates r nearest to a,
 *      a excluded.  Exact distance ties, and the cut at num_to_replace, are ordered by position in the replace
 *      candidates (the reference's sort_unstable_by leaves them unspecified).
 *   2. apply: every source with an entry in any member's edges gets one add_edge_and_prune (index.rs:2264-2341): the
 *      chunk's ids are removed from its list, then the members' edges[source], concatenated in chunk order, are
 *      appended, skipping ids already present; a list with nothing added and nothing removed stays as it is, a list
 *      that fits max_degree is written, and a longer one goes through robust_prune_list (index.rs:2397-2454) at
 *      pruned_degree and alpha, without saturation (the prune kind from the metric, as dab_consolidate).  An id
 *      >= n_points + n_start kept in such a list is left out of the prune pool: it has no row, so robust_prune_list's
 *      fill finds nothing for it (the ids of a list that fits are kept as they are).
 *   3. drop: every member's list is emptied.
 * An id >= n_points + n_start met in a list counts as deleted with no neighbours, as in dab_consolidate (the
 * reference's status or neighbour lookup would fail there); list lengths above max_degree are read as max_degree.
 * Any data id may be given, one that is already deleted included (the reference's delete is idempotent, and repairing
 * a soft-deleted point in place is legitimate).  Afterwards the ids are in the deletion table (as after dab_delete),
 * the rows and every quantized store are untouched, dab_release -> dab_insert reuses the ids, and open paged sessions
 * fail their next page.  num_to_replace = 0 is valid: the edges to the ids are still removed.
 * DAB_ERR_INVALID_ARGUMENT, changing nothing and naming the first offending id: an id >= n_points (start points are
 * frozen), a repeated id; also NULL ids with n > 0, an unknown method, pruned_degree outside [1, max_degree], alpha < 1,
 * for VisitedAndTopK l_value == 0 or l_value + n_start > 1024, a max_degree (or VisitedAndTopK's min(k_value,
 * l_value)) too large for the kernels' shared memory, or any slot holding a batch in flight.  DAB_ERR_NOT_READY when
 * the vectors and graph are missing.  n == 0 returns DAB_OK after these checks.  A failure after them (out of memory,
 * a chunk with 2^31 or more edges, a CUDA error) leaves the chunks before the failing one applied and the failing
 * chunk's ids marked deleted but not repaired: searches leave them out, and dab_consolidate repairs the graph. */
int dab_inplace_delete(dab_index* idx, const uint32_t* ids, uint64_t n, int method, uint32_t num_to_replace, uint32_t k_value,
                       uint32_t l_value, uint32_t pruned_degree, float alpha, uint32_t batch_size);
/* DiskANNIndex::drop_deleted_neighbors (index.rs:1756-1816) for every id in [0, n_points + n_start), in one device pass,
 * which equals the sequential loop in any order since a deleted node's list is never written: a deleted node is left
 * alone; otherwise the pool is its live neighbours in list order, not deduplicated, followed with only_orphans by its
 * deleted neighbours whose own list is not empty, in list order (an id >= n_points + n_start counts as deleted with no
 * neighbours); the pool becomes the list unless the node had no deleted neighbour and the pool holds at most
 * pruned_degree ids.  pruned_degree in [1, max_degree]; refused while any slot holds a batch in flight; open paged
 * sessions fail their next page when a list was written.  out_rewritten (may be NULL): the number of lists written. */
int dab_drop_deleted_neighbors(dab_index* idx, uint32_t pruned_degree, int only_orphans, uint64_t* out_rewritten);

/* Graph checks and the final prune.
 *
 * DiskANNIndex::count_reachable_nodes (diskann/src/graph/index.rs:2161-2189), the reference's health check after a
 * build, a delete or an insert: *out_count = the number of distinct ids its breadth-first walk expands from the n
 * start_ids, the start ids included, each counted once, whatever their order or repeats.  start_ids NULL (n must be 0)
 * walks from the index's start points [n_points, n_points + n_start), what provider().starting_points() returns
 * (diskann-providers/src/model/graph/provider/async_/inmem/provider.rs:326-328); an explicit list of n = 0 reaches
 * nothing.  Deleted ids are walked like any other (get_neighbors does not read the deletion table); list lengths above
 * max_degree are read as max_degree, as the searches read them.  An id >= n_points + n_start in the list of an
 * expanded node makes the reference's get_neighbors fail (SimpleNeighborProviderAsync::get_neighbors_sync has no list
 * for it): the call then returns DAB_ERR_INVALID_ARGUMENT naming the smallest such id the walk reached; one in a list the
 * walk never expands is ignored.  DAB_ERR_INVALID_ARGUMENT, before anything runs, for a start id >= n_points + n_start
 * or NULL start_ids with n > 0; DAB_ERR_NOT_READY without a graph.  Read-only (no paged session is disturbed), so it
 * is allowed while batches are in flight; it runs on the handle's stream and returns with the count.  Its scratch (the
 * visited bitmap and one queue of n_points + n_start ids) is allocated and freed per call, and freeing device memory
 * waits for the whole device: a call made while batches are in flight returns after they have finished. */
int dab_count_reachable(dab_index* idx, const uint32_t* start_ids, uint32_t n, uint64_t* out_count);
/* DiskANNIndex::get_degree_stats (index.rs:2191-2240; DegreeStats, index.rs:69-74) over the list lengths of the n ids,
 * each occurrence counted (a repeated id counts once per occurrence, as the reference's loop).  ids NULL (n must be 0)
 * is provider().iter(): every id in [0, n_points + n_start), start points and deleted ids included (inmem/provider.rs:
 * 330-333); an explicit list of n = 0 gives all zeros, the reference's guard.  out_avg = (float)total / (float)count
 * with total summed exactly and each conversion rounded to nearest, like Rust's `as f32`: bit-exact.  out_less_than_two
 * counts the lists shorter than 2.  List lengths above max_degree are read as max_degree.  DAB_ERR_INVALID_ARGUMENT for
 * an id >= n_points + n_start, NULL ids with n > 0 or a NULL output; DAB_ERR_NOT_READY without a graph.  Read-only,
 * allowed while batches are in flight, on the handle's stream; like dab_count_reachable it frees per-call scratch, so
 * it returns after the batches in flight have finished. */
int dab_degree_stats(dab_index* idx, const uint32_t* ids, uint64_t n, uint32_t* out_max, float* out_avg, uint32_t* out_min,
                     uint64_t* out_less_than_two);
/* DiskANNIndex::prune_range (index.rs:2656-2700), "the final step of graph construction", over the n ids (ids NULL with
 * n = 0: every id in [0, n_points + n_start)): a list of at most pruned_degree entries is left alone; any other becomes
 * robust_prune_list(id, list) (index.rs:2397-2454): the pool is the list's distinct ids (first occurrence kept) without
 * id itself and without the ids >= n_points + n_start, which have no row (view.get finds nothing), however short that
 * leaves it; Distance<T,T> from id's row, sorted by (distance, position), cut to 750, then occlude_list at pruned_degree
 * and alpha without saturation, the prune kind from the metric — the prune dab_consolidate runs.  The full-precision
 * PruneAccessor::fill (inmem/full_precision.rs:145-150) finds a row for every id and reads no deletion table, so a
 * deleted id's list is pruned like any other and deleted neighbours stay in the pools.  Each prune reads only its own
 * list and rows, so all ids run at once and equal the reference's loop; a repeated id equals one occurrence (the
 * second prune is a no-op).  *out_rewritten (may be NULL): the lists written.  The rows and every quantized store are
 * untouched; when a list was written open paged sessions fail their next page.  DAB_ERR_INVALID_ARGUMENT, changing
 * nothing: an id >= n_points + n_start (naming the first), NULL ids with n > 0, pruned_degree outside [1, max_degree],
 * alpha < 1, or any slot holding a batch in flight; DAB_ERR_NOT_READY without the vectors and graph. */
int dab_prune_range(dab_index* idx, const uint32_t* ids, uint64_t n, uint32_t pruned_degree, float alpha, uint64_t* out_rewritten);

/* exact k-NN by exhaustive scan (diskann/src/flat; ground truth for recall):
 * out_ids [nq][k] ascending distance, ties by lower id. */
int dab_flat_knn(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t* out_ids,
                 float* out_dists);

/* The same scan on the tensor cores (a wgmma GEMM with TMA-staged vector tiles and fused
 * ||x||^2 + ||y||^2 expansion): bf16 operands (f32 / f16 rows as a 3-product hi/lo split, i8 / u8 exact),
 * fp32 accumulation in registers,
 * fused score expansion and per-row candidate selection in the epilogue; the candidates are then
 * re-scored with the exact reference-order kernel.  Each query is then certified against a rigorous bound
 * on the approximate scores' error; the queries that cannot be (ill-conditioned data, NaN / inf rows,
 * n < k) are re-run through the exact scan.  So out_ids and out_dists always equal dab_flat_knn's.
 * k <= 24. */
int dab_flat_knn_tc(dab_index* idx, const void* queries, uint32_t nq, uint32_t k, uint32_t* out_ids,
                    float* out_dists);

#ifdef __cplusplus
}
#endif
#endif
