"""Host-side mirror of the reference interface for the distance hot path, over the C ABI.

Names follow the reference: `Metric` (diskann-vector/src/distance/metric.rs:8-20),
`distance_comparer` (distance_provider.rs:44-46), the provider-level snapshot
(`diskann_inmem::Provider`, diskann-inmem/src/provider.rs:71-131) and the batched
`KNN::search` (diskann-benchmark-core/src/search/graph/knn.rs:208-238).  All compute happens
in libdiskann_b200.so on the GPU; numpy is only the host container.
"""
import ctypes as C
import enum
import weakref

import numpy as np

from . import _lib
from ._lib import DabError, check

__all__ = ["Metric", "DType", "GpuIndex", "PagedSearch", "distance_comparer", "pair_distances", "DabError", "launch_count"]


class Metric(enum.IntEnum):
    """#[repr(C)] values of diskann_vector::distance::Metric."""
    Cosine = 0
    InnerProduct = 1
    L2 = 2
    CosineNormalized = 3


class DType(enum.IntEnum):
    f32 = 0
    f16 = 1
    i8 = 2
    u8 = 3


_NP = {DType.f32: np.float32, DType.f16: np.float16, DType.i8: np.int8, DType.u8: np.uint8}


def dtype_of(arr):
    try:
        return {np.dtype(np.float32): DType.f32, np.dtype(np.float16): DType.f16,
                np.dtype(np.int8): DType.i8, np.dtype(np.uint8): DType.u8}[arr.dtype]
    except KeyError:
        raise DabError(1, f"unsupported element type {arr.dtype}") from None


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def launch_count():
    return int(_lib.lib().dab_launch_count())


def pair_distances(x, y, metric, device=0):
    """n independent distances x[i] . y[i] (Distance<T, U>::call for each pair)."""
    x = np.ascontiguousarray(x)
    y = np.ascontiguousarray(y)
    if x.ndim != 2 or y.ndim != 2 or x.shape != y.shape:
        raise DabError(1, f"expected two [n, dim] arrays of equal shape, got {x.shape} and {y.shape}")
    out = np.empty(x.shape[0], np.float32)
    check(_lib.lib().dab_pair_distances(int(dtype_of(x)), int(dtype_of(y)), int(metric), x.shape[1], _ptr(x), _ptr(y),
                                        x.shape[0], _ptr(out), device))
    return out


def distance_comparer(metric, dim=None, device=0):
    """T::distance_comparer(metric, Some(dim)) -> callable(x, y) -> f32.

    Length mismatches raise (the providers' DistanceFunction panics, implementations.rs:105-130;
    the inmem layer returns Err, layers/full.rs:203-213)."""

    def call(x, y):
        x = np.ascontiguousarray(x)
        y = np.ascontiguousarray(y)
        if x.ndim != 1 or x.shape != y.shape or (dim is not None and x.shape[0] != dim):
            raise DabError(1, f"expected slices of length {dim} - instead got {x.shape} and {y.shape}")
        return pair_distances(x[None, :], y[None, :], metric, device)[0]

    return call


def _splitmix64(seed):
    state = seed & 0xFFFFFFFFFFFFFFFF
    while True:
        state = (state + 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF
        z = state
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & 0xFFFFFFFFFFFFFFFF
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & 0xFFFFFFFFFFFFFFFF
        yield z ^ (z >> 31)


class Transform:
    """A Hadamard transform in front of the MinMax quantizer: Transform::PaddingHadamard / Transform::DoubleHadamard of
    diskann-quantization/src/algorithms/transforms, held by the library as a host-side object (dab_transform).

    Build one from the reference's serialized parts (signs as bools, the inner dimension, optional sorted subsample
    indices) with the constructor, or draw a new one with `padding_hadamard` / `double_hadamard`, which apply the
    reference's TargetDim rules exactly.  The random draws there come from SplitMix64(seed), not Rust's StdRng: a
    transform drawn here has the reference's shape but not the signs a reference run with the same seed would draw."""

    PADDING_HADAMARD = 1
    DOUBLE_HADAMARD = 2

    def __init__(self, kind, signs0, inner_dim, signs1=None, subsample=None):
        self._h = C.c_void_p()
        signs0 = np.ascontiguousarray(signs0, np.uint8)
        signs1 = None if signs1 is None else np.ascontiguousarray(signs1, np.uint8)
        subsample = None if subsample is None else np.ascontiguousarray(subsample, np.uint32)
        n_sub = 0 if subsample is None else len(subsample)
        if subsample is not None and n_sub == 0:
            subsample = np.zeros(1, np.uint32)  # present but empty: a non-NULL pointer with no entries
        check(_lib.lib().dab_transform_create(C.byref(self._h), int(kind), len(signs0), int(inner_dim), _ptr(signs0), _ptr(signs1),
                                              _ptr(subsample), n_sub))
        self.kind = int(kind)
        self.signs0, self.signs1, self.inner_dim = signs0, signs1, int(inner_dim)
        self.subsample = None if subsample is None else subsample[:n_sub]

    @staticmethod
    def _target(target):
        """TargetDim: "same", "natural" or an int (Override)."""
        if target in ("same", "natural"):
            return target
        if int(target) < 1:
            raise DabError(1, f"target dim must be positive, got {target}")
        return int(target)

    @staticmethod
    def _subsample(rng, length, amount):
        """`amount` distinct sorted indices of range(length) (subsample_indices, transforms/utils.rs:60-78), by a partial
        Fisher-Yates shuffle."""
        idx = np.arange(length, dtype=np.uint32)
        for i in range(amount):
            j = i + next(rng) % (length - i)
            idx[i], idx[j] = idx[j], idx[i]
        return np.sort(idx[:amount])

    @classmethod
    def padding_hadamard(cls, dim, target="same", seed=0):
        """PaddingHadamard::new (padding_hadamard.rs:94-133): Same -> (padded, output) = (next_pow2(dim), dim), Natural ->
        (next_pow2(dim), next_pow2(dim)), Override(t) -> (next_pow2(max(t, dim)), t); subsampled when padded > output."""
        target = cls._target(target)
        pow2 = lambda v: 1 << (int(v) - 1).bit_length()  # noqa: E731
        if target == "same":
            padded, out = pow2(dim), dim
        elif target == "natural":
            padded = out = pow2(dim)
        else:
            padded, out = pow2(max(target, dim)), target
        rng = _splitmix64(seed)
        signs = np.array([next(rng) >> 63 for _ in range(dim)], np.uint8)
        sub = cls._subsample(rng, padded, out) if padded > out else None
        return cls(cls.PADDING_HADAMARD, signs, padded, subsample=sub)

    @classmethod
    def double_hadamard(cls, dim, target="same", seed=0):
        """DoubleHadamard::new (double_hadamard.rs:98-144): output = dim for Same and Natural, t for Override(t);
        intermediate = max(dim, output) (len(signs1)); subsampled when dim > output."""
        target = cls._target(target)
        out = dim if target in ("same", "natural") else target
        inter = max(dim, out)
        rng = _splitmix64(seed)
        signs0 = np.array([next(rng) >> 63 for _ in range(dim)], np.uint8)
        signs1 = np.array([next(rng) >> 63 for _ in range(inter)], np.uint8)
        sub = cls._subsample(rng, dim, out) if dim > out else None
        return cls(cls.DOUBLE_HADAMARD, signs0, inter, signs1=signs1, subsample=sub)

    @property
    def input_dim(self):
        return int(_lib.lib().dab_transform_input_dim(self._h))

    @property
    def output_dim(self):
        return int(_lib.lib().dab_transform_output_dim(self._h))

    @property
    def preserves_norms(self):
        return self.subsample is None

    def apply(self, vectors, device=0):
        """transform_into for the rows of `vectors` [n, input_dim] f32 -> [n, output_dim] f32 (on the device)."""
        vectors = np.ascontiguousarray(vectors, np.float32)
        if vectors.ndim != 2 or vectors.shape[1] != self.input_dim:
            raise DabError(1, f"Transform.apply: vectors must be [n, {self.input_dim}] f32, got {vectors.shape}")
        out = np.empty((vectors.shape[0], self.output_dim), np.float32)
        check(_lib.lib().dab_transform_apply(self._h, device, _ptr(vectors), vectors.shape[0], _ptr(out)))
        return out

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            _lib.lib().dab_transform_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        self.close()


def minmax_compress(vectors, nbits, grid_scale=1.0, device=0, transform=None):
    """MinMaxQuantizer over the rows of `vectors` [n, dim] f32: (rows u8 [n, 20 + ceil(out_dim * nbits / 8)] in the
    reference's canonical-front Data<NBITS> layout, loss f32 [n]).  transform=None is Transform::Null (out_dim = dim);
    a `Transform` runs first (out_dim = its output_dim).  Raises DabError when a (transformed) vector contains NaN."""
    vectors = np.ascontiguousarray(vectors, np.float32)
    if vectors.ndim != 2:
        raise DabError(1, "minmax_compress: vectors must be [n, dim] f32")
    n, dim = vectors.shape
    if transform is not None and dim != transform.input_dim:
        raise DabError(1, f"minmax_compress: vectors have {dim} values, the transform takes {transform.input_dim}")
    out_dim = dim if transform is None else transform.output_dim
    rb = _lib.lib().dab_minmax_row_bytes(out_dim, nbits)
    rows = np.zeros((n, rb), np.uint8)
    loss = np.zeros(n, np.float32)
    if transform is None:
        check(_lib.lib().dab_minmax_compress(device, grid_scale, dim, nbits, _ptr(vectors), n, _ptr(rows), _ptr(loss)))
    else:
        check(_lib.lib().dab_minmax_compress_transformed(transform._h, device, grid_scale, nbits, _ptr(vectors), n, _ptr(rows), _ptr(loss)))
    return rows, loss


def minmax_distances(metric, nbits_x, nbits_y, dim, x_rows, y_rows, device=0):
    """MinMax{L2Squared, IP, Cosine, CosineNormalized} between compressed rows: out[i] = d(x_rows[i], y_rows[i])."""
    x_rows = np.ascontiguousarray(x_rows, np.uint8)
    y_rows = np.ascontiguousarray(y_rows, np.uint8)
    n = x_rows.shape[0]
    out = np.empty(n, np.float32)
    check(_lib.lib().dab_minmax_distances(device, int(metric), nbits_x, nbits_y, dim, _ptr(x_rows), _ptr(y_rows), n, _ptr(out)))
    return out


def minmax_query_distances(metric, nbits, queries, rows, device=0, transform=None):
    """Full-precision queries [nq, dim] f32 against MinMax-compressed rows [n, row_bytes]: out [nq, n]
    (MinMax{L2Squared, IP, Cosine, CosineNormalized}::evaluate(FullQueryRef, DataRef<NBITS>)).  With a `Transform` the
    queries are checked for NaN, then transformed, and the rows must have been compressed behind the same transform."""
    queries = np.ascontiguousarray(queries, np.float32)
    rows = np.ascontiguousarray(rows, np.uint8)
    nq, dim = queries.shape
    out = np.empty((nq, rows.shape[0]), np.float32)
    if transform is None:
        check(_lib.lib().dab_minmax_query_distances(device, int(metric), nbits, dim, _ptr(queries), nq, _ptr(rows), rows.shape[0], _ptr(out)))
    else:
        if dim != transform.input_dim:
            raise DabError(1, f"minmax_query_distances: queries have {dim} values, the transform takes {transform.input_dim}")
        check(_lib.lib().dab_minmax_query_distances_transformed(transform._h, device, int(metric), nbits, _ptr(queries), nq, _ptr(rows),
                                                                 rows.shape[0], _ptr(out)))
    return out


class GpuIndex:
    """Device-resident snapshot of an in-memory index: vectors + adjacency (+ PQ)."""

    def __init__(self, dtype, metric, dim, n_points, n_start=1, max_degree=83, device=0):
        self._h = C.c_void_p()
        self._inflight = {}  # slot -> (queries, outputs) kept alive while a batch is in flight
        self._paged = weakref.WeakSet()  # open paged searches: dab_destroy releases them
        self._ranges = weakref.WeakSet()  # open range search result sets: dab_destroy releases them too
        self.dtype, self.metric, self.dim = DType(dtype), Metric(metric), int(dim)
        self.n_points, self.n_start, self.max_degree, self.device = int(n_points), int(n_start), int(max_degree), device
        check(_lib.lib().dab_create(C.byref(self._h), int(dtype), int(metric), dim, n_points, n_start, max_degree, device))

    # -- lifecycle
    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            for s in list(getattr(self, "_paged", ())) + list(getattr(self, "_ranges", ())):
                s._h = C.c_void_p()  # released by dab_destroy
            _lib.lib().dab_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    @property
    def n_total(self):
        return self.n_points + self.n_start

    def set_stream(self, cuda_stream_ptr):
        check(_lib.lib().dab_set_stream(self._h, C.c_void_p(cuda_stream_ptr)))

    # -- replication (one process per GPU): NCCL inside the library
    @staticmethod
    def comm_unique_id():
        buf = C.create_string_buffer(128)
        check(_lib.lib().dab_comm_unique_id(buf))
        return buf.raw

    def comm_init(self, unique_id, n_ranks, rank):
        check(_lib.lib().dab_comm_init(self._h, C.c_char_p(unique_id), n_ranks, rank))

    def broadcast_index(self, root=0):
        """One NCCL broadcast per resident buffer (vectors, adjacency, PQ) from `root` to every rank."""
        check(_lib.lib().dab_broadcast_index(self._h, root))

    # -- uploads
    def _rows(self, rows):
        rows = np.ascontiguousarray(rows)
        if rows.ndim != 2 or rows.shape[1] != self.dim or dtype_of(rows) != self.dtype:
            raise DabError(1, f"expected [n, {self.dim}] rows of {self.dtype.name}, got {rows.shape} {rows.dtype}")
        return rows

    def upload_vectors(self, rows, first=0):
        rows = self._rows(rows)
        check(_lib.lib().dab_upload_vectors(self._h, _ptr(rows), first, rows.shape[0]))

    def upload_vectors_device(self, dev_ptr, count, first=0):
        check(_lib.lib().dab_upload_vectors_device(self._h, C.c_void_p(dev_ptr), first, count))

    def upload_graph(self, adj, first=0):
        adj = np.ascontiguousarray(adj, dtype=np.uint32)
        if adj.ndim != 2:
            raise DabError(1, "adjacency must be [n, stride] u32 with row[0] = degree")
        check(_lib.lib().dab_upload_graph(self._h, _ptr(adj), adj.shape[1], first, adj.shape[0]))

    def upload_graph_device(self, dev_ptr, src_stride, count, first=0):
        check(_lib.lib().dab_upload_graph_device(self._h, C.c_void_p(dev_ptr), src_stride, first, count))

    def download_graph(self, first=0, count=None):
        count = self.n_total - first if count is None else count
        adj = np.zeros((count, self.max_degree + 1), np.uint32)
        check(_lib.lib().dab_download_graph(self._h, _ptr(adj), adj.shape[1], first, count))
        return adj

    def upload_pq(self, pivots, offsets, codes=None):
        pivots = np.ascontiguousarray(pivots, np.float32)
        offsets = np.ascontiguousarray(offsets, np.uint64)
        if pivots.ndim != 2 or pivots.shape[1] != self.dim:
            raise DabError(1, f"pivots must be [n_centers, {self.dim}] f32")
        if codes is not None:
            codes = np.ascontiguousarray(codes, np.uint8)
            if codes.shape != (self.n_total, len(offsets) - 1):
                raise DabError(1, f"codes must be [{self.n_total}, {len(offsets) - 1}] u8, got {codes.shape}")
        self.pq_chunks, self.pq_centers = len(offsets) - 1, pivots.shape[0]
        check(_lib.lib().dab_upload_pq(self._h, _ptr(pivots), pivots.shape[0], _ptr(offsets), len(offsets) - 1, _ptr(codes)))

    def pq_train(self, train, n_chunks, n_centers=256, lloyds_reps=5, seed=0):
        """train_pq on the device: k-means++ + Lloyd per chunk over host training rows [n, dim] f32."""
        train = np.ascontiguousarray(train, np.float32)
        if train.ndim != 2 or train.shape[1] != self.dim:
            raise DabError(1, f"training rows must be [n, {self.dim}] f32")
        check(_lib.lib().dab_pq_train(self._h, _ptr(train), train.shape[0], n_chunks, n_centers, lloyds_reps, seed))
        self.pq_chunks, self.pq_centers = n_chunks, n_centers

    def pq_encode_all(self):
        check(_lib.lib().dab_pq_encode_all(self._h))

    def download_pq(self, codes=True):
        """(pivots [n_centers, dim] f32, offsets u64 [n_chunks + 1], codes u8 [n_total, n_chunks] or None)."""
        pivots = np.empty((self.pq_centers, self.dim), np.float32)
        offsets = np.empty(self.pq_chunks + 1, np.uint64)
        c = np.empty((self.n_total, self.pq_chunks), np.uint8) if codes else None
        check(_lib.lib().dab_pq_download(self._h, _ptr(pivots), _ptr(offsets), _ptr(c)))
        return pivots, offsets, c

    # -- distances
    def _queries(self, queries):
        queries = np.ascontiguousarray(queries)
        if queries.ndim != 2 or queries.shape[1] != self.dim or dtype_of(queries) != self.dtype:
            raise DabError(1, f"expected [nq, {self.dim}] queries of {self.dtype.name}, got {queries.shape} {queries.dtype}")
        return queries

    def distances(self, queries, ids):
        """out[q][j] = QueryDistance(queries[q]).evaluate(row ids[q][j]) (expand_beam's distance stage)."""
        queries = self._queries(queries)
        ids = np.ascontiguousarray(ids, np.uint32)
        if ids.ndim != 2 or ids.shape[0] != queries.shape[0]:
            raise DabError(1, "ids must be [nq, c] u32")
        out = np.empty(ids.shape, np.float32)
        check(_lib.lib().dab_distances(self._h, _ptr(queries), queries.shape[0], _ptr(ids), ids.shape[1], _ptr(out)))
        return out

    def row_pair_distances(self, a, b):
        a = np.ascontiguousarray(a, np.uint32)
        b = np.ascontiguousarray(b, np.uint32)
        if a.shape != b.shape or a.ndim != 1:
            raise DabError(1, "a and b must be 1-d u32 arrays of equal length")
        out = np.empty(a.shape[0], np.float32)
        check(_lib.lib().dab_row_pair_distances(self._h, _ptr(a), _ptr(b), a.shape[0], _ptr(out)))
        return out

    def pairwise(self, ids):
        ids = np.ascontiguousarray(ids, np.uint32)
        out = np.empty((ids.shape[0], ids.shape[0]), np.float32)
        check(_lib.lib().dab_pairwise(self._h, _ptr(ids), ids.shape[0], _ptr(out)))
        return out

    # -- search
    def search_batch(self, queries, k, l_search, beam_width=1):
        """KNN::search for the whole batch: (ids [nq,k], dists [nq,k], counts, cmps, hops)."""
        queries = self._queries(queries)
        nq = queries.shape[0]
        ids = np.empty((nq, k), np.uint32)
        dists = np.empty((nq, k), np.float32)
        counts = np.empty(nq, np.uint32)
        cmps = np.empty(nq, np.uint32)
        hops = np.empty(nq, np.uint32)
        check(_lib.lib().dab_search_batch(self._h, _ptr(queries), nq, k, l_search, beam_width, _ptr(ids), _ptr(dists),
                                          _ptr(counts), _ptr(cmps), _ptr(hops)))
        return ids, dists, counts, cmps, hops

    def paged_search(self, queries, l_search):
        """DiskANNIndex::paged_search for the whole batch: a PagedSearch whose next_page(k) returns the next page of
        every query (each query's list and visited set stay on the device between pages)."""
        return PagedSearch(self, self._queries(queries), l_search)

    def paged_search_pq(self, queries, l_search):
        """paged_search with the PQ traversal distances of search_batch_pq (TableL2 / TableIP, DirectCosine for
        Metric::Cosine); pages return those distances (paged search has no rerank)."""
        return PagedSearch(self, self._queries(queries), l_search, _lib.lib().dab_paged_search_begin_pq)

    def paged_search_sq(self, queries, l_search):
        """paged_search through the scalar-quantized store, as search_batch_sq traverses it; no rerank."""
        return PagedSearch(self, self._queries(queries), l_search, _lib.lib().dab_paged_search_begin_sq)

    def paged_search_minmax(self, queries, l_search):
        """paged_search through the MinMax store, as search_batch_minmax traverses it; no rerank.  A query holding a NaN
        after the store's transform fails the call."""
        return PagedSearch(self, self._queries(queries), l_search, _lib.lib().dab_paged_search_begin_minmax)

    def range_search(self, queries, l_search, radius, *, beam_width=1, inner_radius=None, initial_slack=1.0, range_slack=1.0,
                     max_returned=None):
        """Range::search for the whole batch: every point within `radius` of each query, in the reference's order.
        Returns (offsets [nq + 1] u64, ids, dists, cmps, hops, second_round): query q's results are
        ids[offsets[q]:offsets[q + 1]].  max_returned=None: no limit."""
        with self.range_search_set(queries, l_search, radius, beam_width=beam_width, inner_radius=inner_radius,
                                   initial_slack=initial_slack, range_slack=range_slack, max_returned=max_returned) as r:
            offsets, cmps, hops, second = r.offsets()
            ids, dists = r.results()
        return offsets, ids, dists, cmps, hops, second

    def range_search_set(self, queries, l_search, radius, **kw):
        """range_search, keeping the result set on the device: a RangeResults"""
        return RangeResults(self, _lib.lib().dab_range_search, _ptr(self._queries(queries)), len(queries), l_search, radius, **kw)

    def range_search_device(self, d_queries, nq, l_search, radius, *, beam_width=1, inner_radius=None, initial_slack=1.0,
                            range_slack=1.0, max_returned=None):
        """range_search of `nq` queries at the device pointer `d_queries` (an integer): a RangeResults, whose
        results_device copies the results to device buffers"""
        return RangeResults(self, _lib.lib().dab_range_search_device, C.c_void_p(d_queries), nq, l_search, radius, beam_width=beam_width,
                            inner_radius=inner_radius, initial_slack=initial_slack, range_slack=range_slack, max_returned=max_returned)

    def _range_quant(self, store, queries, l_search, radius, rerank=False, **kw):
        with RangeResults(self, getattr(_lib.lib(), f"dab_range_search_{store}"), _ptr(self._queries(queries)), len(queries), l_search, radius,
                          rerank=bool(rerank), **kw) as r:
            offsets, cmps, hops, second = r.offsets()
            ids, dists = r.results()
        return offsets, ids, dists, cmps, hops, second

    def range_search_pq(self, queries, l_search, radius, *, beam_width=1, inner_radius=None, initial_slack=1.0, range_slack=1.0,
                        max_returned=None, rerank=False):
        """range_search with every distance of both phases the PQ store's (those of search_batch_pq).  rerank=True: the
        in_range ids by full-precision distance, those within (inner_radius, radius] of it, sorted by it, with it."""
        return self._range_quant("pq", queries, l_search, radius, beam_width=beam_width, inner_radius=inner_radius, initial_slack=initial_slack,
                                 range_slack=range_slack, max_returned=max_returned, rerank=rerank)

    def range_search_sq(self, queries, l_search, radius, *, beam_width=1, inner_radius=None, initial_slack=1.0, range_slack=1.0,
                        max_returned=None, rerank=False):
        """range_search_pq over the scalar-quantized store (the distances of search_batch_sq)"""
        return self._range_quant("sq", queries, l_search, radius, beam_width=beam_width, inner_radius=inner_radius, initial_slack=initial_slack,
                                 range_slack=range_slack, max_returned=max_returned, rerank=rerank)

    def range_search_minmax(self, queries, l_search, radius, *, beam_width=1, inner_radius=None, initial_slack=1.0, range_slack=1.0,
                            max_returned=None, rerank=False):
        """range_search_pq over the MinMax store (the distances of search_batch_minmax).  A query holding a NaN after the
        store's transform fails the call."""
        return self._range_quant("minmax", queries, l_search, radius, beam_width=beam_width, inner_radius=inner_radius,
                                 initial_slack=initial_slack, range_slack=range_slack, max_returned=max_returned, rerank=rerank)

    def _range_quant_device(self, store, d_queries, nq, l_search, radius, rerank=False, **kw):
        return RangeResults(self, getattr(_lib.lib(), f"dab_range_search_{store}_device"), C.c_void_p(d_queries), nq, l_search, radius,
                            rerank=bool(rerank), **kw)

    def range_search_pq_device(self, d_queries, nq, l_search, radius, *, beam_width=1, inner_radius=None, initial_slack=1.0, range_slack=1.0,
                               max_returned=None, rerank=False):
        """range_search_pq of `nq` queries at the device pointer `d_queries` (an integer): a RangeResults"""
        return self._range_quant_device("pq", d_queries, nq, l_search, radius, beam_width=beam_width, inner_radius=inner_radius,
                                        initial_slack=initial_slack, range_slack=range_slack, max_returned=max_returned, rerank=rerank)

    def range_search_sq_device(self, d_queries, nq, l_search, radius, *, beam_width=1, inner_radius=None, initial_slack=1.0, range_slack=1.0,
                               max_returned=None, rerank=False):
        """range_search_sq of `nq` queries at the device pointer `d_queries` (an integer): a RangeResults"""
        return self._range_quant_device("sq", d_queries, nq, l_search, radius, beam_width=beam_width, inner_radius=inner_radius,
                                        initial_slack=initial_slack, range_slack=range_slack, max_returned=max_returned, rerank=rerank)

    def range_search_minmax_device(self, d_queries, nq, l_search, radius, *, beam_width=1, inner_radius=None, initial_slack=1.0,
                                   range_slack=1.0, max_returned=None, rerank=False):
        """range_search_minmax of `nq` queries at the device pointer `d_queries` (an integer): a RangeResults"""
        return self._range_quant_device("minmax", d_queries, nq, l_search, radius, beam_width=beam_width, inner_radius=inner_radius,
                                        initial_slack=initial_slack, range_slack=range_slack, max_returned=max_returned, rerank=rerank)

    def range_search_filtered(self, queries, masks, l_search, radius, *, match_all=False, beam_width=1, inner_radius=None,
                              initial_slack=1.0, range_slack=1.0, max_returned=None):
        """FilteredRange::search for the whole batch over the label table (upload_labels): every point within `radius` of
        each query that its mask accepts (as search_batch_filtered accepts it; `masks` u64 per query, or one for all).
        Returns range_search's (offsets, ids, dists, cmps, hops, second_round); results are in the reference's order
        (phase 1's matches by distance, then the second round's in the order found).  max_returned=None: no limit."""
        with self.range_search_filtered_set(queries, masks, l_search, radius, match_all=match_all, beam_width=beam_width,
                                            inner_radius=inner_radius, initial_slack=initial_slack, range_slack=range_slack,
                                            max_returned=max_returned) as r:
            offsets, cmps, hops, second = r.offsets()
            ids, dists = r.results()
        return offsets, ids, dists, cmps, hops, second

    def range_search_filtered_set(self, queries, masks, l_search, radius, *, match_all=False, **kw):
        """range_search_filtered, keeping the result set on the device: a RangeResults"""
        queries = self._queries(queries)
        masks = np.ascontiguousarray(np.broadcast_to(np.asarray(masks, np.uint64), (queries.shape[0],)))
        return RangeResults(self, _lib.lib().dab_range_search_filtered, _ptr(queries), len(queries), l_search, radius, masks=_ptr(masks),
                            match_all=match_all, **kw)

    def range_search_filtered_device(self, d_queries, d_masks, nq, l_search, radius, *, match_all=False, beam_width=1, inner_radius=None,
                                     initial_slack=1.0, range_slack=1.0, max_returned=None):
        """range_search_filtered of `nq` queries and masks at the device pointers `d_queries` and `d_masks` (integers): a
        RangeResults"""
        return RangeResults(self, _lib.lib().dab_range_search_filtered_device, C.c_void_p(d_queries), nq, l_search, radius,
                            beam_width=beam_width, inner_radius=inner_radius, initial_slack=initial_slack, range_slack=range_slack,
                            max_returned=max_returned, masks=C.c_void_p(d_masks), match_all=match_all)

    def _range_filtered_quant(self, store, queries, masks, l_search, radius, match_all=False, rerank=False, **kw):
        queries = self._queries(queries)
        masks = np.ascontiguousarray(np.broadcast_to(np.asarray(masks, np.uint64), (queries.shape[0],)))
        with RangeResults(self, getattr(_lib.lib(), f"dab_range_search_filtered_{store}"), _ptr(queries), len(queries), l_search, radius,
                          masks=_ptr(masks), match_all=match_all, rerank=bool(rerank), **kw) as r:
            offsets, cmps, hops, second = r.offsets()
            ids, dists = r.results()
        return offsets, ids, dists, cmps, hops, second

    def range_search_filtered_pq(self, queries, masks, l_search, radius, *, match_all=False, beam_width=1, inner_radius=None,
                                 initial_slack=1.0, range_slack=1.0, max_returned=None, rerank=False):
        """range_search_filtered with every distance of both phases the PQ store's (those of search_batch_pq).
        rerank=True: the returned matches (start points and deleted ids dropped) by full-precision distance, sorted by it
        (NaN last), those above inner_radius, with it; no outer-radius filter, as in FilteredRange::search."""
        return self._range_filtered_quant("pq", queries, masks, l_search, radius, match_all=match_all, beam_width=beam_width,
                                          inner_radius=inner_radius, initial_slack=initial_slack, range_slack=range_slack,
                                          max_returned=max_returned, rerank=rerank)

    def range_search_filtered_sq(self, queries, masks, l_search, radius, *, match_all=False, beam_width=1, inner_radius=None,
                                 initial_slack=1.0, range_slack=1.0, max_returned=None, rerank=False):
        """range_search_filtered_pq over the scalar-quantized store (the distances of search_batch_sq)"""
        return self._range_filtered_quant("sq", queries, masks, l_search, radius, match_all=match_all, beam_width=beam_width,
                                          inner_radius=inner_radius, initial_slack=initial_slack, range_slack=range_slack,
                                          max_returned=max_returned, rerank=rerank)

    def range_search_filtered_minmax(self, queries, masks, l_search, radius, *, match_all=False, beam_width=1, inner_radius=None,
                                     initial_slack=1.0, range_slack=1.0, max_returned=None, rerank=False):
        """range_search_filtered_pq over the MinMax store (the distances of search_batch_minmax).  A query holding a NaN
        after the store's transform fails the call."""
        return self._range_filtered_quant("minmax", queries, masks, l_search, radius, match_all=match_all, beam_width=beam_width,
                                          inner_radius=inner_radius, initial_slack=initial_slack, range_slack=range_slack,
                                          max_returned=max_returned, rerank=rerank)

    def _range_filtered_quant_device(self, store, d_queries, d_masks, nq, l_search, radius, match_all=False, rerank=False, **kw):
        return RangeResults(self, getattr(_lib.lib(), f"dab_range_search_filtered_{store}_device"), C.c_void_p(d_queries), nq, l_search,
                            radius, masks=C.c_void_p(d_masks), match_all=match_all, rerank=bool(rerank), **kw)

    def range_search_filtered_pq_device(self, d_queries, d_masks, nq, l_search, radius, *, match_all=False, beam_width=1,
                                        inner_radius=None, initial_slack=1.0, range_slack=1.0, max_returned=None, rerank=False):
        """range_search_filtered_pq of `nq` queries and masks at the device pointers `d_queries` and `d_masks` (integers):
        a RangeResults"""
        return self._range_filtered_quant_device("pq", d_queries, d_masks, nq, l_search, radius, match_all=match_all, beam_width=beam_width,
                                                 inner_radius=inner_radius, initial_slack=initial_slack, range_slack=range_slack,
                                                 max_returned=max_returned, rerank=rerank)

    def range_search_filtered_sq_device(self, d_queries, d_masks, nq, l_search, radius, *, match_all=False, beam_width=1,
                                        inner_radius=None, initial_slack=1.0, range_slack=1.0, max_returned=None, rerank=False):
        """range_search_filtered_sq of `nq` queries and masks at the device pointers `d_queries` and `d_masks` (integers):
        a RangeResults"""
        return self._range_filtered_quant_device("sq", d_queries, d_masks, nq, l_search, radius, match_all=match_all, beam_width=beam_width,
                                                 inner_radius=inner_radius, initial_slack=initial_slack, range_slack=range_slack,
                                                 max_returned=max_returned, rerank=rerank)

    def range_search_filtered_minmax_device(self, d_queries, d_masks, nq, l_search, radius, *, match_all=False, beam_width=1,
                                            inner_radius=None, initial_slack=1.0, range_slack=1.0, max_returned=None, rerank=False):
        """range_search_filtered_minmax of `nq` queries and masks at the device pointers `d_queries` and `d_masks`
        (integers): a RangeResults"""
        return self._range_filtered_quant_device("minmax", d_queries, d_masks, nq, l_search, radius, match_all=match_all,
                                                 beam_width=beam_width, inner_radius=inner_radius, initial_slack=initial_slack,
                                                 range_slack=range_slack, max_returned=max_returned, rerank=rerank)

    def search_batch_device(self, d_queries, nq, k, l_search, beam_width, d_ids, d_dists, d_counts=0, d_cmps=0, d_hops=0):
        """Same with device pointers (integers); results stay in HBM."""
        check(_lib.lib().dab_search_batch_device(self._h, C.c_void_p(d_queries), nq, k, l_search, beam_width,
                                                 C.c_void_p(d_ids), C.c_void_p(d_dists), C.c_void_p(d_counts or None),
                                                 C.c_void_p(d_cmps or None), C.c_void_p(d_hops or None)))

    def upload_attributes(self, values, present=None, first=0):
        """The attribute of ids first .. first + len(values) - 1 for search_batch_diverse: `values` u32, `present` bool
        (None: every id of the range has its value; False: the id has no attribute, so diverse search skips it)."""
        values = np.ascontiguousarray(values, np.uint32).ravel()
        pres = None if present is None else np.ascontiguousarray(present, np.uint8).ravel()
        if pres is not None and pres.shape != values.shape:
            raise ValueError("upload_attributes: present must have one entry per value")
        check(_lib.lib().dab_upload_attributes(self._h, _ptr(values), None if pres is None else _ptr(pres), first, values.shape[0]))

    def search_batch_diverse(self, queries, k, l_search, diverse_k, beam_width=1):
        """Diverse::search for the whole batch: at most diverse_k results per attribute value (upload_attributes);
        (ids [nq,k], dists [nq,k], counts, cmps, hops)."""
        queries = self._queries(queries)
        nq = queries.shape[0]
        ids = np.empty((nq, k), np.uint32)
        dists = np.empty((nq, k), np.float32)
        counts, cmps, hops = (np.empty(nq, np.uint32) for _ in range(3))
        check(_lib.lib().dab_search_batch_diverse(self._h, _ptr(queries), nq, k, l_search, beam_width, diverse_k, _ptr(ids), _ptr(dists),
                                                  _ptr(counts), _ptr(cmps), _ptr(hops)))
        return ids, dists, counts, cmps, hops

    def search_batch_diverse_device(self, d_queries, nq, k, l_search, diverse_k, beam_width, d_ids, d_dists, d_counts=0, d_cmps=0,
                                    d_hops=0):
        """search_batch_diverse with device pointers (integers); results stay in HBM."""
        check(_lib.lib().dab_search_batch_diverse_device(self._h, C.c_void_p(d_queries), nq, k, l_search, beam_width, diverse_k,
                                                         C.c_void_p(d_ids), C.c_void_p(d_dists), C.c_void_p(d_counts or None),
                                                         C.c_void_p(d_cmps or None), C.c_void_p(d_hops or None)))

    def upload_labels(self, labels, first=0):
        """The 64-bit label sets of ids first .. first + len(labels) - 1 for search_batch_filtered (u64 each)."""
        labels = np.ascontiguousarray(labels, np.uint64).ravel()
        check(_lib.lib().dab_upload_labels(self._h, _ptr(labels), first, labels.shape[0]))

    @staticmethod
    def _adaptive(adaptive_l):
        if adaptive_l is None:
            return 0, 1.0
        samples, scale = adaptive_l
        if samples == 0:
            raise ValueError("adaptive_l: sample count cannot be zero")
        return int(samples), float(scale)

    def search_batch_filtered(self, queries, masks, k, l_search, beam_width=1, match_all=False, adaptive_l=None):
        """InlineFilterSearch::search for the whole batch over the label table (upload_labels): query q accepts id i when
        labels[i] & masks[q] != 0 (match_all=False) or == masks[q] (match_all=True); `masks` u64 per query (or one for
        all); adaptive_l: None or (samples, scale).  (ids [nq,k], dists [nq,k], counts, cmps, hops)."""
        queries = self._queries(queries)
        nq = queries.shape[0]
        masks = np.ascontiguousarray(np.broadcast_to(np.asarray(masks, np.uint64), (nq,)))
        samples, scale = self._adaptive(adaptive_l)
        ids = np.empty((nq, k), np.uint32)
        dists = np.empty((nq, k), np.float32)
        counts, cmps, hops = (np.empty(nq, np.uint32) for _ in range(3))
        check(_lib.lib().dab_search_batch_filtered(self._h, _ptr(queries), nq, k, l_search, beam_width, _ptr(masks), int(bool(match_all)),
                                                   samples, scale, _ptr(ids), _ptr(dists), _ptr(counts), _ptr(cmps), _ptr(hops)))
        return ids, dists, counts, cmps, hops

    def search_batch_filtered_device(self, d_queries, nq, k, l_search, beam_width, d_masks, d_ids, d_dists, d_counts=0, d_cmps=0,
                                     d_hops=0, match_all=False, adaptive_l=None):
        """search_batch_filtered with device pointers (integers), the masks included; results stay in HBM, complete on
        return."""
        samples, scale = self._adaptive(adaptive_l)
        check(_lib.lib().dab_search_batch_filtered_device(self._h, C.c_void_p(d_queries), nq, k, l_search, beam_width, C.c_void_p(d_masks),
                                                          int(bool(match_all)), samples, scale, C.c_void_p(d_ids), C.c_void_p(d_dists),
                                                          C.c_void_p(d_counts or None), C.c_void_p(d_cmps or None),
                                                          C.c_void_p(d_hops or None)))

    def _filtered_quant(self, store, queries, masks, k, l_search, beam_width, match_all, adaptive_l, rerank):
        queries = self._queries(queries)
        nq = queries.shape[0]
        masks = np.ascontiguousarray(np.broadcast_to(np.asarray(masks, np.uint64), (nq,)))
        samples, scale = self._adaptive(adaptive_l)
        ids = np.empty((nq, k), np.uint32)
        dists = np.empty((nq, k), np.float32)
        counts, cmps, hops = (np.empty(nq, np.uint32) for _ in range(3))
        fn = getattr(_lib.lib(), f"dab_search_batch_filtered_{store}")
        check(fn(self._h, _ptr(queries), nq, k, l_search, beam_width, _ptr(masks), int(bool(match_all)), samples, scale, int(bool(rerank)),
                 _ptr(ids), _ptr(dists), _ptr(counts), _ptr(cmps), _ptr(hops)))
        return ids, dists, counts, cmps, hops

    def _filtered_quant_device(self, store, d_queries, nq, k, l_search, beam_width, d_masks, d_ids, d_dists, d_counts, d_cmps, d_hops,
                               match_all, adaptive_l, rerank):
        samples, scale = self._adaptive(adaptive_l)
        fn = getattr(_lib.lib(), f"dab_search_batch_filtered_{store}_device")
        check(fn(self._h, C.c_void_p(d_queries), nq, k, l_search, beam_width, C.c_void_p(d_masks), int(bool(match_all)), samples, scale,
                 int(bool(rerank)), C.c_void_p(d_ids), C.c_void_p(d_dists), C.c_void_p(d_counts or None), C.c_void_p(d_cmps or None),
                 C.c_void_p(d_hops or None)))

    def search_batch_filtered_pq(self, queries, masks, k, l_search, beam_width=1, match_all=False, adaptive_l=None, rerank=False):
        """search_batch_filtered with the traversal distances of search_batch_pq (PQ store); rerank=True reranks the
        first L matches by full-precision distance."""
        return self._filtered_quant("pq", queries, masks, k, l_search, beam_width, match_all, adaptive_l, rerank)

    def search_batch_filtered_sq(self, queries, masks, k, l_search, beam_width=1, match_all=False, adaptive_l=None, rerank=False):
        """search_batch_filtered with the traversal distances of search_batch_sq (scalar-quantized store)."""
        return self._filtered_quant("sq", queries, masks, k, l_search, beam_width, match_all, adaptive_l, rerank)

    def search_batch_filtered_minmax(self, queries, masks, k, l_search, beam_width=1, match_all=False, adaptive_l=None, rerank=False):
        """search_batch_filtered with the traversal distances of search_batch_minmax (MinMax store)."""
        return self._filtered_quant("minmax", queries, masks, k, l_search, beam_width, match_all, adaptive_l, rerank)

    def search_batch_filtered_pq_device(self, d_queries, nq, k, l_search, beam_width, d_masks, d_ids, d_dists, d_counts=0, d_cmps=0,
                                        d_hops=0, match_all=False, adaptive_l=None, rerank=False):
        """search_batch_filtered_pq with device pointers (integers), the masks included; results stay in HBM, complete on
        return."""
        self._filtered_quant_device("pq", d_queries, nq, k, l_search, beam_width, d_masks, d_ids, d_dists, d_counts, d_cmps, d_hops,
                                    match_all, adaptive_l, rerank)

    def search_batch_filtered_sq_device(self, d_queries, nq, k, l_search, beam_width, d_masks, d_ids, d_dists, d_counts=0, d_cmps=0,
                                        d_hops=0, match_all=False, adaptive_l=None, rerank=False):
        """search_batch_filtered_sq with device pointers (integers), the masks included; results stay in HBM, complete on
        return."""
        self._filtered_quant_device("sq", d_queries, nq, k, l_search, beam_width, d_masks, d_ids, d_dists, d_counts, d_cmps, d_hops,
                                    match_all, adaptive_l, rerank)

    def search_batch_filtered_minmax_device(self, d_queries, nq, k, l_search, beam_width, d_masks, d_ids, d_dists, d_counts=0, d_cmps=0,
                                            d_hops=0, match_all=False, adaptive_l=None, rerank=False):
        """search_batch_filtered_minmax with device pointers (integers), the masks included; results stay in HBM, complete
        on return."""
        self._filtered_quant_device("minmax", d_queries, nq, k, l_search, beam_width, d_masks, d_ids, d_dists, d_counts, d_cmps, d_hops,
                                    match_all, adaptive_l, rerank)

    def _diverse_quant(self, store, queries, k, l_search, diverse_k, beam_width, rerank):
        queries = self._queries(queries)
        nq = queries.shape[0]
        ids = np.empty((nq, k), np.uint32)
        dists = np.empty((nq, k), np.float32)
        counts, cmps, hops = (np.empty(nq, np.uint32) for _ in range(3))
        fn = getattr(_lib.lib(), f"dab_search_batch_diverse_{store}")
        check(fn(self._h, _ptr(queries), nq, k, l_search, beam_width, diverse_k, int(bool(rerank)), _ptr(ids), _ptr(dists), _ptr(counts),
                 _ptr(cmps), _ptr(hops)))
        return ids, dists, counts, cmps, hops

    def _diverse_quant_device(self, store, d_queries, nq, k, l_search, diverse_k, beam_width, rerank, d_ids, d_dists, d_counts, d_cmps,
                              d_hops):
        fn = getattr(_lib.lib(), f"dab_search_batch_diverse_{store}_device")
        check(fn(self._h, C.c_void_p(d_queries), nq, k, l_search, beam_width, diverse_k, int(bool(rerank)), C.c_void_p(d_ids),
                 C.c_void_p(d_dists), C.c_void_p(d_counts or None), C.c_void_p(d_cmps or None), C.c_void_p(d_hops or None)))

    def search_batch_diverse_pq(self, queries, k, l_search, diverse_k, beam_width=1, rerank=False):
        """search_batch_diverse with the traversal distances of search_batch_pq (PQ store); rerank=True reranks the
        post-processed list by full-precision distance."""
        return self._diverse_quant("pq", queries, k, l_search, diverse_k, beam_width, rerank)

    def search_batch_diverse_sq(self, queries, k, l_search, diverse_k, beam_width=1, rerank=False):
        """search_batch_diverse with the traversal distances of search_batch_sq (scalar-quantized store)."""
        return self._diverse_quant("sq", queries, k, l_search, diverse_k, beam_width, rerank)

    def search_batch_diverse_minmax(self, queries, k, l_search, diverse_k, beam_width=1, rerank=False):
        """search_batch_diverse with the traversal distances of search_batch_minmax (MinMax store)."""
        return self._diverse_quant("minmax", queries, k, l_search, diverse_k, beam_width, rerank)

    def search_batch_diverse_pq_device(self, d_queries, nq, k, l_search, diverse_k, beam_width, d_ids, d_dists, d_counts=0, d_cmps=0,
                                       d_hops=0, rerank=False):
        """search_batch_diverse_pq with device pointers (integers); results stay in HBM, complete on return."""
        self._diverse_quant_device("pq", d_queries, nq, k, l_search, diverse_k, beam_width, rerank, d_ids, d_dists, d_counts, d_cmps, d_hops)

    def search_batch_diverse_sq_device(self, d_queries, nq, k, l_search, diverse_k, beam_width, d_ids, d_dists, d_counts=0, d_cmps=0,
                                       d_hops=0, rerank=False):
        """search_batch_diverse_sq with device pointers (integers); results stay in HBM, complete on return."""
        self._diverse_quant_device("sq", d_queries, nq, k, l_search, diverse_k, beam_width, rerank, d_ids, d_dists, d_counts, d_cmps, d_hops)

    def search_batch_diverse_minmax_device(self, d_queries, nq, k, l_search, diverse_k, beam_width, d_ids, d_dists, d_counts=0, d_cmps=0,
                                           d_hops=0, rerank=False):
        """search_batch_diverse_minmax with device pointers (integers); results stay in HBM, complete on return."""
        self._diverse_quant_device("minmax", d_queries, nq, k, l_search, diverse_k, beam_width, rerank, d_ids, d_dists, d_counts, d_cmps,
                                   d_hops)

    def search_batch_async(self, slot, queries, k, l_search, beam_width=1, out=None):
        """Queue a batch on `slot` (host buffers) and return its output arrays without waiting; they are
        valid after wait(slot).  `queries` is used as passed (it must stay alive and unchanged until then);
        `out` = (ids, dists, counts, cmps, hops) re-uses caller-owned (e.g. pinned) arrays."""
        nq = queries.shape[0]
        if out is None:
            out = (np.empty((nq, k), np.uint32), np.empty((nq, k), np.float32), np.empty(nq, np.uint32),
                   np.empty(nq, np.uint32), np.empty(nq, np.uint32))
        ids, dists, counts, cmps, hops = out
        check(_lib.lib().dab_search_batch_async(self._h, slot, _ptr(queries), nq, k, l_search, beam_width, _ptr(ids), _ptr(dists),
                                                _ptr(counts), _ptr(cmps), _ptr(hops)))
        self._inflight[slot] = (queries, out)
        return out

    def search_batch_device_async(self, slot, d_queries, nq, k, l_search, beam_width, d_ids, d_dists, d_counts=0, d_cmps=0, d_hops=0):
        """Device-pointer flavour of search_batch_async; results stay in HBM."""
        check(_lib.lib().dab_search_batch_device_async(self._h, slot, C.c_void_p(d_queries), nq, k, l_search, beam_width,
                                                       C.c_void_p(d_ids), C.c_void_p(d_dists), C.c_void_p(d_counts or None),
                                                       C.c_void_p(d_cmps or None), C.c_void_p(d_hops or None)))

    def _quantized_async(self, fn, slot, queries, k, l_search, beam_width, rerank, out):
        queries = self._queries(queries)
        nq = queries.shape[0]
        if out is None:
            out = (np.empty((nq, k), np.uint32), np.empty((nq, k), np.float32), np.empty(nq, np.uint32),
                   np.empty(nq, np.uint32), np.empty(nq, np.uint32))
        ids, dists, counts, cmps, hops = out
        check(fn(self._h, slot, _ptr(queries), nq, k, l_search, beam_width, int(bool(rerank)), _ptr(ids), _ptr(dists),
                 _ptr(counts), _ptr(cmps), _ptr(hops)))
        self._inflight[slot] = (queries, out)
        return out

    def _quantized_device_async(self, fn, slot, d_queries, nq, k, l_search, beam_width, d_ids, d_dists, d_counts, d_cmps, d_hops,
                                rerank):
        check(fn(self._h, slot, C.c_void_p(d_queries), nq, k, l_search, beam_width, int(bool(rerank)), C.c_void_p(d_ids),
                 C.c_void_p(d_dists), C.c_void_p(d_counts or None), C.c_void_p(d_cmps or None), C.c_void_p(d_hops or None)))

    def search_batch_pq_async(self, slot, queries, k, l_search, beam_width=1, rerank=False, out=None):
        """search_batch_pq as a batch in flight on `slot`: returns the output arrays that wait(slot) fills (see
        search_batch_async)."""
        return self._quantized_async(_lib.lib().dab_search_batch_pq_async, slot, queries, k, l_search, beam_width, rerank, out)

    def search_batch_pq_device_async(self, slot, d_queries, nq, k, l_search, beam_width, d_ids, d_dists, d_counts=0, d_cmps=0,
                                     d_hops=0, rerank=True):
        """Device-pointer flavour of search_batch_pq_async; results stay in HBM."""
        self._quantized_device_async(_lib.lib().dab_search_batch_pq_device_async, slot, d_queries, nq, k, l_search, beam_width,
                                     d_ids, d_dists, d_counts, d_cmps, d_hops, rerank)

    def search_batch_sq_async(self, slot, queries, k, l_search, beam_width=1, rerank=False, out=None):
        """search_batch_sq as a batch in flight on `slot`: returns the output arrays that wait(slot) fills."""
        return self._quantized_async(_lib.lib().dab_search_batch_sq_async, slot, queries, k, l_search, beam_width, rerank, out)

    def search_batch_sq_device_async(self, slot, d_queries, nq, k, l_search, beam_width, d_ids, d_dists, d_counts=0, d_cmps=0,
                                     d_hops=0, rerank=True):
        self._quantized_device_async(_lib.lib().dab_search_batch_sq_device_async, slot, d_queries, nq, k, l_search, beam_width,
                                     d_ids, d_dists, d_counts, d_cmps, d_hops, rerank)

    def search_batch_minmax_async(self, slot, queries, k, l_search, beam_width=1, rerank=False, out=None):
        """search_batch_minmax as a batch in flight on `slot`: returns the output arrays that wait(slot) fills.  A query
        holding a NaN after the transform makes wait(slot) fail."""
        return self._quantized_async(_lib.lib().dab_search_batch_minmax_async, slot, queries, k, l_search, beam_width, rerank, out)

    def search_batch_minmax_device_async(self, slot, d_queries, nq, k, l_search, beam_width, d_ids, d_dists, d_counts=0, d_cmps=0,
                                         d_hops=0, rerank=False):
        self._quantized_device_async(_lib.lib().dab_search_batch_minmax_device_async, slot, d_queries, nq, k, l_search, beam_width,
                                     d_ids, d_dists, d_counts, d_cmps, d_hops, rerank)

    def wait(self, slot):
        """Join the batch in flight on `slot` (no-op when idle)."""
        check(_lib.lib().dab_wait(self._h, slot))
        return self._inflight.pop(slot, (None, None))[1]

    # -- PQ
    def pq_populate_lut(self, queries, metric=None):
        queries = np.ascontiguousarray(queries, np.float32)
        out = np.empty((queries.shape[0], self.pq_chunks, self.pq_centers), np.float32)
        check(_lib.lib().dab_pq_populate_lut(self._h, _ptr(queries), queries.shape[0],
                                             int(self.metric if metric is None else metric), _ptr(out)))
        return out

    def pq_distances(self, queries, ids):
        queries = np.ascontiguousarray(queries, np.float32)
        ids = np.ascontiguousarray(ids, np.uint32)
        out = np.empty(ids.shape, np.float32)
        check(_lib.lib().dab_pq_distances(self._h, _ptr(queries), queries.shape[0], _ptr(ids), ids.shape[1], _ptr(out)))
        return out

    def search_batch_pq(self, queries, k, l_search, beam_width=1, rerank=False):
        """KNN::search with PQ ADC traversal distances (providers' QuantAccessor); rerank=True adds the
        providers' full-precision Rerank post-processing."""
        queries = self._queries(queries)
        nq = queries.shape[0]
        ids = np.empty((nq, k), np.uint32)
        dists = np.empty((nq, k), np.float32)
        counts = np.empty(nq, np.uint32)
        cmps = np.empty(nq, np.uint32)
        hops = np.empty(nq, np.uint32)
        fn = _lib.lib().dab_search_batch_pq_rerank if rerank else _lib.lib().dab_search_batch_pq
        check(fn(self._h, _ptr(queries), nq, k, l_search, beam_width, _ptr(ids), _ptr(dists), _ptr(counts), _ptr(cmps), _ptr(hops)))
        return ids, dists, counts, cmps, hops

    def search_batch_pq_device(self, d_queries, nq, k, l_search, beam_width, d_ids, d_dists, d_counts=0, d_cmps=0, d_hops=0,
                               rerank=True):
        """Same with device pointers (integers); results stay in HBM."""
        check(_lib.lib().dab_search_batch_pq_device(self._h, C.c_void_p(d_queries), nq, k, l_search, beam_width, int(bool(rerank)),
                                                    C.c_void_p(d_ids), C.c_void_p(d_dists), C.c_void_p(d_counts or None),
                                                    C.c_void_p(d_cmps or None), C.c_void_p(d_hops or None)))

    def pq_self_distances(self, a, b):
        """DistanceComputer over two stored codes (the PQ prune path): out[i] = d(code[a[i]], code[b[i]])."""
        a = np.ascontiguousarray(a, np.uint32)
        b = np.ascontiguousarray(b, np.uint32)
        if a.shape != b.shape or a.ndim != 1:
            raise DabError(1, "a and b must be 1-d u32 arrays of equal length")
        out = np.empty(a.shape[0], np.float32)
        check(_lib.lib().dab_pq_self_distances(self._h, _ptr(a), _ptr(b), a.shape[0], _ptr(out)))
        return out

    # -- scalar-quantized store
    def upload_sq(self, nbits, shift, scale, shift_square_norm, mean_norm=0.0, rows=None):
        """SQStore<NBITS>: the quantizer and (optionally) the canonical-front rows
        (f32 compensation | dense N-bit codes) of every point including the start points."""
        shift = np.ascontiguousarray(shift, np.float32)
        if shift.shape != (self.dim,):
            raise DabError(1, "shift must have dim entries")
        row_bytes = 4 + (self.dim * nbits + 7) // 8
        if rows is not None:
            rows = np.ascontiguousarray(rows, np.uint8)
            if rows.shape != (self.n_points + self.n_start, row_bytes):
                raise DabError(1, "rows must be (n_points + n_start) x (4 + ceil(dim * nbits / 8)) bytes")
        check(_lib.lib().dab_upload_sq(self._h, int(nbits), _ptr(shift), float(scale), float(shift_square_norm),
                                       float(mean_norm), _ptr(rows) if rows is not None else None))
        self.sq_nbits = int(nbits)

    def sq_encode_all(self):
        check(_lib.lib().dab_sq_encode_all(self._h))

    def download_sq(self):
        rows = np.empty((self.n_points + self.n_start, 4 + (self.dim * self.sq_nbits + 7) // 8), np.uint8)
        check(_lib.lib().dab_sq_download(self._h, _ptr(rows)))
        return rows

    def search_batch_sq(self, queries, k, l_search, beam_width=1, rerank=False):
        """KNN::search through the scalar-quantized accessor; rerank=True adds the full-precision Rerank."""
        queries = self._queries(queries)
        nq = queries.shape[0]
        ids = np.empty((nq, k), np.uint32)
        dists = np.empty((nq, k), np.float32)
        counts = np.empty(nq, np.uint32)
        cmps = np.empty(nq, np.uint32)
        hops = np.empty(nq, np.uint32)
        check(_lib.lib().dab_search_batch_sq(self._h, _ptr(queries), nq, k, l_search, beam_width, int(bool(rerank)),
                                             _ptr(ids), _ptr(dists), _ptr(counts), _ptr(cmps), _ptr(hops)))
        return ids, dists, counts, cmps, hops

    def search_batch_sq_device(self, d_queries, nq, k, l_search, beam_width, d_ids, d_dists, d_counts=0, d_cmps=0, d_hops=0,
                               rerank=True):
        check(_lib.lib().dab_search_batch_sq_device(self._h, C.c_void_p(d_queries), nq, k, l_search, beam_width, int(bool(rerank)),
                                                    C.c_void_p(d_ids), C.c_void_p(d_dists), C.c_void_p(d_counts or None),
                                                    C.c_void_p(d_cmps or None), C.c_void_p(d_hops or None)))

    # -- MinMax store
    def upload_minmax(self, nbits, grid_scale=1.0, transform=None, rows=None):
        """MinMaxElement<NBITS> as the index's vector representation: MinMaxQuantizer(transform or Transform::Null,
        grid_scale) and (optionally) the canonical-front Data<NBITS> rows of every point including the start points.
        The index keeps its own copy of `transform`."""
        out_dim = self.dim if transform is None else transform.output_dim
        row_bytes = _lib.lib().dab_minmax_row_bytes(out_dim, int(nbits))
        if rows is not None:
            rows = np.ascontiguousarray(rows, np.uint8)
            if row_bytes and rows.shape != (self.n_points + self.n_start, row_bytes):
                raise DabError(1, f"rows must be (n_points + n_start) x {row_bytes} bytes")
        check(_lib.lib().dab_upload_minmax(self._h, int(nbits), float(grid_scale), transform._h if transform is not None else None,
                                           _ptr(rows) if rows is not None else None))
        self.mm_row_bytes = row_bytes

    def minmax_encode_all(self):
        check(_lib.lib().dab_minmax_encode_all(self._h))

    def download_minmax(self):
        rows = np.empty((self.n_points + self.n_start, self.mm_row_bytes), np.uint8)
        check(_lib.lib().dab_minmax_download(self._h, _ptr(rows)))
        return rows

    def search_batch_minmax(self, queries, k, l_search, beam_width=1, rerank=False):
        """KNN::search through the MinMax store; rerank=True adds the full-precision Rerank."""
        queries = self._queries(queries)
        nq = queries.shape[0]
        ids = np.empty((nq, k), np.uint32)
        dists = np.empty((nq, k), np.float32)
        counts = np.empty(nq, np.uint32)
        cmps = np.empty(nq, np.uint32)
        hops = np.empty(nq, np.uint32)
        check(_lib.lib().dab_search_batch_minmax(self._h, _ptr(queries), nq, k, l_search, beam_width, int(bool(rerank)),
                                                 _ptr(ids), _ptr(dists), _ptr(counts), _ptr(cmps), _ptr(hops)))
        return ids, dists, counts, cmps, hops

    def search_batch_minmax_device(self, d_queries, nq, k, l_search, beam_width, d_ids, d_dists, d_counts=0, d_cmps=0, d_hops=0,
                                   rerank=False):
        check(_lib.lib().dab_search_batch_minmax_device(self._h, C.c_void_p(d_queries), nq, k, l_search, beam_width, int(bool(rerank)),
                                                        C.c_void_p(d_ids), C.c_void_p(d_dists), C.c_void_p(d_counts or None),
                                                        C.c_void_p(d_cmps or None), C.c_void_p(d_hops or None)))

    def pq_encode(self, vectors):
        vectors = np.ascontiguousarray(vectors, np.float32)
        out = np.empty((vectors.shape[0], self.pq_chunks), np.uint8)
        check(_lib.lib().dab_pq_encode(self._h, _ptr(vectors), vectors.shape[0], _ptr(out)))
        return out

    # -- build-side reuse / ground truth
    def robust_prune(self, pool_ids, pool_dists, pool_lens, locations, degree, alpha=1.2):
        """robust_prune for a batch of pools -> (ids [n_pools, degree] padded UINT32_MAX, counts)."""
        pool_ids = np.ascontiguousarray(pool_ids, np.uint32)
        pool_dists = np.ascontiguousarray(pool_dists, np.float32)
        pool_lens = np.ascontiguousarray(pool_lens, np.uint32)
        locations = np.ascontiguousarray(locations, np.uint32)
        if pool_ids.ndim != 2 or pool_ids.shape != pool_dists.shape or pool_lens.shape != (pool_ids.shape[0],) \
                or locations.shape != pool_lens.shape:
            raise DabError(1, "robust_prune: expected pool_ids/pool_dists [n_pools, cap], pool_lens/locations [n_pools]")
        out = np.empty((pool_ids.shape[0], degree), np.uint32)
        counts = np.empty(pool_ids.shape[0], np.uint32)
        check(_lib.lib().dab_robust_prune(self._h, _ptr(pool_ids), _ptr(pool_dists), _ptr(pool_lens), _ptr(locations),
                                          pool_ids.shape[0], pool_ids.shape[1], degree, alpha, _ptr(out), _ptr(counts)))
        return out, counts

    def build(self, pruned_degree, l_build, alpha=1.2, batch_size=0):
        check(_lib.lib().dab_build(self._h, pruned_degree, l_build, alpha, batch_size))

    def insert(self, ids, rows, pruned_degree, l_build, alpha=1.2, batch_size=0):
        """DiskANNIndex::insert / multi_insert into the graph as it stands: rows[i] becomes point ids[i] (in the index and
        in every quantized store that holds rows) and is linked in consecutive chunks of batch_size (0: 65536)."""
        ids = np.ascontiguousarray(ids, np.uint32).ravel()
        rows = self._rows(rows)
        if rows.shape[0] != ids.shape[0]:
            raise DabError(1, f"insert: {ids.shape[0]} ids for {rows.shape[0]} rows")
        check(_lib.lib().dab_insert(self._h, _ptr(ids), _ptr(rows), ids.shape[0], pruned_degree, l_build, alpha, batch_size))

    # -- deletion (Delete of the providers' TableDeleteProviderAsync; DiskANNIndex::consolidate_vector)
    def delete(self, ids):
        """Marks data points deleted: every k-NN search then leaves them out of its results."""
        ids = np.ascontiguousarray(ids, np.uint32).ravel()
        check(_lib.lib().dab_delete(self._h, _ptr(ids), ids.shape[0]))

    def release(self, ids):
        """Clears the deletion mark of deleted points and empties their adjacency rows."""
        ids = np.ascontiguousarray(ids, np.uint32).ravel()
        check(_lib.lib().dab_release(self._h, _ptr(ids), ids.shape[0]))

    def delete_status(self, ids):
        """bool [n]: which of `ids` are deleted."""
        ids = np.ascontiguousarray(ids, np.uint32).ravel()
        out = np.zeros(ids.shape[0], np.uint8)
        check(_lib.lib().dab_delete_status(self._h, _ptr(ids), ids.shape[0], _ptr(out)))
        return out.astype(bool)

    def consolidate(self, pruned_degree, alpha=1.2):
        """consolidate_vector for every node: repairs the lists around deleted points; returns the lists rewritten."""
        n = C.c_uint64()
        check(_lib.lib().dab_consolidate(self._h, pruned_degree, alpha, C.byref(n)))
        return int(n.value)

    INPLACE_METHODS = {"visited_and_topk": 0, "two_hop_and_one_hop": 1, "one_hop": 2}

    def inplace_delete(self, ids, num_to_replace, method, pruned_degree, alpha=1.2, k_value=20, l_value=50, batch_size=1):
        """multi_inplace_delete: deletes `ids` and repairs only the lists around them, in consecutive chunks of batch_size
        (1: inplace_delete id by id; 0: one chunk).  `method`: "visited_and_topk" (k_value, l_value),
        "two_hop_and_one_hop" or "one_hop", or the DAB_INPLACE_* number."""
        ids = np.ascontiguousarray(ids, np.uint32).ravel()
        m = self.INPLACE_METHODS[method] if isinstance(method, str) else int(method)
        check(_lib.lib().dab_inplace_delete(self._h, _ptr(ids), ids.shape[0], m, num_to_replace, k_value, l_value, pruned_degree, alpha,
                                            batch_size))

    def drop_deleted_neighbors(self, pruned_degree, only_orphans=False):
        """drop_deleted_neighbors for every node: removes the edges to deleted points; returns the lists rewritten."""
        n = C.c_uint64()
        check(_lib.lib().dab_drop_deleted_neighbors(self._h, pruned_degree, 1 if only_orphans else 0, C.byref(n)))
        return int(n.value)

    # -- graph checks (DiskANNIndex::count_reachable_nodes / get_degree_stats) and the final prune (prune_range)
    @staticmethod
    def _id_list(ids):
        """(pointer, n) of an explicit id list; an empty list still passes a valid pointer (None means "the default")"""
        ids = np.ascontiguousarray(ids, np.uint32).ravel()
        return _ptr(ids if ids.size else np.zeros(1, np.uint32)), ids.shape[0], ids

    def count_reachable(self, start_ids=None):
        """count_reachable_nodes: the ids a breadth-first walk reaches from start_ids (None: the start points)."""
        n = C.c_uint64()
        if start_ids is None:
            check(_lib.lib().dab_count_reachable(self._h, None, 0, C.byref(n)))
        else:
            p, k, _keep = self._id_list(start_ids)
            check(_lib.lib().dab_count_reachable(self._h, p, k, C.byref(n)))
        return int(n.value)

    def degree_stats(self, ids=None):
        """get_degree_stats over ids (None: every id) -> (max_degree, avg_degree as np.float32, min_degree,
        cnt_less_than_two)."""
        mx, avg, mn, lt2 = C.c_uint32(), C.c_float(), C.c_uint32(), C.c_uint64()
        p, k, _keep = (None, 0, None) if ids is None else self._id_list(ids)
        check(_lib.lib().dab_degree_stats(self._h, p, k, C.byref(mx), C.byref(avg), C.byref(mn), C.byref(lt2)))
        return int(mx.value), np.float32(avg.value), int(mn.value), int(lt2.value)

    def prune_range(self, ids, pruned_degree, alpha=1.2):
        """prune_range over ids (None: every id): robust_prune_list of every list longer than pruned_degree; returns the
        lists rewritten.  Arguments in the C ABI's order, as the C++ and Rust bindings take them."""
        n = C.c_uint64()
        p, k, _keep = (None, 0, None) if ids is None else self._id_list(ids)
        check(_lib.lib().dab_prune_range(self._h, p, k, pruned_degree, alpha, C.byref(n)))
        return int(n.value)

    def flat_knn(self, queries, k):
        queries = self._queries(queries)
        ids = np.empty((queries.shape[0], k), np.uint32)
        dists = np.empty((queries.shape[0], k), np.float32)
        check(_lib.lib().dab_flat_knn(self._h, _ptr(queries), queries.shape[0], k, _ptr(ids), _ptr(dists)))
        return ids, dists

    def flat_knn_tc(self, queries, k):
        """The exhaustive scan as a wgmma GEMM with fused candidate selection + exact re-scoring."""
        queries = self._queries(queries)
        ids = np.empty((queries.shape[0], k), np.uint32)
        dists = np.empty((queries.shape[0], k), np.float32)
        check(_lib.lib().dab_flat_knn_tc(self._h, _ptr(queries), queries.shape[0], k, _ptr(ids), _ptr(dists)))
        return ids, dists


class PagedSearch:
    """PagedSearch (diskann/src/graph/search/paged.rs) over a query batch: successive, non-overlapping pages of one
    resumable search per query.  Use as a context manager or call close(); closing the index closes it too."""

    def __init__(self, index, queries, l_search, begin=None):
        """`begin`: the entry point that opens the session (dab_paged_search_begin, or a quantized store's form)"""
        self._h = C.c_void_p()
        self.index, self.nq, self.l_search = index, queries.shape[0], int(l_search)
        begin = begin or _lib.lib().dab_paged_search_begin
        check(begin(index._h, _ptr(queries), self.nq, self.l_search, C.byref(self._h)))
        index._paged.add(self)

    def next_page(self, k):
        """(ids [nq, k], dists [nq, k], counts, cmps, hops): the next page of at most k results per query, padded with
        UINT32_MAX / +inf; counts[q] == 0 once query q is exhausted; cmps / hops are the session's cumulative counts."""
        if not self._h.value:
            raise DabError(1, "next_page: the paged search is closed")
        ids = np.empty((self.nq, k), np.uint32)
        dists = np.empty((self.nq, k), np.float32)
        counts = np.empty(self.nq, np.uint32)
        cmps = np.empty(self.nq, np.uint32)
        hops = np.empty(self.nq, np.uint32)
        check(_lib.lib().dab_paged_search_next(self._h, k, _ptr(ids), _ptr(dists), _ptr(counts), _ptr(cmps), _ptr(hops)))
        return ids, dists, counts, cmps, hops

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            _lib.lib().dab_paged_search_end(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class RangeResults:
    """One range search batch's results, resident on the device (dab_range): a snapshot that later writes to the index
    do not change.  Use as a context manager or call close(); closing the index closes it too."""

    def __init__(self, index, search, queries, nq, l_search, radius, beam_width=1, inner_radius=None, initial_slack=1.0,
                 range_slack=1.0, max_returned=None, rerank=None, masks=None, match_all=False):
        """`rerank`: None for the full-precision call, else the rerank flag of a quantized store's call; `masks`: None,
        else the masks pointer of a filtered call, which takes match_all after it (and the rerank flag after that over a
        store)"""
        self._h = C.c_void_p()
        self.nq = int(nq)
        store_args = () if masks is None else (masks, int(bool(match_all)))
        if rerank is not None:
            store_args += (int(bool(rerank)),)
        check(search(index._h, queries, self.nq, l_search, beam_width, radius, int(inner_radius is not None),
                     0.0 if inner_radius is None else inner_radius, initial_slack, range_slack, max_returned or 0, *store_args,
                     C.byref(self._h)))
        # the index outlives the set: when both are collected together, close() sees whether dab_destroy already freed it
        self._index = index
        index._ranges.add(self)

    def _live(self):
        if not self._h.value:
            raise DabError(1, "the range search results are closed")
        return self._h

    def offsets(self):
        """(offsets [nq + 1] u64, cmps, hops, second_round [nq] bool)"""
        offsets = np.empty(self.nq + 1, np.uint64)
        cmps, hops = np.empty(self.nq, np.uint32), np.empty(self.nq, np.uint32)
        second = np.empty(self.nq, np.uint8)
        check(_lib.lib().dab_range_offsets(self._live(), _ptr(offsets), _ptr(cmps), _ptr(hops), _ptr(second)))
        return offsets, cmps, hops, second.astype(bool)

    def total(self):
        offsets = np.empty(self.nq + 1, np.uint64)
        check(_lib.lib().dab_range_offsets(self._live(), _ptr(offsets), None, None, None))
        return int(offsets[-1])

    def results(self):
        """(ids, dists) of every query, in query order"""
        n = self.total()
        ids, dists = np.empty(n, np.uint32), np.empty(n, np.float32)
        check(_lib.lib().dab_range_results(self._live(), _ptr(ids), _ptr(dists)))
        return ids, dists

    def results_device(self, d_ids, d_dists):
        """the results into device buffers (integers) of total() entries each"""
        check(_lib.lib().dab_range_results_device(self._live(), C.c_void_p(d_ids), C.c_void_p(d_dists)))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            if self._index._h.value:  # else released by dab_destroy
                _lib.lib().dab_range_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()
