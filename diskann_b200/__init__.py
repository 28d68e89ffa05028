"""diskann_b200 — H100-native (sm_90a) batched distance hot path for microsoft/DiskANN.

The package is a thin host-side mirror of the reference interface for this path over the C ABI
in include/diskann_b200.h (libdiskann_b200.so).  It holds no CPU implementation: importing
works anywhere, but every compute entry point needs the CUDA library and a GPU.
"""
from .index import (DabError, DType, GpuIndex, Metric, PagedSearch, RangeResults, Transform, distance_comparer, launch_count, minmax_compress,  # noqa: F401
                    minmax_distances, minmax_query_distances, pair_distances)
from ._lib import LIB_PATH, SYMBOLS, lib  # noqa: F401

MAX_SLOTS = 4  # DAB_MAX_SLOTS (include/diskann_b200.h): batches that can be in flight on one index

__all__ = ["DabError", "DType", "GpuIndex", "Metric", "PagedSearch", "RangeResults", "distance_comparer", "launch_count", "pair_distances", "minmax_compress", "minmax_distances", "minmax_query_distances",
           "Transform", "LIB_PATH", "SYMBOLS", "lib", "MAX_SLOTS"]
