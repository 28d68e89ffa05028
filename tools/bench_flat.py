"""tuning aid: exhaustive scan, exact CUDA-core kernel vs the tensor-core (wgmma) path (CUDA-event timing of the whole call
minus host copies is not separated here: both go through the host API with the same copies)."""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import diskann_b200 as dab

n, d = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000, 128
rng = np.random.default_rng(0)
centers = rng.standard_normal((1024, d), dtype=np.float32)
base = np.empty((n + 1, d), np.float32)
for i in range(0, n + 1, 1 << 18):
    m = min(1 << 18, n + 1 - i)
    base[i:i + m] = centers[rng.integers(0, 1024, m)] + np.float32(0.3) * rng.standard_normal((m, d), dtype=np.float32)
with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, d, n, 1, 8) as g:
    g.upload_vectors(base)
    for nq in (1000, 10000):
        q = centers[rng.integers(0, 1024, nq)] + np.float32(0.3) * rng.standard_normal((nq, d), dtype=np.float32)
        g.flat_knn_tc(q[:128], 10)  # builds the bf16 operand copy of the base
        for name, fn in (("exact", g.flat_knn), ("wgmma", g.flat_knn_tc)):
            fn(q, 10)
            t0 = time.perf_counter()
            ids, dist = fn(q, 10)
            dt = time.perf_counter() - t0
            print(f"{name:8s} nq={nq:6d} n={n}: {dt * 1e3:8.2f} ms  ({2.0 * nq * n * d / dt / 1e12:6.1f} useful TFLOP/s)", flush=True)
            if name == "exact":
                want = (ids, dist)
            else:
                print("   ids equal:", bool(np.array_equal(ids, want[0])), " dist bits equal:", bool(np.array_equal(dist.view(np.uint32), want[1].view(np.uint32))))
