"""debug aid: one small pass over every kernel family, sized to run under
`compute-sanitizer --tool memcheck` (or racecheck / initcheck) in about a minute."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import diskann_b200 as dab

rng = np.random.default_rng(0)
if len(sys.argv) > 1 and sys.argv[1] == "pq":
    # only the product-quantization kernels (search_kernel_pqs with its cp.async row hand-off and the two-tile merge,
    # pq_fused_kernel, the global-table kernel, rerank): `compute-sanitizer --tool racecheck python tools/sanitize_check.py pq`
    for dt, ddt, d, chunks in ((np.float32, dab.DType.f32, 100, 25), (np.int8, dab.DType.i8, 32, 4), (np.float32, dab.DType.f32, 40, 7)):
        n = 1500
        base = (rng.normal(size=(n + 1, d)) * (30 if dt == np.int8 else 1)).astype(dt)
        with dab.GpuIndex(ddt, dab.Metric.L2, d, n, 1, 41) as g:
            g.upload_vectors(base)
            adj = np.zeros((n + 1, 42), np.uint32)             # a random 24-regular graph: traversal only, no build kernels here
            adj[:, 0] = 24
            adj[:, 1:25] = rng.integers(0, n, (n + 1, 24))
            g.upload_graph(adj)
            g.pq_train(base[:1200].astype(np.float32), chunks, 64, 2, 7)
            g.pq_encode_all()
            a = g.search_batch_pq(base[:48], 5, 40, 1, rerank=True)
            b = g.search_batch_pq(base[:48], 5, 600, 1, rerank=True)   # list longer than one merge tile
            c = g.search_batch_pq(base[:48], 5, 64, 2)
            ids = rng.integers(0, n + 1, (20, 300)).astype(np.uint32)
            lut = g.pq_populate_lut(base[:20].astype(np.float32))
            dd = g.pq_distances(base[:20].astype(np.float32), ids)
            pq = g.download_pq()
        # the same index and codes once more, with the per-warp tables in global memory (search_kernel_pq, pq_lut_kernel)
        os.environ["DAB_TEST_PQ_GLOBAL_LUT"] = "1"
        with dab.GpuIndex(ddt, dab.Metric.L2, d, n, 1, 41) as g:
            g.upload_vectors(base)
            g.upload_graph(adj)
            g.upload_pq(*pq)
            a2 = g.search_batch_pq(base[:48], 5, 40, 1, rerank=True)
            dd2 = g.pq_distances(base[:20].astype(np.float32), ids)
        del os.environ["DAB_TEST_PQ_GLOBAL_LUT"]
        assert np.array_equal(a[0], a2[0]) and np.array_equal(dd.view(np.uint32), dd2.view(np.uint32))
        print(dt.__name__, d, chunks, "pq ok", int(a[2].min()), int(b[2].min()), int(c[2].min()), lut.shape)
    for nb in (8, 4, 1):                                                       # MinMax quantizer: compress + distances
        v = rng.uniform(-1, 1, (200, 77)).astype(np.float32)
        rows, loss = dab.minmax_compress(v, nb, 0.9)
        dmm = dab.minmax_distances(dab.Metric.L2, nb, nb, 77, rows, rows[::-1].copy())
        r8, _ = dab.minmax_compress(v, 8)
        dmx = dab.minmax_distances(dab.Metric.Cosine, 8, nb, 77, r8, rows)
        dq = dab.minmax_query_distances(dab.Metric.L2, nb, v[:9], rows)           # full-precision queries x compressed rows
        print("minmax", nb, rows.shape, bool(np.isfinite(dmm).all() and np.isfinite(dmx).all() and np.isfinite(dq).all()))
    print("sanitize_check pq done")
    sys.exit(0)
for dt, ddt, metric, d in ((np.float32, dab.DType.f32, dab.Metric.L2, 100), (np.float16, dab.DType.f16, dab.Metric.InnerProduct, 61),
                           (np.int8, dab.DType.i8, dab.Metric.L2, 33)):
    n = 3000
    base = (rng.normal(size=(n + 1, d)) * (30 if dt == np.int8 else 1)).astype(dt)
    with dab.GpuIndex(ddt, metric, d, n, 1, 41) as g:
        g.upload_vectors(base)
        g.build(32, 64, 1.2)                                     # search (records) + prune + back-edge kernels
        adj = g.download_graph()
        ids = rng.integers(0, n + 1, (50, 83)).astype(np.uint32)
        ids[0, :5] = 0xFFFFFFFF
        out = g.distances(base[:50], ids)                        # frontier kernels (wide for f32 / f16)
        pairs = g.row_pair_distances(ids[1, :40], ids[2, :40])
        block = g.pairwise(ids[3, :17])
        got = g.search_batch(base[:64], 5, 64, 1)                # search_kernel_v2
        got4 = g.search_batch(base[:64], 5, 40, 4)
        g.upload_attributes(rng.integers(0, 7, n + 1), rng.random(n + 1) < 0.9)
        div = g.search_batch_diverse(base[:64], 5, 40, 2, 1)     # diverse_kernel
        div4 = g.search_batch_diverse(base[:64], 5, 300, 1, 4)
        g.upload_labels(rng.integers(0, 1 << 8, n + 1).astype(np.uint64))
        flt = g.search_batch_filtered(base[:64], 0b101, 5, 40, 1)  # filtered_kernel
        flt4 = g.search_batch_filtered(base[:64], 0b11, 5, 40, 4, match_all=True, adaptive_l=(50, 8.0))
        rad = float(np.median(got[1][:, 4]))                     # range_kernel, range_scan, range_compact
        rng1 = g.range_search(base[:64], 20, rad, initial_slack=0.2)
        rng4 = g.range_search(base[:64], 10, rad * 2, beam_width=4, max_returned=70)
        frng = g.range_search_filtered(base[:64], 0b101, 20, rad * 2, initial_slack=0.2)  # filtered_range_kernel
        frng4 = g.range_search_filtered(base[:64], 0b11, 10, rad * 2, match_all=True, beam_width=4, max_returned=70)
        knn = g.flat_knn(base[:16], 5)
        knn_tc = g.flat_knn_tc(base[:16], 5)                     # wgmma + TMA path
        assert np.array_equal(knn[0], knn_tc[0])
        if dt != np.float16:
            g.pq_train(base[:1500].astype(np.float32), 4, 32, 2, 7)  # k-means++ / Lloyd kernels
            g.pq_encode_all()
            pq = g.search_batch_pq(base[:32], 5, 40, 1, rerank=True)  # PQ traversal + rerank kernel
            g.pq_self_distances(ids[4, :20], ids[5, :20])
            for rr in (False, True):                                 # diverse_kernel_quant<0>, then rerank
                g.search_batch_diverse_pq(base[:32], 5, 40, 2, 1, rerank=rr)
                # search_kernel_pq_starts, range_kernel_quant<0>, then range_rerank_kernel and the segmented sort
                g.range_search_pq(base[:32], 20, rad, initial_slack=0.2, rerank=rr)
                g.search_batch_filtered_pq(base[:32], 0b101, 5, 40, 2, adaptive_l=(30, 4.0), rerank=rr)  # filtered_kernel_quant<0>
                # filtered_range_kernel_quant<0>, then range_rerank_kernel, its unbounded count and filter, the sort
                g.range_search_filtered_pq(base[:32], 0b101, 20, rad * 2, initial_slack=0.2, rerank=rr)
        f32 = base.astype(np.float32)
        std = float(f32.std())
        shift = (f32.mean(0) - np.float32(2.5 * std)).astype(np.float32)
        g.upload_sq(8, shift, 5.0 * std, -float((shift * shift).sum()))
        g.sq_encode_all()
        g.upload_minmax(4, 1.0, None)
        g.minmax_encode_all()
        for rr in (False, True):                                     # diverse_kernel_quant<1> and <2>
            g.search_batch_diverse_sq(base[:32], 5, 40, 2, 2, rerank=rr)
            g.search_batch_diverse_minmax(base[:32], 5, 40, 2, 1, rerank=rr)
            g.range_search_sq(base[:32], 20, rad * 2, beam_width=4, initial_slack=0.2, rerank=rr)  # range_kernel_quant<1> and <2>
            g.range_search_minmax(base[:32], 10, rad * 2, max_returned=70, initial_slack=0.2, rerank=rr)
            g.search_batch_filtered_sq(base[:32], 0b11, 5, 40, 4, match_all=True, rerank=rr)  # filtered_kernel_quant<1> and <2>
            g.search_batch_filtered_minmax(base[:32], 0b101, 5, 40, 1, adaptive_l=(50, 8.0), rerank=rr)
            # filtered_range_kernel_quant<1> and <2>
            g.range_search_filtered_sq(base[:32], 0b11, 10, rad * 2, match_all=True, beam_width=4, max_returned=70, rerank=rr)
            g.range_search_filtered_minmax(base[:32], 0b101, 20, rad * 2, initial_slack=0.2, rerank=rr)
        print(dt.__name__, "deg max", int(adj[:, 0].max()), "search ok", int(got[2].min()), int(got4[2].min()), int(div[2].min()), int(div4[2].min()),
              "filtered", int(flt[2].sum()), int(flt4[2].sum()),
              "finite", bool(np.isfinite(out[1:]).all() and np.isfinite(pairs).all() and np.isfinite(block).all()), knn[0].shape)
print("sanitize_check done")
