#!/usr/bin/env python3
"""Extracts the portable golden vectors of the reference's own tests into tests/golden/.

Run against a checkout of the reference (the tests only read the JSON files this writes):
    python tests/golden/make_golden.py <path to the reference checkout>

Sources (paths relative to the reference checkout):
  * diskann-vector/src/distance/distance_provider.rs:744-828  — 2x256 f32 literal vectors whose
    SquaredL2 must be exactly 429141.2 (pins the V3 summation order).
  * diskann/test/generated/graph/test/cases/grid_search/search_{1_100,3_5,4_4}.json — checked-in
    greedy-search baselines (query, top-10 (id, distance), hops, comparisons, beam width).
  * diskann-wide/test_data/float16_conversion.txt — f16 <-> f32 conversion table (a sample).
  * diskann/test/generated/graph/test/cases/grid_insert/insert_{1_100,3_5,4_4}_single/ibc_none.json —
    searches after inserting the lattice points one by one (driver grid_insert.rs:46-250).
  * diskann/test/generated/graph/test/cases/grid_insert/insert_*_batch_*/ibc_none.json — the same after
    DiskANNIndex::multi_insert over fixed chunks of the lattice points (intra_batch_candidates = None).
  * diskann/test/generated/flat/test/cases/flat_knn_search/search_{1_100,2_5,3_4}.json — exhaustive-scan
    baselines (brute-force ground truth ordered by (distance, id), k in the reference's sweep).
Only data (numeric literals / JSON payloads) is extracted; no reference source is copied.
"""
import json
import os
import re
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else "."
OUT = os.path.dirname(os.path.abspath(__file__))


def kat_l2():
    src = open(f"{REF}/diskann-vector/src/distance/distance_provider.rs").read().splitlines()
    # locate `fn distance_test()` and the literal array that follows
    start = next(i for i, l in enumerate(src) if "fn distance_test()" in l)
    text = []
    depth = None
    for l in src[start:]:
        if depth is None:
            if "v: [" in l and "f32" not in l:
                depth = 1
            continue
        if "]," in l and not re.search(r"\d", l):
            break
        text.append(l)
    nums = [float(t) for t in re.findall(r"-?\d+\.\d+(?:e-?\d+)?", " ".join(text))]
    assert len(nums) == 512, len(nums)
    expect_line = next(l for l in src[start:] if "assert_eq!(distance," in l)
    expected = float(re.search(r"assert_eq!\(distance,\s*([0-9.]+)\)", expect_line).group(1))
    json.dump({"source": "diskann-vector/src/distance/distance_provider.rs:744-828",
               "dim": 256, "metric": "L2", "values": nums, "expected": expected},
              open(f"{OUT}/kat_l2_f32_256.json", "w"))
    print("kat_l2_f32_256.json", len(nums), expected)


def grid_search():
    out = []
    for name in ("search_1_100", "search_3_5", "search_4_4"):
        path = f"{REF}/diskann/test/generated/graph/test/cases/grid_search/{name}.json"
        payload = json.load(open(path))["payload"]
        for p in payload:
            out.append({
                "case": name,
                "grid_dims": p["grid_dims"], "grid_size": p["grid_size"],
                "beam_width": p["beam_width"], "query": p["query"],
                "num_results": p["num_results"], "results": p["results"],
                "comparisons": p["comparisons"], "hops": p["hops"],
            })
    json.dump({"source": "diskann/test/generated/graph/test/cases/grid_search/*.json "
                         "(driver diskann/src/graph/test/cases/grid_search.rs:86-207: k=10, L=10, "
                         "L2, start point id u32::MAX at (size,..,size) linked to the last node)",
               "cases": out}, open(f"{OUT}/grid_search.json", "w"), indent=0)
    print("grid_search.json", len(out))


def grid_insert():
    out = []
    for name in ("insert_1_100_single", "insert_3_5_single", "insert_4_4_single"):
        path = f"{REF}/diskann/test/generated/graph/test/cases/grid_insert/{name}/ibc_none.json"
        p = json.load(open(path))["payload"]
        out.append({
            "case": name, "grid_dims": p["grid_dims"], "grid_size": p["grid_size"], "num_inserted": p["num_inserted"],
            "set_neighbors": p["insert_metrics"]["set_neighbors"], "append_neighbors": p["insert_metrics"]["append_neighbors"],
            "searches": [{"beam_width": q["beam_width"], "query": q["query"], "num_results": q["num_results"],
                          "results": q["results"], "comparisons": q["comparisons"], "hops": q["hops"]} for q in p["searches"]],
        })
    json.dump({"source": "diskann/test/generated/graph/test/cases/grid_insert/insert_*_single/ibc_none.json (driver "
                         "diskann/src/graph/test/cases/grid_insert.rs:46-250: empty provider with the start point at "
                         "(size,..,size), max_degree = 2*dims, pruned degree = max(max_degree - 2, 2), L_build = 100, L2, "
                         "points inserted one by one in lattice order; then k = 10, L = 10 searches)",
               "cases": out}, open(f"{OUT}/grid_insert.json", "w"), indent=0)
    print("grid_insert.json", len(out))


def flat_knn():
    out = []
    for name in ("search_1_100", "search_2_5", "search_3_4"):
        path = f"{REF}/diskann/test/generated/flat/test/cases/flat_knn_search/{name}.json"
        for p in json.load(open(path))["payload"]:
            out.append({"case": name, "grid_dims": p["grid_dims"], "grid_size": p["grid_size"], "k": p["k"],
                        "query": p["query"], "ground_truth": p["ground_truth"], "top_k_distances": p["top_k_distances"],
                        "comparisons": p["comparisons"], "result_count": p["result_count"]})
    json.dump({"source": "diskann/test/generated/flat/test/cases/flat_knn_search/*.json (driver "
                         "diskann/src/flat/test/cases/flat_knn_search.rs:95-196: size^dims lattice rows, L2, "
                         "ground truth sorted by (distance asc, id asc))",
               "cases": out}, open(f"{OUT}/flat_knn.json", "w"), indent=0)
    print("flat_knn.json", len(out))


def f16_table():
    path = f"{REF}/diskann-wide/test_data/float16_conversion.txt"
    lines = open(path).read().splitlines()
    assert len(lines) == 65536
    sample = []
    for i in range(0, 65536, 97):
        bits, val = [t.strip() for t in lines[i].split(",")]
        sample.append([int(bits, 16), val])
    json.dump({"source": "diskann-wide/test_data/float16_conversion.txt (every 97th of 65536 rows)",
               "rows": sample}, open(f"{OUT}/float16_sample.json", "w"))
    print("float16_sample.json", len(sample))


def grid_insert_batch():
    out = []
    for name, batch in (("insert_1_100_batch_100", 100), ("insert_3_5_batch_125", 125), ("insert_3_5_batch_25", 25),
                        ("insert_4_4_batch_25", 25), ("insert_4_4_batch_256", 256)):
        path = f"{REF}/diskann/test/generated/graph/test/cases/grid_insert/{name}/ibc_none.json"
        p = json.load(open(path))["payload"]
        out.append({
            "case": name, "batch": batch, "grid_dims": p["grid_dims"], "grid_size": p["grid_size"], "num_inserted": p["num_inserted"],
            "set_neighbors": p["insert_metrics"]["set_neighbors"], "append_neighbors": p["insert_metrics"]["append_neighbors"],
            "searches": [{"beam_width": q["beam_width"], "query": q["query"], "num_results": q["num_results"],
                          "results": q["results"], "comparisons": q["comparisons"], "hops": q["hops"]} for q in p["searches"]],
        })
    json.dump({"source": "diskann/test/generated/graph/test/cases/grid_insert/insert_*_batch_*/ibc_none.json (driver "
                         "diskann/src/graph/test/cases/grid_insert.rs:46-250, run_build with batchsize = Some(batch): "
                         "DiskANNIndex::multi_insert over consecutive chunks of the lattice points, intra_batch_candidates = None; "
                         "same provider / degrees / L_build as the single-insert cases; then k = 10, L = 10 searches)",
               "cases": out}, open(f"{OUT}/grid_insert_batch.json", "w"), indent=0)
    print("grid_insert_batch.json", len(out))


if __name__ == "__main__":
    if not os.path.isdir(REF):
        sys.exit("reference checkout not present; fixtures are already committed")
    kat_l2()
    grid_search()
    grid_insert()
    grid_insert_batch()
    flat_knn()
    f16_table()
