#!/usr/bin/env python3
"""Extracts the reference's inline filtered-search baselines into tests/golden/inline_search.json.

Run against a checkout of the reference (the tests only read the JSON file this writes):
    python tests/golden/make_golden_inline.py <path to the reference checkout>

Source (relative to the reference checkout): diskann/test/generated/graph/test/cases/inline/*.json, the 12 baselines of
InlineFilterSearch (driver diskann/src/graph/test/cases/inline.rs).  Their payloads do not record the graph, the filter
or the AdaptiveL settings; the driver's are written here per case:
  * "grid_1d": test_provider::Provider::grid(Grid::One, 100), L2; the filter is a set of ids; Setup1D's no_scaling /
    linear / logarithmic / max settings, run without AdaptiveL ("inline_fixed_*") and with it ("inline_adaptive_l_*").
  * "three_level": build_three_level_labeled_provider (start 0, ids 1-14, max_degree 3, L2); the filter accepts the
    final level, ids 7-14.
  * "reaches_matches": build_1d_index from multihop.rs (start 10 at 5.0, ids 0-4, max_degree 4, L2); EvenFilter.
Only the JSON payloads are extracted; no reference source is copied.
"""
import json
import os
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else "."
OUT = os.path.dirname(os.path.abspath(__file__))
SETUPS = {  # Setup1D: filter ids, k, l, AdaptiveL (samples, scale)
    "no_scaling": (list(range(40, 100)), 5, 5, (5, 16.0)),
    "linear": ([43, 44, 92, 95], 5, 5, (10, 16.0)),
    "logarithmic": ([43, 95], 5, 5, (20, 16.0)),
    "max": ([10, 20, 30, 50], 3, 5, (5, 16.0)),
}


def cases():
    out = []
    for setup, (ids, k, l, adaptive) in SETUPS.items():
        for kind in ("fixed", "adaptive_l"):
            name = f"inline_{kind}_{setup}"
            out.append({"case": name, "graph": "grid_1d", "accept": ids, "k": k, "l": l,
                        "adaptive_l": list(adaptive) if kind == "adaptive_l" else None})
    out.append({"case": "inline_search_returns_only_final_level_matches", "graph": "three_level", "accept": list(range(7, 15)),
                "k": 8, "l": 32, "adaptive_l": None})
    out.append({"case": "inline_search_three_level_no_adaptive_l_with_l1_finds_no_matches", "graph": "three_level",
                "accept": list(range(7, 15)), "k": 1, "l": 1, "adaptive_l": None})
    out.append({"case": "inline_search_three_level_adaptive_l_with_l1_finds_matches", "graph": "three_level",
                "accept": list(range(7, 15)), "k": 1, "l": 1, "adaptive_l": [1, 16.0]})
    out.append({"case": "inline_search_reaches_matches_through_non_matching_nodes", "graph": "reaches_matches", "accept": "even",
                "k": 5, "l": 20, "adaptive_l": None})
    for c in out:
        p = json.load(open(f"{REF}/diskann/test/generated/graph/test/cases/inline/{c['case']}.json"))["payload"]
        assert p["k"] == c["k"] and p["l"] == c["l"], c["case"]
        if "results" in p:
            ids, dists = [r[0] for r in p["results"]], [r[1] for r in p["results"]]
        else:
            ids, dists = p["result_ids"], p["result_distances"]
        c.update(query=p["query"], result_count=p["result_count"], result_ids=ids, result_distances=dists,
                 comparisons=p["comparisons"], hops=p["hops"])
    return out


if __name__ == "__main__":
    if not os.path.isdir(REF):
        sys.exit("reference checkout not present; the fixture is already committed")
    out = cases()
    json.dump({"source": "diskann/test/generated/graph/test/cases/inline/*.json (driver diskann/src/graph/test/cases/inline.rs; "
                         "the graph, filter and AdaptiveL of each case are the driver's; Knn::new_default(l), beam width 1)",
               "cases": out}, open(f"{OUT}/inline_search.json", "w"), indent=0)
    print("inline_search.json", len(out))
