#!/usr/bin/env python3
"""Extracts the reference's range-search baselines into tests/golden/range_search.json.

Run against a checkout of the reference (the tests only read the JSON file this writes):
    python tests/golden/make_golden_range.py <path to the reference checkout>

Source (relative to the reference checkout):
  * diskann/test/generated/graph/test/cases/range_search/{basic_range_search,inner_radius_filtering,two_round_search,
    max_results_respected_means_no_second_round,max_results_respected_and_second_round_triggered}.json — one range
    search over the 5^3 lattice, query (5, 5, 5) (driver diskann/src/graph/test/cases/range_search.rs).  The two
    max_results cases run with max_returned 4 and 5, which their payloads do not record: they are written here.
Only the JSON payloads are extracted; no reference source is copied.
"""
import json
import os
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else "."
OUT = os.path.dirname(os.path.abspath(__file__))
CASES = {"basic_range_search": None, "inner_radius_filtering": None, "two_round_search": None,
         "max_results_respected_means_no_second_round": 4, "max_results_respected_and_second_round_triggered": 5}


def range_search():
    out = []
    for name, max_returned in CASES.items():
        p = json.load(open(f"{REF}/diskann/test/generated/graph/test/cases/range_search/{name}.json"))["payload"]
        out.append({"case": name, "grid_dims": p["grid_dims"], "grid_size": p["grid_size"], "query": p["query"],
                    "starting_l": p["starting_l"], "radius": p["radius"], "inner_radius": p["inner_radius"],
                    "max_returned": max_returned, "results": p["results"], "result_count": p["result_count"],
                    "comparisons": p["comparisons"], "hops": p["hops"],
                    "range_search_second_round": p["range_search_second_round"]})
    json.dump({"source": "diskann/test/generated/graph/test/cases/range_search/*.json (driver "
                         "diskann/src/graph/test/cases/range_search.rs: test_provider::Provider::grid, L2, start point at "
                         "(size,..,size) linked to the last node; Range::builder(starting_l, radius) with beam_width 1, "
                         "initial_slack 1, range_slack 1, the case's inner_radius and max_returned; results as (id, distance) "
                         "in output order)",
               "cases": out}, open(f"{OUT}/range_search.json", "w"), indent=0)
    print("range_search.json", len(out))


if __name__ == "__main__":
    if not os.path.isdir(REF):
        sys.exit("reference checkout not present; the fixture is already committed")
    range_search()
