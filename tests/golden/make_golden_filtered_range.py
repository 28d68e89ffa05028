#!/usr/bin/env python3
"""Extracts the reference's filtered range-search baselines into tests/golden/filtered_range_search.json.

Run against a checkout of the reference (the tests only read the JSON file this writes):
    python tests/golden/make_golden_filtered_range.py <path to the reference checkout>

Source (relative to the reference checkout):
  * diskann/test/generated/graph/test/cases/filtered_range_search/*.json — one filtered range search over the 5^3
    lattice, query (5, 5, 5) (driver diskann/src/graph/test/cases/filtered_range_search.rs).  The two max_results cases
    run with max_returned 4 and 200, and the filter of each case is the driver's AlwaysTrueFilter or
    DivisibleByFourFilter; the payloads record neither, so both are written here.
Only the JSON payloads are extracted; no reference source is copied.
"""
import json
import os
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else "."
OUT = os.path.dirname(os.path.abspath(__file__))
# case: (max_returned, filter)
CASES = {"basic_range_search": (None, "always_true"), "inner_radius_filtering": (None, "always_true"),
         "two_round_search": (None, "always_true"), "max_results_respected_means_no_second_round": (4, "always_true"),
         "max_results_respected_and_second_round_triggered": (200, "always_true"),
         "divisible_by_four_filter_second_round_triggered": (None, "divisible_by_four"),
         "divisible_by_four_filter_no_second_round_from_l_search": (None, "divisible_by_four")}


def filtered_range_search():
    out = []
    for name, (max_returned, flt) in CASES.items():
        p = json.load(open(f"{REF}/diskann/test/generated/graph/test/cases/filtered_range_search/{name}.json"))["payload"]
        out.append({"case": name, "filter": flt, "grid_dims": p["grid_dims"], "grid_size": p["grid_size"], "query": p["query"],
                    "starting_l": p["starting_l"], "radius": p["radius"], "inner_radius": p["inner_radius"],
                    "max_returned": max_returned, "results": p["results"], "result_count": p["result_count"],
                    "comparisons": p["comparisons"], "hops": p["hops"],
                    "range_search_second_round": p["range_search_second_round"]})
    json.dump({"source": "diskann/test/generated/graph/test/cases/filtered_range_search/*.json (driver "
                         "diskann/src/graph/test/cases/filtered_range_search.rs: test_provider::Provider::grid, L2, start "
                         "point at (size,..,size) linked to the last node; FilteredRange with beam_width 1, initial_slack 1, "
                         "range_slack 1, the case's inner_radius and max_returned, over labeled::Filtered with the case's "
                         "filter: always_true accepts every id, divisible_by_four the ids id % 4 == 0, the start point "
                         "included; results as (id, distance) in output order)",
               "cases": out}, open(f"{OUT}/filtered_range_search.json", "w"), indent=0)
    print("filtered_range_search.json", len(out))


if __name__ == "__main__":
    if not os.path.isdir(REF):
        sys.exit("reference checkout not present; the fixture is already committed")
    filtered_range_search()
