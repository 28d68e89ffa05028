#!/usr/bin/env python3
"""Extracts the reference's paged-search baselines into tests/golden/paged_search.json.

Run against a checkout of the reference (the tests only read the JSON file this writes):
    python tests/golden/make_golden_paged.py <path to the reference checkout>

Source (relative to the reference checkout):
  * diskann/test/generated/graph/test/cases/paged_search/{basic_paged_search,single_page,small_page_size}.json —
    every page of one paged search over the 5^3 lattice, query (5, 5, 5) (driver
    diskann/src/graph/test/cases/paged_search.rs).
Only the JSON payloads are extracted; no reference source is copied.
"""
import json
import os
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else "."
OUT = os.path.dirname(os.path.abspath(__file__))


def paged_search():
    out = []
    for name in ("basic_paged_search", "single_page", "small_page_size"):
        p = json.load(open(f"{REF}/diskann/test/generated/graph/test/cases/paged_search/{name}.json"))["payload"]
        out.append({"case": name, "grid_dims": p["dims"], "grid_size": p["grid_size"], "query": p["query"], "search_l": p["search_l"],
                    "page_size": p["page_size"], "pages": p["pages"], "total_results": p["total_results"]})
    json.dump({"source": "diskann/test/generated/graph/test/cases/paged_search/*.json (driver "
                         "diskann/src/graph/test/cases/paged_search.rs: test_provider::Provider::grid, L2, start point at "
                         "(size,..,size) linked to the last node; DiskANNIndex::paged_search(query, search_l), then next_page(page_size) "
                         "until a page is empty (single_page: one page); every page as (id, distance))",
               "cases": out}, open(f"{OUT}/paged_search.json", "w"), indent=0)
    print("paged_search.json", len(out))


if __name__ == "__main__":
    if not os.path.isdir(REF):
        sys.exit("reference checkout not present; the fixture is already committed")
    paged_search()
