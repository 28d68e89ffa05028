"""The distance schemas compiled into the library follow the reference's rule (DESIGN §4): Metric::Cosine over float
operands and f16 x f16 operands run the two-accumulator schema (NA = 2, Strategy2x4), every other float schema NA = 4;
integer CosineNormalized is Cosine, so no integer kernel is built for (InnerProduct, 1 - v).  Kernels of any other
schema could never be launched.  Reads the objects build() leaves in diskann_b200/csrc (cuobjdump, cu++filt)."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "diskann_b200", "csrc")
OBJECTS = ("distance_kernels", "build_kernels", "flat_kernels", "search_kernel_pq", "search_kernel_v2", "search_kernel_v3")
KIND_IP, KIND_COS = 1, 2
POST_ONE_MINUS = 2
FLOAT = ("float", "__half")
INT = ("signed char", "unsigned char")

# family -> (query operand, row operand, NA, KIND, POST) from its template arguments; the query operand of the flat
# scan and the frontier gather is the f32-widened query
FLOAT_FAMILIES = {
    "pair_float_kernel": lambda a: (a[0], a[1], a[2], a[3], a[4]),
    "rowpair_float_kernel": lambda a: (a[0], a[0], a[1], a[2], a[3]),
    "frontier_float_kernel": lambda a: (a[0], a[2], a[3], a[4], a[5]),
    "prune_pools_kernel": lambda a: (a[0], a[0], a[1], a[2], a[3]),
    "backedge_kernel": lambda a: (a[0], a[0], a[1], a[2], a[3]),
    "flat_generic_kernel": lambda a: ("float", a[0], a[1], a[2], a[3]),
    "rerank_kernel": lambda a: (a[0], a[0], a[3], a[1], a[2]),
}
# family -> (is an integer instantiation, KIND, POST)
INT_FAMILIES = {
    "pair_int_kernel": lambda a: (True, a[1], a[2]),
    "rowpair_int_kernel": lambda a: (True, a[1], a[2]),
    "frontier_int_kernel": lambda a: (True, a[1], a[2]),
    "frontier_int_wide_kernel": lambda a: (True, a[1], a[2]),
    "prune_pools_kernel": lambda a: (a[4] == 1, a[2], a[3]),
    "backedge_kernel": lambda a: (a[4] == 1, a[2], a[3]),
    "flat_generic_kernel": lambda a: (a[4] == 1, a[2], a[3]),
    "rerank_kernel": lambda a: (a[0] in INT, a[1], a[2]),
    "search_kernel_v2": lambda a: (a[0] in INT, a[1], a[2]),
    "search_kernel_v3": lambda a: (a[0] in INT, a[1], a[2]),
}


def expected_na(tq, td, kind):
    return 2 if kind == KIND_COS or (tq, td) == ("__half", "__half") else 4


def template_args(demangled):
    """'void dab::name<float, (int)2, (bool)1>(...)' -> ('name', ['float', 2, 1])"""
    m = re.match(r"void dab::(\w+)<([^<>]*)>\(", demangled)
    if not m:
        return None, None
    args = []
    for a in m.group(2).split(", "):
        c = re.fullmatch(r"\((?:int|bool)\)(\d+)", a)
        args.append(int(c.group(1)) if c else a)
    return m.group(1), args


@pytest.fixture(scope="module")
def kernels():
    out = []
    for name in OBJECTS:
        sass = subprocess.run(["cuobjdump", "-sass", os.path.join(CSRC, name + ".o")], capture_output=True, text=True,
                              check=True).stdout
        mangled = re.findall(r"Function : (\S+)", sass)
        demangled = subprocess.run(["cu++filt"], input="\n".join(mangled) + "\n", capture_output=True, text=True,
                                   check=True).stdout.splitlines()
        out += [template_args(d) for d in demangled]
    return [(f, a) for f, a in out if f]


def test_float_kernels_have_the_rule_s_accumulator_count(kernels):
    seen = set()
    for family, args in kernels:
        if family in FLOAT_FAMILIES:
            tq, td, na, kind, post = FLOAT_FAMILIES[family](args)
            if td in FLOAT:
                seen.add(family)
                assert na == expected_na(tq, td, kind), f"{family}<{args}>: {tq} x {td}, kind {kind}"
    assert seen == set(FLOAT_FAMILIES)


def test_no_integer_kernel_for_inner_product_one_minus(kernels):
    seen = set()
    for family, args in kernels:
        if family in INT_FAMILIES:
            is_int, kind, post = INT_FAMILIES[family](args)
            if is_int:
                seen.add(family)
                assert (kind, post) != (KIND_IP, POST_ONE_MINUS), f"{family}<{args}>"
    assert seen == set(INT_FAMILIES)


def test_frontier_float_kernel_only_for_cosine(kernels):
    kinds = [FLOAT_FAMILIES["frontier_float_kernel"](a)[3] for f, a in kernels if f == "frontier_float_kernel"]
    assert kinds and set(kinds) == {KIND_COS}


def test_search_kernel_v3_only_for_one_merge_tile(kernels):
    """v3_prepare takes lists of L + #start <= 24 only: every search_kernel_v3<T, kind, post, QT, FAST> merges its list in
    one register tile (QT = 4, up to 128 entries); a kernel with a longer tile could never be launched."""
    tiles = [a[3] for f, a in kernels if f == "search_kernel_v3"]
    assert tiles and set(tiles) == {4}
