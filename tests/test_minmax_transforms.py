"""The Hadamard transforms in front of the MinMax quantizer (diskann-quantization/src/algorithms/hadamard.rs,
transforms/{padding_hadamard.rs, double_hadamard.rs}, minmax/quantizer.rs).

CPU: the oracle's restatement (oracle/transform.cpp) against Sylvester's matrix and the reference's own transform tests
(dimension tables, ErrorSetup tolerances), and the try_from_parts validation of dab_transform_create, which touches no
device.  GPU: dab_transform_apply, the transformed compress and the three query layouts of the reference's
minmax-exhaustive jobs, bit for bit against the oracle.  NaN results compare as NaN: x86 and the GPU give inf - inf
different payloads."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import diskann_b200 as dab
import oracle_lib as O

T = dab.Transform
METRICS = [O.L2, O.INNER_PRODUCT, O.COSINE, O.COSINE_NORMALIZED]


_TLIB = None


def olib():
    """oracle/transform.cpp's entry points: liboracle_transform.so (oracle/transform.mk, built by build())."""
    global _TLIB
    if _TLIB is None:
        path = os.path.join(O.ORACLE_DIR, "liboracle_transform.so")
        src = os.path.join(O.ORACLE_DIR, "transform.cpp")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(src):
            subprocess.check_call(["make", "-C", O.ORACLE_DIR, "-s", "-f", "transform.mk"], stdout=subprocess.DEVNULL)
        L = C.CDLL(path)
        vp, sz, i = C.c_void_p, C.c_size_t, C.c_int
        L.orc_hadamard_8.restype, L.orc_hadamard_8.argtypes = None, [vp]
        L.orc_hadamard.restype, L.orc_hadamard.argtypes = i, [vp, sz, i]
        L.orc_padding_hadamard.restype, L.orc_padding_hadamard.argtypes = i, [vp, sz, sz, vp, sz, vp, vp]
        L.orc_double_hadamard.restype, L.orc_double_hadamard.argtypes = i, [vp, sz, vp, sz, vp, sz, vp, vp]
        L.orc_transform_full_query_meta.restype, L.orc_transform_full_query_meta.argtypes = i, [vp, sz, vp, sz, vp, vp]
        _TLIB = L
    return _TLIB


def sylvester(n):
    h = np.ones((1, 1))
    while h.shape[0] < n:
        h = np.block([[h, h], [h, -h]])
    return h


def hadamard(x, scalar_order=False):
    x = np.array(x, np.float32)
    assert olib().orc_hadamard(O.ptr(x), len(x), int(scalar_order)) == 0
    return x


def oracle_apply(t, vectors):
    """transform_into of the oracle for every row of `vectors`, with the parts held by the Transform `t`."""
    L = olib()
    vectors = np.ascontiguousarray(vectors, np.float32)
    out = np.zeros((vectors.shape[0], t.output_dim), np.float32)
    sub = t.subsample
    n_sub = 0 if sub is None else len(sub)
    for r in range(vectors.shape[0]):
        if t.kind == T.PADDING_HADAMARD:
            rc = L.orc_padding_hadamard(O.ptr(t.signs0), len(t.signs0), t.inner_dim, O.ptr(sub), n_sub, O.ptr(vectors[r]), O.ptr(out[r]))
        else:
            rc = L.orc_double_hadamard(O.ptr(t.signs0), len(t.signs0), O.ptr(t.signs1), t.inner_dim, O.ptr(sub), n_sub, O.ptr(vectors[r]),
                                       O.ptr(out[r]))
        assert rc == 0
    return out


def same_bits(a, b):
    """Bit-identical, every NaN counting as the same value."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32)))


# ---------------------------------------------------------------- CPU: the Hadamard transform of the oracle

def test_hadamard_8_is_sylvester():
    """hadamard.rs test_hadamard_8."""
    h = np.zeros(64, np.float32)
    olib().orc_hadamard_8(O.ptr(h))
    assert np.array_equal(h.reshape(8, 8), sylvester(8).astype(np.float32))


@pytest.mark.parametrize("scalar_order", [False, True])
def test_hadamard_against_float64_sylvester_product(scalar_order):
    """hadamard.rs test_hadamard_transform_*: H x / sqrt(P) for P = 1 .. 4096."""
    rng = np.random.default_rng(7)
    for k in range(13):
        p = 1 << k
        x = rng.standard_normal(p).astype(np.float32)
        want = sylvester(p) @ x.astype(np.float64) / np.sqrt(p)
        got = hadamard(x, scalar_order)
        tol = 2e-7 * max(1, k) * float(np.linalg.norm(x.astype(np.float64)))
        assert np.abs(got - want).max() <= tol, p


def test_hadamard_of_basis_vectors_is_exact():
    """Every output of H e_i is +-1 / sqrt(P), rounded once."""
    for k in range(11):
        p = 1 << k
        h = sylvester(p).astype(np.float32)
        m = np.float32(1.0) / np.sqrt(np.float32(p)) if p > 1 else np.float32(1.0)
        for i in range(p):
            e = np.zeros(p, np.float32)
            e[i] = 1.0
            assert np.array_equal(hadamard(e).view(np.uint32), (h[:, i] * m).astype(np.float32).view(np.uint32)), (p, i)


def test_v3_order_differs_from_the_scalar_order():
    """micro_kernel_64's FMA chains add eight inputs in sequence where the scalar recursion adds pairs: the two round
    differently.  Below 64 both are the same butterflies."""
    rng = np.random.default_rng(0)
    differs = None
    for seed in range(100):
        x = np.random.default_rng(seed).standard_normal(64).astype(np.float32)
        if not np.array_equal(hadamard(x).view(np.uint32), hadamard(x, True).view(np.uint32)):
            differs = seed
            break
    assert differs is not None
    for p in (2, 4, 8, 16, 32):
        x = rng.standard_normal(p).astype(np.float32)
        assert np.array_equal(hadamard(x).view(np.uint32), hadamard(x, True).view(np.uint32))


def test_signed_zeros():
    """The 8-point chains start from +0.0: a 64-block of -0.0 gives +0.0 everywhere.  Plain butterflies (lengths up to
    32) keep output 0 of all -0.0 inputs at -0.0."""
    for p in (64, 128, 1024):
        out = hadamard(np.full(p, -0.0, np.float32))
        assert (out.view(np.uint32) == 0).all(), p
        assert np.signbit(hadamard(np.full(p, -0.0, np.float32), True)[0])  # the scalar order would keep it
    for p in (2, 4, 8, 16, 32):
        out = hadamard(np.full(p, -0.0, np.float32))
        assert np.signbit(out[0]) and not np.signbit(out[1:]).any(), p


def test_subnormals_are_kept():
    x = np.zeros(64, np.float32)
    x[3] = np.float32(1e-42)  # subnormal
    out = hadamard(x)
    assert (out != 0).all() and (np.abs(out) < np.finfo(np.float32).tiny).all()


# ---------------------------------------------------------------- CPU: dimension rules (no device needed)

PADDING_TABLE = [  # padding_hadamard.rs:472-486 (input, output, preserves norms, target)
    (15, 16, True, 16), (15, 16, True, "natural"), (16, 16, True, "same"), (16, 16, True, "natural"), (16, 32, True, 32),
    (16, 64, True, 64), (100, 128, True, 128), (100, 128, True, "natural"), (256, 256, True, 256),
    (1000, 1000, False, "same"), (500, 1000, False, 1000),
    # padding_hadamard.rs:570-574 (the serialization round trip)
    (5, 5, False, "same"), (10, 16, True, "natural"), (16, 16, True, "natural"), (8, 12, False, 12), (15, 10, False, 10),
]
DOUBLE_TABLE = [  # double_hadamard.rs:425-441
    (15, 15, True, "same"), (15, 15, True, "natural"), (16, 16, True, "same"), (16, 16, True, "natural"), (256, 256, True, "same"),
    (1000, 1000, True, "same"), (15, 16, True, 16), (100, 128, True, 128), (15, 32, True, 32), (16, 64, True, 64),
    (1024, 1023, False, 1023), (1000, 999, False, 999),
    # double_hadamard.rs:527-541
    (5, 5, True, "same"), (8, 8, True, "same"), (10, 10, True, "natural"), (16, 16, True, "natural"), (8, 12, True, 12),
    (10, 12, True, 12), (15, 16, True, 16), (16, 16, True, 16), (15, 32, True, 32), (16, 32, True, 32), (15, 10, False, 10),
    (16, 10, False, 10),
]


@pytest.mark.parametrize("kind", ["padding", "double"])
def test_dimension_tables(kind):
    table = PADDING_TABLE if kind == "padding" else DOUBLE_TABLE
    make = T.padding_hadamard if kind == "padding" else T.double_hadamard
    for seed, (inp, out, preserves, target) in enumerate(table):
        t = make(inp, target, seed)
        assert (t.input_dim, t.output_dim, t.preserves_norms) == (inp, out, preserves), (inp, target)
        if t.subsample is not None:
            assert len(t.subsample) == out and (np.diff(t.subsample.astype(np.int64)) > 0).all() and t.subsample[-1] < t.inner_dim
        if kind == "double":
            assert t.inner_dim == max(inp, out) == len(t.signs1)


def within_ulp(got, expected, ulp):
    got, expected = np.float32(got), np.float32(expected)
    for _ in range(ulp + 1):
        if got == expected:
            return True
        got = np.nextafter(got, expected, dtype=np.float32)
    return False


def check(kind, got, expected):
    """test_util.rs Check: ('ulp', n), ('absrel', abs, rel) or None (skip)."""
    if kind is None:
        return True
    if kind[0] == "ulp":
        return within_ulp(got, expected, kind[1])
    d = abs(float(got) - float(expected))
    m = max(abs(float(got)), abs(float(expected)))
    return d <= kind[1] or (m > 0 and d / m <= kind[2])


@pytest.mark.parametrize("kind", ["padding", "double"])
def test_error_setup_tolerances(kind):
    """test_padding_hadamard / test_double_hadamard (transforms/test_utils.rs check_errors): norms, L2 and inner products of
    StandardNormal pairs survive the oracle transform within the reference's bounds.  Norms are the SIMD inner product of
    a vector with itself."""
    if kind == "padding":
        table, make = PADDING_TABLE[:11], T.padding_hadamard
        natural = (("ulp", 4), ("ulp", 4), ("absrel", 5e-6, 2e-4))
        sub = (("absrel", 0.0, 1e-1), ("absrel", 0.0, 1e-1), None)
    else:
        table, make = DOUBLE_TABLE[:12], T.double_hadamard
        natural = (("ulp", 5), ("ulp", 5), ("absrel", 2.5e-5, 2e-4))
        sub = (("absrel", 0.0, 2e-2), ("absrel", 0.0, 2e-2), None)
    rng = np.random.default_rng(0x6D1699AB)
    for combo, (inp, out, preserves, target) in enumerate(table):
        errors = natural if preserves else sub
        for trial in range(3):
            t = make(inp, target, 1000 * combo + trial)
            x = rng.standard_normal((2 * 10, inp)).astype(np.float32)
            y = oracle_apply(t, x)
            for i in range(0, x.shape[0], 2):
                for a, b in ((i, i), (i + 1, i + 1)):
                    assert check(errors[0], -O.distance(y[a], y[b], O.INNER_PRODUCT), -O.distance(x[a], x[b], O.INNER_PRODUCT)), (inp, target, "norm")
                assert check(errors[1], O.distance(y[i], y[i + 1], O.L2), O.distance(x[i], x[i + 1], O.L2)), (inp, target, "l2")
                assert check(errors[2], -O.distance(y[i], y[i + 1], O.INNER_PRODUCT), -O.distance(x[i], x[i + 1], O.INNER_PRODUCT)), (inp, target, "ip")


# ---------------------------------------------------------------- CPU: try_from_parts, rejected before any device work

def rejects(match, *args, **kw):
    with pytest.raises(dab.DabError) as e:
        T(*args, **kw)
    assert e.value.code == 1 and match in str(e.value), str(e.value)


def test_padding_hadamard_parts_are_validated():
    """PaddingHadamard::try_from_parts (padding_hadamard.rs:137-173) and its serialization tests (:599-662)."""
    P = T.PADDING_HADAMARD
    rejects("InvalidSignRepresentation", P, [0, 2, 0], 4)
    rejects("InvalidSignRepresentation", P, [0, 2, 0, 0, 0], 4)  # the reference's order: signs before lengths
    rejects("SignsTooLong", P, [0] * 5, 4)
    rejects("DimNotPowerOfTwo", P, [0] * 5, 5)
    rejects("SubsampleEmpty", P, [0] * 4, 4, subsample=[])
    rejects("SubsampleNotMonotonic", P, [0] * 4, 4, subsample=[0, 2, 2])
    rejects("LastSubsampleTooLarge", P, [0] * 4, 4, subsample=[0, 1, 2, 3, 4])
    rejects("LastSubsampleTooLarge", P, [0] * 4, 4, subsample=[0, 4])
    rejects("65536", P, [0] * 40000, 65536)  # one vector has to fit a warp's shared memory
    t = T(P, [1, 0, 1], 4, subsample=[1, 3])
    assert (t.input_dim, t.output_dim) == (3, 2)


def test_double_hadamard_parts_are_validated():
    """DoubleHadamard::try_from_parts (double_hadamard.rs:146-206), errors in its order."""
    D = T.DOUBLE_HADAMARD
    rejects("Signs0Empty", D, [], 4, signs1=[0] * 4)
    rejects("Signs1TooSmall", D, [0] * 5, 4, signs1=[0] * 4)
    rejects("Signs1TooSmall", D, [3] * 5, 4, signs1=[0] * 4)
    rejects("Signs0Invalid", D, [0, 7], 4, signs1=[0] * 4)
    rejects("Signs1Invalid", D, [0, 1], 4, signs1=[0, 1, 2, 0])
    rejects("SubsampleNotMonotonic", D, [0] * 4, 4, signs1=[0] * 4, subsample=[2, 1])
    rejects("LastSubsampleTooLarge", D, [0] * 4, 4, signs1=[0] * 4, subsample=[0, 4])
    rejects("InvalidSubsampleLength", D, [0] * 4, 4, signs1=[0] * 4, subsample=[])
    rejects("32769", D, [0] * 32769, 32769, signs1=[0] * 32769)
    t = T(D, [1, 0, 1], 5, signs1=[0, 1, 1, 0, 1])
    assert (t.input_dim, t.output_dim) == (3, 5)


def test_entry_points_validate_before_any_device_work():
    L = dab.lib()
    assert L.dab_transform_create(None, 1, 4, 4, None, None, None, 0) == 1
    h = C.c_void_p()
    assert L.dab_transform_create(C.byref(h), 3, 4, 4, None, None, None, 0) == 1 and b"kind" in L.dab_last_error()
    assert L.dab_transform_apply(None, 0, None, 1, None) == 1
    assert L.dab_minmax_compress_transformed(None, 0, 1.0, 4, None, 1, None, None) == 1
    t = T.padding_hadamard(100, "same")
    assert L.dab_minmax_compress_transformed(t._h, 0, 1.0, 3, None, 1, None, None) == 1
    assert L.dab_minmax_query_distances_transformed(t._h, 0, 9, 4, None, 1, None, 1, None) == 1
    assert L.dab_transform_output_dim(None) == 0
    L.dab_transform_destroy(None)  # no-op


# ---------------------------------------------------------------- GPU: bit for bit against the oracle

DIMS = [1, 2, 3, 7, 8, 15, 16, 31, 32, 63, 64, 65, 100, 127, 128, 129, 384, 768, 1000, 1024, 4096]


def awkward_rows(dim, rng, n=5):
    """Normal rows, then rows of signed zeros, subnormals, infinities and wide magnitudes."""
    x = rng.standard_normal((n, dim)).astype(np.float32)
    pick = lambda vals, size: np.array(vals, np.float32)[rng.integers(0, len(vals), size)]  # noqa: E731
    x[1] = pick([0.0, -0.0, 1e-40, -3e-39, 1e-45, 1.0], dim)
    x[2] = -0.0
    if n > 3:
        x[3] = pick([np.inf, -np.inf, 1.0, -2.0, 0.0], dim)
    if n > 4:
        x[4] = x[4] * np.float32(10.0) ** rng.integers(-30, 30, dim).astype(np.float32)
    return x


def targets_of(dim):
    return ["same", "natural", max(1, dim // 2), dim * 2 + 3]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["padding", "double"])
def test_apply_is_bit_identical_to_the_oracle(kind):
    make = T.padding_hadamard if kind == "padding" else T.double_hadamard
    rng = np.random.default_rng(11)
    for dim in DIMS:
        for ti, target in enumerate(targets_of(dim)):
            t = make(dim, target, dim * 10 + ti)
            x = awkward_rows(dim, rng)
            assert same_bits(t.apply(x), oracle_apply(t, x)), (kind, dim, target)


@pytest.mark.gpu
def test_apply_at_the_size_limit():
    rng = np.random.default_rng(12)
    for t in (T.padding_hadamard(32768, "same", 1), T.padding_hadamard(20000, "natural", 2), T.padding_hadamard(20000, 30000, 3),
              T.double_hadamard(32768, "same", 4), T.double_hadamard(30000, 32768, 5), T.double_hadamard(32768, 1000, 6)):
        x = awkward_rows(t.input_dim, rng, 3)
        assert same_bits(t.apply(x), oracle_apply(t, x)), (t.kind, t.input_dim, t.output_dim)
    with pytest.raises(dab.DabError, match="32769"):
        T.double_hadamard(32769, "same")
    with pytest.raises(dab.DabError, match="65536"):
        T.padding_hadamard(32769, "same")


# the reference job shapes (minmax-exhaustive.json) at 128 dimensions, plus DoubleHadamard
JOB_SHAPES = [("padding", "same"), ("padding", "natural"), ("padding", 100), ("double", "same"), ("double", 100), ("double", 160)]


def job_transform(kind, target, dim=128, seed=5):
    return (T.padding_hadamard if kind == "padding" else T.double_hadamard)(dim, target, seed)


@pytest.mark.gpu
@pytest.mark.parametrize("nbits", [1, 2, 4, 8])
def test_compress_is_bit_identical_to_the_oracle(nbits):
    rng = np.random.default_rng(20 + nbits)
    x = rng.standard_normal((70, 128)).astype(np.float32)
    for kind, target in JOB_SHAPES:
        t = job_transform(kind, target)
        tx = oracle_apply(t, x)
        for scale in (0.9, 1.0, 1.1):
            rows, loss = dab.minmax_compress(x, nbits, scale, transform=t)
            want_rows, want_loss, nan = O.minmax_compress(tx, nbits, scale)
            assert not nan.any()
            assert rows.shape == want_rows.shape and int(rows[0, :4].view(np.uint32)[0]) == t.output_dim
            assert np.array_equal(rows, want_rows), (kind, target, nbits, scale)
            assert np.array_equal(loss.view(np.uint32), want_loss.view(np.uint32)), (kind, target, nbits, scale)


@pytest.mark.gpu
def test_compress_nan_names_the_first_row():
    t = job_transform("padding", "natural")
    x = np.random.default_rng(3).standard_normal((40, 128)).astype(np.float32)
    x[17, 5] = np.nan
    x[30, 0] = np.nan
    with pytest.raises(dab.DabError, match="vector 17 contains NaN"):
        dab.minmax_compress(x, 4, transform=t)


@pytest.mark.gpu
def test_two_infinities_fail_compress_but_not_the_full_query():
    """quantizer.rs:192-221 checks the transformed vector, :398-401 the input: +inf and -inf in one vector transform to
    NaN, which compress reports and the full-precision query does not."""
    t = job_transform("padding", "same")
    x = np.random.default_rng(4).standard_normal((8, 128)).astype(np.float32)
    x[6, 3], x[6, 9] = np.inf, -np.inf
    assert np.isnan(oracle_apply(t, x[6:7])).any()
    with pytest.raises(dab.DabError, match="vector 6 contains NaN"):
        dab.minmax_compress(x, 8, transform=t)
    rows, _ = dab.minmax_compress(x[:6], 8, transform=t)
    got = dab.minmax_query_distances(dab.Metric.L2, 8, x[6:7], rows, transform=t)
    assert same_bits(got, oracle_full_query(t, O.L2, 8, x[6:7], rows))
    x[6, 9] = np.nan
    with pytest.raises(dab.DabError, match="query 0 contains NaN"):
        dab.minmax_query_distances(dab.Metric.L2, 8, x[6:7], rows, transform=t)


def oracle_full_query(t, metric, nbits, queries, rows):
    L = olib()
    tq = oracle_apply(t, queries)
    out = np.zeros((len(queries), len(rows)), np.float32)
    for qi in range(len(queries)):
        s, ns = np.zeros(1, np.float32), np.zeros(1, np.float32)
        assert L.orc_transform_full_query_meta(O.ptr(queries[qi]), queries.shape[1], O.ptr(tq[qi]), tq.shape[1], O.ptr(s), O.ptr(ns)) == 0
        for r in range(len(rows)):
            out[qi, r] = O.lib().orc_minmax_query_distance(metric, nbits, O.ptr(tq[qi]), float(s[0]), float(ns[0]), O.ptr(rows[r]))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("nbits", [1, 2, 4, 8])
def test_query_layouts_are_bit_identical_to_the_oracle(nbits):
    """The three query layouts of minmax-exhaustive.json: full_precision (the transformed f32 query against the rows),
    same_as_data (queries compressed at the data's width, N x N) and eight_bit (queries compressed at 8 bits, 8 x N)."""
    rng = np.random.default_rng(40 + nbits)
    data = rng.standard_normal((48, 128)).astype(np.float32)
    queries = rng.standard_normal((6, 128)).astype(np.float32)
    for kind, target in JOB_SHAPES:
        t = job_transform(kind, target)
        rows, _ = dab.minmax_compress(data, nbits, 1.0, transform=t)
        qi, ri = np.repeat(np.arange(len(queries)), len(rows)), np.tile(np.arange(len(rows)), len(queries))
        for m in METRICS:
            got = dab.minmax_query_distances(dab.Metric(m), nbits, queries, rows, transform=t)
            assert same_bits(got, oracle_full_query(t, m, nbits, queries, rows)), (kind, target, nbits, m, "full_precision")
            for qbits in (nbits, 8):
                qrows, _ = dab.minmax_compress(queries, qbits, 1.0, transform=t)
                got = dab.minmax_distances(dab.Metric(m), qbits, nbits, t.output_dim, qrows[qi], rows[ri])
                want = O.minmax_distances(m, qbits, nbits, qrows[qi], rows[ri])
                assert same_bits(got, want), (kind, target, nbits, m, qbits)
