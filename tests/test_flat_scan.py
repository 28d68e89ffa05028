"""The two exhaustive scans that every recall figure is measured against, at the shapes and values where they go wrong.

* dab_flat_knn: flat_float_kernel / flat_generic_kernel, then flat_topk_kernel, which carries each query's top-k across
  row blocks.
* dab_flat_knn_tc: the wgmma GEMM over bf16 hi / lo splits with per-range candidate selection, exact re-scoring, and a
  per-query certificate; the queries it cannot certify are re-run through the exact scan.

Every device result is checked two ways: bit for bit against the oracle's brute force, and against a float64 numpy
brute force.  The second check catches a mistake the oracle and the kernels share, such as a wrong metric convention.
The CPU tests check the oracle's NaN rule and the error bound the tensor-core certificate relies on."""
import numpy as np
import pytest

import oracle_lib as O

METRICS = [O.L2, O.INNER_PRODUCT, O.COSINE, O.COSINE_NORMALIZED]
DTYPES = [np.float32, np.float16, np.int8, np.uint8]
FLT_MIN = float(np.finfo(np.float32).tiny)
NO_ID = 0xFFFFFFFF
FALLBACK_KERNELS = ("flat_float_kernel", "flat_generic_kernel", "flat_topk_kernel")


@pytest.fixture(scope="module")
def dab():
    import diskann_b200
    diskann_b200.lib()
    return diskann_b200


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same_bits(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.array_equal(bits(a)[~(np.isnan(a) & np.isnan(b))], bits(b)[~(np.isnan(a) & np.isnan(b))]) and \
        np.array_equal(np.isnan(a), np.isnan(b))


def fuzz(rng, dt, shape):
    if dt in (np.float32, np.float16):
        return rng.normal(0.0, 1.0, shape).astype(dt)
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max + 1, shape).astype(dt)


def clustered(rng, n, d, centers):
    return (centers[rng.integers(0, len(centers), n)] + 0.3 * rng.normal(size=(n, d))).astype(np.float32)


def row_block(n, nq):
    """dab_flat_knn's row block: the distance tile of nq x rb floats stays around 1 GiB."""
    rb = min(n, max(1024, (1 << 28) // nq))
    return (rb + 31) & ~31


def index(dab, base, metric):
    """An index over `base` (one extra start row, which is not data)."""
    n, dim = base.shape
    g = dab.GpuIndex(O.dtype_code(base), metric, dim, n, 1, 4)
    g.upload_vectors(np.concatenate([base, base[:1]]))
    return g


# ---------------------------------------------------------------- float64 reference

def f64_distances(base, q, metric):
    """float64 distances of one query to every row, with the reference's conventions: squared L2; -q.b; Cosine
    1 - clamp(q.b / (|q| |b|), -1, 1), where a squared norm below FLT_MIN gives cos = 0 and NaN clamps to 1 (Rust's
    f32::min / max return the non-NaN operand); CosineNormalized 1 - q.b for floats and Cosine for integers.  Also
    returns the scale of the fp32 rounding error of each distance."""
    b, q = base.astype(np.float64), q.astype(np.float64)
    is_int = base.dtype in (np.int8, np.uint8)
    with np.errstate(all="ignore"):
        if metric == O.L2:
            d = ((q - b) ** 2).sum(1)
            return d, d
        xy = (q * b).sum(1)
        if metric == O.INNER_PRODUCT:
            return -xy, np.abs(q * b).sum(1)
        if metric == O.COSINE_NORMALIZED and not is_int:
            return 1.0 - xy, np.abs(q * b).sum(1) + 1.0
        nq2, nb2 = (q * q).sum(), (b * b).sum(1)
        v = np.fmax(-1.0, np.fmin(1.0, xy / (np.sqrt(nq2) * np.sqrt(nb2))))
        v = np.where((nq2 < FLT_MIN) | (nb2 < FLT_MIN), 0.0, v)
        return 1.0 - v, np.full(len(b), 2.0)


def check_f64(base, queries, metric, k, ids, dists, which=None):
    """Where the float64 gap between the k-th and (k+1)-th distance exceeds 1e-4 relative, the id sets agree; every
    returned distance is within 1e-5 relative plus a dim-scaled fp32 term of its float64 value; NaN never returns."""
    dim = base.shape[1]
    which = range(len(queries)) if which is None else which
    for row, i in enumerate(which):
        d, scale = f64_distances(base, queries[i], metric)
        valid = ~np.isnan(d)
        vals = np.sort(d[valid])
        m = min(k, len(vals))
        assert np.all(ids[row, m:] == NO_ID) and np.all(np.isposinf(dists[row, m:])), i
        got = ids[row, :m].astype(np.int64)
        assert np.all(got < len(base)) and len(set(got)) == m, i
        ref, got_d = d[got], dists[row, :m].astype(np.float64)
        assert not np.isnan(ref).any(), i
        fin = np.isfinite(ref)
        assert np.array_equal(got_d[~fin], ref[~fin]), i
        tol = 1e-5 * np.abs(ref[fin]) + dim * 2.0 ** -22 * scale[got][fin]
        assert np.all(np.abs(got_d[fin] - ref[fin]) <= tol), (i, np.max(np.abs(got_d[fin] - ref[fin]) - tol))
        if m < len(vals):
            lo, hi = vals[m - 1], vals[m]
            if np.isfinite(lo) and np.isfinite(hi) and hi - lo > 1e-4 * max(abs(lo), abs(hi)):
                assert set(got) == set(np.flatnonzero(valid & (d <= lo))), i
        else:
            assert set(got) == set(np.flatnonzero(valid)), i


def check_exact(base, queries, metric, k, ids, dists, which=None):
    """Both checks of one dab_flat_knn result (rows of `which`, default all, of the query batch)."""
    sub = queries if which is None else queries[which]
    want_ids, want_d = O.bruteforce_knn(base, sub, metric, k)
    assert np.array_equal(ids, want_ids), int((ids != want_ids).any(1).sum())
    assert same_bits(dists, want_d)
    check_f64(base, queries, metric, k, ids, dists, which)


# ---------------------------------------------------------------- dab_flat_knn

@pytest.mark.gpu
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("dt", DTYPES)
def test_exact_scan_every_k(dab, dt, metric):
    """k from 1 to the 2048 limit, exact duplicate rows (lower id first), and k > n (padded with UINT32_MAX / +inf)."""
    rng = np.random.default_rng(7 + 3 * DTYPES.index(dt) + metric)
    base = fuzz(rng, dt, (3000, 24))
    base[1500] = base[900]
    queries = fuzz(rng, dt, (64, 24))
    queries[0] = base[900]
    with index(dab, base, metric) as g:
        results = {k: g.flat_knn(queries, k) for k in (1, 24, 100, 2048)}
    for k, (ids, dists) in results.items():
        check_exact(base, queries, metric, k, ids, dists)
    small = base[:700]
    with index(dab, small, metric) as g:
        ids, dists = g.flat_knn(queries, 1000)
    check_exact(small, queries, metric, 1000, ids, dists)


@pytest.mark.gpu
@pytest.mark.timeout(300)
@pytest.mark.parametrize("dt,metric,k", [
    (np.float32, O.L2, 24), (np.float16, O.INNER_PRODUCT, 24), (np.float32, O.COSINE, 24), (np.uint8, O.L2, 24),
    (np.int8, O.COSINE_NORMALIZED, 24), (np.float16, O.COSINE_NORMALIZED, 100), (np.float32, O.L2, 2048),
])
def test_exact_scan_across_row_blocks(dab, dt, metric, k):
    """nq x n > 2^28: three row blocks, the top-k carried between them through top_n.  Duplicates of a query sit at
    ids rb - 1 and rb, on both sides of the first block boundary.  k = 2048 fills 128 KB of flat_topk_kernel's shared
    memory per block."""
    nq, n, dim = 16384, 40000, 16
    rb = row_block(n, nq)
    assert -(-n // rb) == 3
    rng = np.random.default_rng(k + dim)
    base = fuzz(rng, dt, (n, dim))
    queries = fuzz(rng, dt, (nq, dim))
    probes = [5, nq - 1]
    if metric == O.INNER_PRODUCT:
        base[rb - 1] = base[rb] = queries[5].astype(np.float32) * 8  # the largest inner product
    else:
        base[rb - 1] = base[rb] = queries[5]
    base[2 * rb] = base[2 * rb + 7] = queries[nq - 1]
    with index(dab, base, metric) as g:
        ids, dists = g.flat_knn(queries, k)
    assert list(ids[5, :2]) == [rb - 1, rb]
    if metric != O.INNER_PRODUCT:
        assert list(ids[nq - 1, :2]) == [2 * rb, 2 * rb + 7]
    which = np.unique(np.concatenate([np.arange(128), rng.choice(nq, 256, replace=False), np.arange(nq - 128, nq), probes]))
    check_exact(base, queries, metric, k, ids[which], dists[which], which)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("dt,dim", [(np.float32, 800), (np.float32, 1000), (np.float16, 1000)])
def test_exact_scan_wide_float_rows(dab, dt, dim, metric):
    """The float kernel holds 64 queries in shared memory while 64 x dim x 4 B <= 200 KB (dim 800); wider rows take the
    generic kernel."""
    rng = np.random.default_rng(dim + metric)
    base = fuzz(rng, dt, (3000, dim))
    queries = fuzz(rng, dt, (64, dim))
    with index(dab, base, metric) as g:
        ids, dists = g.flat_knn(queries, 100)
    check_exact(base, queries, metric, 100, ids, dists)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("dt", DTYPES)
def test_exact_scan_non_finite_and_zero_rows(dab, dt, metric):
    """NaN rows and rows with one NaN element are never returned (under Cosine their clamped cosine is 1, distance 0,
    as in the reference); +-inf rows; zero rows and a zero query (cosine 0 below FLT_MIN)."""
    rng = np.random.default_rng(11 + 4 * DTYPES.index(dt) + metric)
    n, dim = 2000, 32
    base = fuzz(rng, dt, (n, dim))
    queries = fuzz(rng, dt, (40, dim))
    base[[3, 500, 1999]] = 0
    queries[1] = 0
    if dt in (np.float32, np.float16):
        base[[10, 11, 700, 1024, 1998]] = np.nan
        for r in (12, 301, 1500, 1501, 1997):
            base[r, rng.integers(dim)] = np.nan
        for r, v in ((40, np.inf), (41, -np.inf), (900, np.inf), (901, -np.inf)):
            base[r, rng.integers(dim)] = v
        base[[1200, 1201]] = np.inf
        queries[2] = base[12]
    with index(dab, base, metric) as g:
        results = {k: g.flat_knn(queries, k) for k in (10, 100)}
    for k, (ids, dists) in results.items():
        check_exact(base, queries, metric, k, ids, dists)
        if metric != O.COSINE:
            assert not np.isnan(dists).any()


# ---------------------------------------------------------------- dab_flat_knn_tc: well-conditioned data

def tc_data(rng, dt, metric, n, d, nq):
    if dt in (np.float32, np.float16):
        centers = rng.normal(size=(50, d)).astype(np.float32)
        base, queries = clustered(rng, n, d, centers), clustered(rng, nq, d, centers)
        if metric == O.COSINE_NORMALIZED:
            base /= np.linalg.norm(base, axis=1, keepdims=True)
            queries /= np.linalg.norm(queries, axis=1, keepdims=True)
        return base.astype(dt), queries.astype(dt)
    return fuzz(rng, dt, (n, d)), fuzz(rng, dt, (nq, d))


@pytest.mark.gpu
@pytest.mark.timeout(180)
@pytest.mark.parametrize("dt,metric,n,d,nq", [
    (np.float32, O.L2, 100, 64, 129), (np.float32, O.INNER_PRODUCT, 20, 16, 5), (np.float16, O.INNER_PRODUCT, 1279, 33, 128),
    (np.int8, O.L2, 1281, 100, 127), (np.uint8, O.COSINE, 2000, 40, 1), (np.float32, O.COSINE_NORMALIZED, 3001, 100, 128),
    (np.float32, O.COSINE, 5000, 128, 2000), (np.float16, O.L2, 20000, 96, 4000), (np.int8, O.COSINE_NORMALIZED, 4000, 64, 1000),
])
def test_tensor_core_scan_equals_the_exact_scan(dab, dt, metric, n, d, nq):
    """Both instantiations (k <= 10 keeps 16 candidates per range, k <= 24 keeps 32), n below one tile and one off a
    tile multiple, 3 dim not a multiple of 64, one to a few thousand queries (fewer than 48 ranges), k > n."""
    rng = np.random.default_rng(n + d + nq)
    base, queries = tc_data(rng, dt, metric, n, d, nq)
    with index(dab, base, metric) as g:
        for k in (1, 10, 11, 24):
            want_ids, want_d = g.flat_knn(queries, k)
            got_ids, got_d = g.flat_knn_tc(queries, k)
            assert np.array_equal(bits(got_d), bits(want_d)), k
            assert np.array_equal(got_ids, want_ids), (k, int((got_ids != want_ids).any(1).sum()))
    if nq <= 200:
        check_exact(base, queries, metric, 24, got_ids, got_d)


@pytest.mark.gpu
def test_tensor_core_scan_refuses_k_outside_1_to_24(dab):
    rng = np.random.default_rng(3)
    base = fuzz(rng, np.float32, (500, 32))
    with index(dab, base, O.L2) as g:
        for k in (0, 25):
            with pytest.raises(Exception, match="k must be in"):
                g.flat_knn_tc(base[:4], k)


# ---------------------------------------------------------------- dab_flat_knn_tc: ill-conditioned data

def plant_near_duplicates(rng, base, queries, scale, ulps):
    """For each of the first 8 queries: 40 copies (times `scale`) inside one 128-row tile, more than the 32 candidates a
    range keeps, plus 4 in other ranges, each with 1 to `ulps` random elements moved by one ulp."""
    rows = np.concatenate([np.arange(1280, 1320), [77, 9000, 9001, 19990]])
    for j, q in enumerate(queries[:8]):
        for r in rows + j * 128 * 8:
            v = (q.astype(np.float32) * scale).astype(base.dtype)
            e = rng.choice(base.shape[1], rng.integers(1, ulps + 1), replace=False)
            if base.dtype == np.uint8:
                v[e] -= 1
            else:
                v[e] = np.nextafter(v[e], np.where(rng.random(len(e)) < 0.5, np.inf, -np.inf).astype(base.dtype))
            base[r % len(base)] = v


def ill_conditioned(case, rng):
    if case == "f32_l2_offset":  # ||b||^2 ~ 1.28e6: the fp32 score's ulp is 0.125, neighbours differ by ~0.03
        base = (100 + 0.01 * rng.normal(size=(20000, 128))).astype(np.float32)
        return base, (100 + 0.01 * rng.normal(size=(300, 128))).astype(np.float32), O.L2, (10, 24)
    if case == "f32_l2_near_duplicates":  # 1-ulp copies of a query
        centers = rng.normal(size=(50, 64)).astype(np.float32)
        base, queries = clustered(rng, 20000, 64, centers), clustered(rng, 64, 64, centers)
        plant_near_duplicates(rng, base, queries, 1.0, 3)
        return base, queries, O.L2, (10, 24)
    if case == "f16_ip_norm_spread":  # row norms over 10^-3 .. 10^3, and copies of queries at norm ~10^3
        dirs = rng.normal(size=(20000, 64))
        base = (dirs / np.linalg.norm(dirs, axis=1, keepdims=True) * 10 ** rng.uniform(-3, 3, (20000, 1))).astype(np.float16)
        queries = rng.normal(size=(200, 64)).astype(np.float16)
        plant_near_duplicates(rng, base, queries, 125.0, 3)
        return base, queries, O.INNER_PRODUCT, (10, 24)
    if case == "u8_l2_dim768_high":  # sums of products past 2^24 are no longer exact in fp32: the score's ulp is 4
        base = rng.integers(240, 256, (20000, 768)).astype(np.uint8)
        queries = rng.integers(240, 256, (100, 768)).astype(np.uint8)
        plant_near_duplicates(rng, base, queries, 1.0, 3)
        return base, queries, O.L2, (10, 24)
    assert case == "f32_cosine_underflow"  # rows whose ||b||^2 underflows: exact distance 1, nearer than every other row
    center = rng.normal(size=(1, 64)).astype(np.float32)
    base = -clustered(rng, 5000, 64, center)
    base[rng.choice(5000, 300, replace=False)] *= np.float32(1e-21)
    return base, clustered(rng, 100, 64, center), O.COSINE, (10, 24)


@pytest.mark.gpu
@pytest.mark.timeout(180)
@pytest.mark.parametrize("case", ["f32_l2_offset", "f32_l2_near_duplicates", "f16_ip_norm_spread", "u8_l2_dim768_high",
                                  "f32_cosine_underflow"])
def test_tensor_core_scan_on_ill_conditioned_data(dab, case):
    """Data where the approximate scores cannot rank the true neighbours: the queries the selection may have got wrong
    must be found and re-run, so the result still equals the exact scan."""
    rng = np.random.default_rng(sum(map(ord, case)))
    base, queries, metric, ks = ill_conditioned(case, rng)
    with index(dab, base, metric) as g:
        for k in ks:
            want_ids, want_d = g.flat_knn(queries, k)
            got_ids, got_d = g.flat_knn_tc(queries, k)
            assert np.array_equal(got_ids, want_ids), (k, f"{int((got_ids != want_ids).any(1).sum())} of {len(queries)} queries differ")
            assert np.array_equal(bits(got_d), bits(want_d)), k
    which = np.arange(min(len(queries), 64))
    check_exact(base, queries, metric, ks[-1], want_ids[which], want_d[which], which)


PROFILE_TC = """
import json, sys
import numpy as np, torch
import test_flat_scan as T
rng = np.random.default_rng(96)
centers = rng.normal(size=(50, 96)).astype(np.float32)
cases = {"clustered": (T.clustered(rng, 50000, 96, centers), T.clustered(rng, 1000, 96, centers), T.O.L2)}
base, queries, metric, _ = T.ill_conditioned("f32_l2_offset", rng)
cases["offset"] = (base, queries, metric)
out = {}
import diskann_b200 as dab
for name, (base, queries, metric) in cases.items():
    with T.index(dab, base, metric) as g:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            ids, d = g.flat_knn_tc(queries, 10)
            torch.cuda.synchronize()
        want_ids, want_d = g.flat_knn(queries, 10)
    out[name] = {"kernels": sorted(e.key for e in prof.key_averages()),
                 "equal": bool(np.array_equal(ids, want_ids) and np.array_equal(T.bits(d), T.bits(want_d)))}
print(json.dumps(out))
"""


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_tensor_core_scan_falls_back_only_where_it_cannot_certify():
    """Clustered f32 data (96-d, 50K rows, k = 10) is certified whole: no exact-scan kernel runs.  The offset data
    re-runs queries through it.  (The profiler runs in a process of its own, so its CUPTI session cannot affect the
    other tests' traces.)"""
    import json
    import os
    import subprocess
    import sys

    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([here, os.path.dirname(here), os.environ.get("PYTHONPATH", "")]))
    p = subprocess.run([sys.executable, "-c", PROFILE_TC], capture_output=True, text=True, timeout=280, env=env, cwd=here)
    assert p.returncode == 0, p.stderr[-3000:]
    out = json.loads(p.stdout.strip().splitlines()[-1])
    names = out["clustered"]["kernels"]
    assert any("flat_tc_kernel" in k for k in names) and any("certify_kernel" in k for k in names), names
    assert not any(f in k for k in names for f in FALLBACK_KERNELS), names
    names = out["offset"]["kernels"]
    assert any("flat_float_kernel" in k for k in names) and any("flat_topk_kernel" in k for k in names), names
    assert out["clustered"]["equal"] and out["offset"]["equal"]


# ---------------------------------------------------------------- CPU: the oracle and the error bound

@pytest.mark.parametrize("metric", METRICS)
def test_oracle_bruteforce_skips_nan(metric):
    """orc_bruteforce_knn drops NaN distances like the reference's queue (neighbor/queue.rs:131-134), so a NaN row can
    neither be returned nor break the heap's order."""
    rng = np.random.default_rng(metric)
    base = rng.normal(size=(300, 16)).astype(np.float32)
    nan_rows = [0, 1, 57, 150, 299]
    base[nan_rows] = np.nan
    base[200, 3] = np.nan
    queries = rng.normal(size=(20, 16)).astype(np.float32)
    for k in (5, 50, 400):
        ids, dists = O.bruteforce_knn(base, queries, metric, k)
        check_f64(base, queries, metric, k, ids, dists)
        if metric != O.COSINE:  # a NaN cosine clamps to 1: distance 0, as in the reference
            assert not np.isin(ids, nan_rows + [200]).any() and not np.isnan(dists).any()


def bf16(x):
    """float32 -> bfloat16 round-to-nearest-even (__float2bfloat16_rn for finite values), as float32."""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16).astype(np.uint32).view(np.float32)


def to_f32(x, mode):
    """float64 -> float32, round-to-nearest or toward zero."""
    r = x.astype(np.float32)
    if mode == "rz":
        over = np.abs(r.astype(np.float64)) > np.abs(x)
        r[over] = np.nextafter(r[over], np.float32(0))
    return r


def tc_score_model(q, b, kind, mode, order, rng):
    """flat_tc's approximate score of query q against each row of b: bf16 (hi, lo) splits, the three products (one for
    integers), summed in fp32 in the given order and rounding, then the epilogue."""
    is_int = b.dtype in (np.int8, np.uint8)
    qf, bf = q.astype(np.float32), b.astype(np.float32)
    if is_int:
        terms = [qf.astype(np.float64) * bf.astype(np.float64)]
    else:
        qh, bh = bf16(qf), bf16(bf)
        ql, bl = bf16(qf - qh), bf16(bf - bh)
        terms = [qh.astype(np.float64) * bh, qh.astype(np.float64) * bl, ql.astype(np.float64) * bh]
    t = np.concatenate(terms, axis=1)  # [rows][kp]
    if order == "ascending":
        t = np.take_along_axis(t, np.argsort(np.abs(t), axis=1), 1)
    elif order == "descending":
        t = np.take_along_axis(t, np.argsort(-np.abs(t), axis=1), 1)
    elif order == "random":
        t = t[:, rng.permutation(t.shape[1])]
    acc = np.zeros(len(b), np.float32)
    for j in range(t.shape[1]):
        acc = to_f32(acc.astype(np.float64) + t[:, j], mode)
    nn = np.zeros(len(b), np.float32)
    for j in range(b.shape[1]):  # fmaf chain of the prep kernel
        nn = (nn.astype(np.float64) + bf[:, j].astype(np.float64) ** 2).astype(np.float32)
    a64 = acc.astype(np.float64)
    if kind == "l2":
        return (nn.astype(np.float64) - 2.0 * a64).astype(np.float32)
    if kind == "ip":
        return -acc
    alpha = np.where(nn > 0, -(1.0 / np.sqrt(nn.astype(np.float64))).astype(np.float32), np.float32(0))
    return (a64 * alpha.astype(np.float64)).astype(np.float32)


def tc_score_bound(kind, dim, kp, qn, B, is_int):
    """certify_kernel's bound on the approximate score's error (flat_tc.cu header), without the 1.01 factor and the
    exact distance's own rounding."""
    u = 2.0 ** -24
    gamma = lambda n, v: n * v / (1 - n * v)  # noqa: E731
    g_dim, g_kp = gamma(dim, u), gamma(kp, 2.0 ** -23)
    e = (0.0 if qn * B < 2.0 ** 24 else 1.03 * g_kp) if is_int else 2.0 ** -14 + 1.03 * g_kp
    e_dot = e * qn * B + (0.0 if is_int else kp * 2.0 ** -125 * (qn + B + 1))
    if kind == "l2":
        return 2 * e_dot + (g_dim + 2 * u) * (B * B + 2 * qn * B)
    if kind == "ip":
        return e_dot
    rho = 2.0 ** -22 + g_dim + u
    return qn * ((e + 1) * rho + e) + (0.0 if is_int else kp * 2.0 ** -70 * (qn + 1))


def adversarial(name, rng):
    if name == "offset":
        return (100 + 0.01 * rng.normal(size=(4, 128))).astype(np.float32), (100 + 0.01 * rng.normal(size=(200, 128))).astype(np.float32)
    if name == "mixed_magnitudes":
        m = lambda s: (rng.normal(size=s) * 10 ** rng.uniform(-3, 3, s)).astype(np.float32)  # noqa: E731
        return m((4, 96)), m((200, 96))
    if name == "cancellation":  # q.b ~ 0 out of large terms
        q = rng.normal(size=(4, 96)).astype(np.float32) * 30
        signs = np.where(np.arange(96) % 2 == 0, 1.0, -1.0)
        b = (q[rng.integers(0, 4, 200)] * signs * (1 + 1e-3 * rng.normal(size=(200, 96)))).astype(np.float32)
        return q, b
    if name == "bf16_halfway":  # every element halfway between two bf16 values
        half = lambda s: ((1 + (2 * rng.integers(0, 128, s) + 1) * 2.0 ** -8) * 2.0 ** rng.integers(-4, 5, s)  # noqa: E731
                          * rng.choice([-1, 1], s)).astype(np.float32)
        return half((4, 64)), half((200, 64))
    if name == "u8_dim768_high":
        return rng.integers(240, 256, (4, 768)).astype(np.uint8), rng.integers(240, 256, (200, 768)).astype(np.uint8)
    assert name == "i8_full_range"
    return rng.integers(-128, 128, (4, 128)).astype(np.int8), rng.integers(-128, 128, (200, 128)).astype(np.int8)


@pytest.mark.parametrize("kind", ["l2", "ip", "cos"])
@pytest.mark.parametrize("name", ["offset", "mixed_magnitudes", "cancellation", "bf16_halfway", "u8_dim768_high", "i8_full_range"])
def test_tensor_core_score_error_is_within_the_certified_bound(name, kind):
    """A numpy model of the tensor-core score, with fp32 accumulation rounded to nearest and toward zero in ascending,
    descending, random and GEMM order, stays within the bound certify_kernel subtracts from each range's W."""
    rng = np.random.default_rng(len(name) * 7 + len(kind))
    qs, b = adversarial(name, rng)
    is_int = b.dtype in (np.int8, np.uint8)
    dim = b.shape[1]
    kp = -(-(dim if is_int else 3 * dim) // 64) * 64
    b64 = b.astype(np.float64)
    nb2 = (b64 ** 2).sum(1)
    bn = np.sqrt(nb2)
    worst = 0.0
    for q in qs:
        q64 = q.astype(np.float64)
        qn, xy = np.sqrt((q64 ** 2).sum()), b64 @ q64
        exact = {"l2": nb2 - 2 * xy, "ip": -xy, "cos": -xy / bn}[kind]
        bound = np.array([tc_score_bound(kind, dim, kp, qn, B, is_int) for B in bn])
        for mode in ("rn", "rz"):
            for order in ("gemm", "ascending", "descending", "random"):
                err = np.abs(tc_score_model(q, b, kind, mode, order, rng).astype(np.float64) - exact)
                assert np.all(err <= bound), (mode, order, float(np.max(err / bound)))
                worst = max(worst, float(np.max(err / bound)))
    if name == "i8_full_range" and kind != "cos":
        assert worst == 0.0  # integer dots and scores below 2^24 are exact, whatever the order and rounding
    else:
        assert worst > 0.0
