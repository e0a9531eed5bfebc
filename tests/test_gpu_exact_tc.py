"""Exhaustive search on the tensor cores (csrc/exact_tc.cu: wgmma 3xTF32 filter + exact fp32 re-rank) against the SIMT
kernels (csrc/exact.cu), which are themselves pinned to usearch_exact_search (tests/test_gpu_golden.py): same offsets,
bit-identical distances, ties included -- the tensor cores only decide WHICH rows get the exact arithmetic.

Equal final answers cannot show that the filter works: a query it cannot certify is answered by the SIMT kernels.  So the
filter itself is checked through api.exact_tc_probe, which returns its norms, candidate lists, dropped bounds and
certified flags: approximate distances against a float64 reference within the error bound eps the kernel uses, the list
and dropped-bound bookkeeping, and the certification rate."""
import os

import numpy as np
import pytest

from util import structured

pytestmark = pytest.mark.gpu

NONE = 0xFFFFFFFF
TINY = 2.0 ** -149  # smallest fp32 subnormal


def both(eng, X, Q, k, metric):
    os.environ["LB200_EXACT"] = "simt"
    try:
        ks, ds = eng.exact_search(X, Q, k, metric)
        os.environ["LB200_EXACT"] = "tc"
        os.environ["LB200_EXACT_REPORT"] = "1"
        kt, dt = eng.exact_search(X, Q, k, metric)
    finally:
        os.environ.pop("LB200_EXACT", None)
        os.environ.pop("LB200_EXACT_REPORT", None)
    return ks, ds, kt, dt


def simt(eng, X, Q, k, metric):
    os.environ["LB200_EXACT"] = "simt"
    try:
        return eng.exact_search(X, Q, k, metric)
    finally:
        os.environ.pop("LB200_EXACT", None)


def gaussian(n, d, seed):
    return np.random.default_rng(seed).standard_normal((n, d)).astype(np.float32)


def d64(X, Q, metric):
    """float64 distance matrix [nq][n], with exact.cu's zero-norm cases for cos."""
    X64, Q64 = X.astype(np.float64), Q.astype(np.float64)
    with np.errstate(all="ignore"):
        dot = Q64 @ X64.T
        qn, xn = np.sum(Q64 * Q64, 1)[:, None], np.sum(X64 * X64, 1)[None, :]
        if metric == "l2sq":
            return np.maximum(qn + xn - 2 * dot, 0.0)
        d = 1 - dot / (np.sqrt(qn) * np.sqrt(xn))
        d = np.where((qn == 0) | (xn == 0), 1.0, d)
        return np.where((qn == 0) & (xn == 0), 0.0, d)


def d64_direct(X, Q, metric):
    """Same, without the norm expansion (no cancellation; NaN / inf propagate as in the fp32 kernels)."""
    out = np.empty((len(Q), len(X)))
    X64 = X.astype(np.float64)
    with np.errstate(all="ignore"):
        for i, q in enumerate(Q.astype(np.float64)):
            if metric == "l2sq":
                out[i] = np.sum((X64 - q) ** 2, 1)
            else:
                out[i] = d64(X, Q[i:i + 1], metric)[0]
    return out


def eps64(pr, metric, qn, xn):
    """The kernel's bound (approx_eps in exact_tc.cu) in float64 from the probe's fp32 norms and constants."""
    qn, xn = qn.astype(np.float64), xn.astype(np.float64)
    with np.errstate(all="ignore"):
        a, b = np.sqrt(qn), np.sqrt(xn)
        dot_err = pr["eps_rel"] * a * b + pr["eps_lin"] * (a + b) + pr["eps_abs"]
        if metric == "l2sq":
            return 2 * dot_err + pr["eps_sum"] * (qn + xn)
        ok = (qn >= 2.0 ** -100) & (xn >= 2.0 ** -100) & np.isfinite(qn) & np.isfinite(xn)
        e = np.where(ok, dot_err / (a * b) + pr["eps_sum"], np.inf)
        return np.where((qn == 0) | (xn == 0), pr["eps_rel"] + pr["eps_sum"], e)


def approx_matrix(pr, n):
    """The candidate lists as an [nq][n] matrix (NaN where a row is in no list) plus how often each pair occurs."""
    nq = len(pr["qn"])
    ids = pr["cand_i"].reshape(nq, -1)
    vals = pr["cand_d"].reshape(nq, -1)
    valid = ids != NONE
    qidx = np.broadcast_to(np.arange(nq)[:, None], ids.shape)[valid]
    A = np.full((nq, n), np.nan)
    A[qidx, ids[valid]] = vals[valid]
    counts = np.zeros((nq, n), np.int64)
    np.add.at(counts, (qidx, ids[valid].astype(np.int64)), 1)
    return A, counts


def assert_equal_bits(k1, d1, k2, d2, what):
    assert np.array_equal(k1, k2), (what, float(np.mean(k1 == k2)))
    assert np.array_equal(d1.view(np.uint32), d2.view(np.uint32)), what


def assert_matches_float64(keys, dists, X, Q, metric, k):
    """The SIMT answer against float64 top-k: distances within exact.cu's 1e-5 relative contract (plus the absolute error of
    fp32 subnormal arithmetic), ids equal outside near-ties.  NaN ranks after +inf; distances past fp32's range are +inf.
    l2sq is relative to the distance itself: exact.cu sums (q - x)^2 directly, q_i - x_i is exact or relatively rounded and
    every term is non-negative, so cancellation (common offsets, near-duplicates) costs it nothing.  cos is 1 - a ratio
    that fp32 rounds relative to 1, so its tolerance is absolute."""
    n, d = X.shape
    R = d64_direct(X, Q, metric)
    with np.errstate(all="ignore"):
        R32 = R.astype(np.float32).astype(np.float64)  # overflow -> inf, as in fp32
        qn = np.sum(Q.astype(np.float64) ** 2, 1)
        xn = np.sum(X.astype(np.float64) ** 2, 1)
    m = min(n, k)
    for q in range(len(Q)):
        r = R32[q]
        with np.errstate(all="ignore"):
            if metric == "l2sq":
                tol = 1e-5 * np.abs(r) + 8 * d * TINY
            else:
                tol = 1e-5 + 1e-6 + 8 * d * TINY * (1 / np.maximum(qn[q], TINY) + 1 / np.maximum(xn, TINY))
        order = np.lexsort((np.arange(n), np.nan_to_num(r, nan=np.inf, posinf=np.inf), np.isnan(r)))[:m]
        got_k, got_d = keys[q, :m].astype(np.int64), dists[q, :m].astype(np.float64)
        assert len(set(got_k.tolist())) == m and (got_k < n).all(), (q, got_k)
        assert (keys[q, m:] == np.uint64(2 ** 64 - 1)).all() and np.isinf(dists[q, m:]).all(), q

        def same(a, b, t):
            return (np.isnan(a) and np.isnan(b)) or a == b or abs(a - b) <= t

        for i in range(m):
            ref = r[order[i]]
            assert same(got_d[i], ref, tol[order[i]]), (q, i, got_d[i], ref)
            if got_k[i] != order[i]:  # only inside a near-tie group
                assert same(r[got_k[i]], ref, 2 * max(tol[got_k[i]], tol[order[i]])), (q, i, got_k[i], order[i])


def check_filter_bound(pr, X, Q, metric):
    """|approx - float64| <= eps on every pair the lists hold; returns the largest |approx - d64| / eps."""
    A, _ = approx_matrix(pr, len(X))
    D = d64(X, Q, metric)
    E = eps64(pr, metric, pr["qn"][:, None], pr["xn"][None, :])
    held = ~np.isnan(A)
    with np.errstate(all="ignore"):
        ratio = np.where(held, np.abs(A - D) / E, 0.0)
    worst = float(ratio.max())
    assert worst <= 1.0, "largest |approx - d64| / eps = %.3f at (query, row) %s" % (
        worst, np.unravel_index(int(ratio.argmax()), ratio.shape))
    return worst


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("data", ["structured", "gaussian"])
@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("n,d,nq,k", [(70_000, 96, 300, 10), (40_000, 100, 130, 100), (5_000, 768, 64, 10), (300, 32, 5, 20)])
def test_tensor_core_exact_search_equals_simt(eng, metric, n, d, nq, k, data):
    """Same answer as the SIMT kernels, and the filter certifies every query on continuous data (no SIMT fallback)."""
    gen = structured if data == "structured" else gaussian
    X, Q = gen(n, d, seed=5), gen(nq, d, seed=6)
    ks, ds = simt(eng, X, Q, k, metric)
    pr = eng.exact_tc_probe(X, Q, k, metric)
    assert_equal_bits(pr["keys"], pr["dists"], ks, ds, "probe vs simt")
    kt, dt = both(eng, X, Q, k, metric)[2:]
    assert_equal_bits(kt, dt, ks, ds, "tc vs simt")
    print("CERTIFIED %s %s n=%d d=%d nq=%d k=%d: %d of %d" % (data, metric, n, d, nq, k, nq - int(pr["unsafe"].sum()), nq))
    assert not pr["unsafe"].any(), "certified %d of %d" % (nq - int(pr["unsafe"].sum()), nq)


def test_tensor_core_exact_search_with_exact_ties_and_zero_rows(eng):
    """Integer vectors: whole groups of rows at exactly the same distance (the order is by offset); zero rows and a zero query
    exercise the cosine special cases (index_plugins.hpp:1022-1026)."""
    rng = np.random.default_rng(3)
    X = rng.integers(-2, 3, (20_000, 24)).astype(np.float32)
    X[::997] = 0
    Q = rng.integers(-2, 3, (40, 24)).astype(np.float32)
    Q[3] = 0
    for metric in ("l2sq", "cos"):
        ks, ds, kt, dt = both(eng, X, Q, 25, metric)
        assert np.array_equal(kt, ks) and np.array_equal(dt.view(np.uint32), ds.view(np.uint32))


def test_default_path_uses_the_tensor_cores_for_large_problems(eng, capfd):
    """No environment override: n >= 32768 rows of f32 take the tensor-core path (its report line proves it ran, and that it
    certified every query); results equal the forced SIMT run."""
    X = structured(40_000, 64, seed=9)
    Q = structured(50, 64, seed=10)
    capfd.readouterr()
    os.environ["LB200_EXACT_REPORT"] = "1"
    try:
        k0, d0 = eng.exact_search(X, Q, 10, "l2sq")
    finally:
        os.environ.pop("LB200_EXACT_REPORT", None)
    err = capfd.readouterr().err
    assert "tensor-core filter certified 50 of 50 queries" in err, err
    k1, d1 = simt(eng, X, Q, 10, "l2sq")
    assert_equal_bits(k0, d0, k1, d1, "default vs simt")


@pytest.mark.parametrize("k", [150, 160, 192])
def test_default_path_with_large_k(eng, capfd, k):
    """k >= 150 (KP = 256) with one query tile: the re-rank's sort of groups * KP upper bounds must fit in shared memory."""
    X = structured(40_000, 96, seed=11)
    Q = structured(64, 96, seed=12)
    capfd.readouterr()
    os.environ["LB200_EXACT_REPORT"] = "1"
    try:
        k0, d0 = eng.exact_search(X, Q, k, "l2sq")
    finally:
        os.environ.pop("LB200_EXACT_REPORT", None)
    assert "tensor-core filter certified" in capfd.readouterr().err
    k1, d1 = simt(eng, X, Q, k, "l2sq")
    assert_equal_bits(k0, d0, k1, d1, "default vs simt")


# ---- the filter's approximate distances against float64 --------------------------------------------------------------
# k = 192 gives KP = 256 >= the 128 rows of the single row tile each group gets when n = 2000 (16 tiles <= groups): every list
# holds its whole group, so the probe returns the full approximate distance matrix.
FULL_N, FULL_K = 2000, 192


def full_matrix_case(eng, d, nq, metric, positive=False):
    if positive:
        rng = np.random.default_rng(d)
        X = rng.uniform(0.5, 1.0, (FULL_N, d)).astype(np.float32)
        Q = rng.uniform(0.5, 1.0, (nq, d)).astype(np.float32)
    else:
        X = structured(FULL_N, d, seed=20 + d)
        Q = structured(nq, d, seed=21 + d)
        X[7] *= 1e3  # norm-dominated pairs in both directions
        Q[0] *= 1e-3
    pr = eng.exact_tc_probe(X, Q, FULL_K, metric)
    assert pr["KP"] == 256 and pr["groups"] * 128 >= FULL_N, (pr["KP"], pr["groups"])
    _, counts = approx_matrix(pr, FULL_N)
    assert (counts == 1).all(), "pairs held %s times" % np.unique(counts)
    worst = check_filter_bound(pr, X, Q, metric)
    ks, ds = simt(eng, X, Q, FULL_K, metric)
    assert_equal_bits(pr["keys"], pr["dists"], ks, ds, "probe vs simt")
    print("MARGIN full-matrix%s %s d=%d nq=%d: max |approx - d64| / eps = %.4f, certified %d of %d" % (
        " positive" if positive else "", metric, d, nq, worst, nq - int(pr["unsafe"].sum()), nq))
    return worst


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("d", [1, 3, 4, 28, 31, 32, 33, 100, 127, 128, 129, 768, 2048])
def test_filter_distances_within_eps_of_float64_across_dims(eng, metric, d):
    """k-block (32 floats) and lane-chunk (128 floats) edges."""
    full_matrix_case(eng, d, 129, metric)


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("d", [128, 768, 2048])
def test_filter_distances_within_eps_of_float64_on_positive_data(eng, metric, d):
    """Positive, nearly parallel vectors: every product and partial sum has the same sign, so rounding errors of the
    tensor-core accumulation add up instead of cancelling -- the data closest to the bound's worst case."""
    full_matrix_case(eng, d, 129, metric, positive=True)


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("nq", [1, 127, 128, 129, 300])
def test_filter_distances_within_eps_of_float64_across_query_tiles(eng, metric, nq):
    """Query-tile (128) and MMA-warpgroup (64) edges."""
    full_matrix_case(eng, 100, nq, metric)


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("n,d,nq", [(200_000, 64, 64), (34_000, 2048, 32)])
def test_filter_lists_and_dropped_bounds_at_large_n(eng, metric, n, d, nq):
    """Many row tiles per CTA (both stages and the accumulator tile wrap many times).  Row group g holds tiles g, g + G, ...
    For each (query, group) with a full list, every absent row is at least as far as the list's worst approximation minus eps,
    and dropped_lb lies between the absent rows' min(d64 - 2 eps) and min(d64).  Query 0 sees the rows in order of decreasing
    distance, so its lists only ever evict: dropped_lb then comes from evicted roots alone."""
    k = 10
    X = structured(n, d, seed=30)
    Q = structured(nq, d, seed=31)
    X = X[np.argsort(-d64(X, Q[:1], metric)[0], kind="stable")]
    pr = eng.exact_tc_probe(X, Q, k, metric)
    G, KP = pr["groups"], pr["KP"]
    assert (n + 127) // 128 >= 2 * G, G
    A, counts = approx_matrix(pr, n)
    assert counts.max() == 1
    D = d64(X, Q, metric)
    E = eps64(pr, metric, pr["qn"][:, None], pr["xn"][None, :])
    held = ~np.isnan(A)
    ratio = np.where(held, np.abs(np.where(held, A, 0) - D) / E, 0.0)
    assert ratio.max() <= 1.0, ratio.max()
    group_of = (np.arange(n) // 128) % G
    rows_of = [np.nonzero(group_of == g)[0] for g in range(G)]
    for q in range(nq):
        for g, rows in enumerate(rows_of):
            inlist = held[q, rows]
            if inlist.sum() < KP:
                assert inlist.all() and pr["dropped_lb"][q, g] == np.inf, (q, g)
                continue
            absent = rows[~inlist]
            worst = A[q, rows[inlist]].max()
            assert (D[q, absent] >= worst - E[q, absent]).all(), (q, g)
            lb = pr["dropped_lb"][q, g]
            assert lb <= D[q, absent].min(), (q, g, lb, D[q, absent].min())
            assert lb >= (D[q, absent] - 2 * E[q, absent]).min(), (q, g, lb)
    # the bound holds against the exact kernel's own fp32 arithmetic (pair_distance_kernel: exact.cu's lane layout and
    # reduction, bit-identical to the search's distances -- checked on the final answer first)
    ks = pr["keys"].astype(np.int64)
    qi = np.repeat(np.arange(nq), k)
    s = eng.distance_batch(Q[qi], X[ks.ravel()], metric)
    assert np.array_equal(s.view(np.uint32), pr["dists"].ravel().view(np.uint32))
    rng = np.random.default_rng(0)
    pq, pi = np.nonzero(held)
    pick = rng.choice(len(pq), min(20_000, len(pq)), replace=False)
    pq, pi = pq[pick], pi[pick]
    s = eng.distance_batch(Q[pq], X[pi], metric).astype(np.float64)
    r2 = np.abs(A[pq, pi] - s) / E[pq, pi]
    assert r2.max() <= 1.0, r2.max()
    print("MARGIN large-n %s n=%d d=%d: max |approx - d64| / eps = %.4f, vs fp32 exact %.4f, certified %d of %d" % (
        metric, n, d, float(ratio.max()), float(r2.max()), nq - int(pr["unsafe"].sum()), nq))
    assert not pr["unsafe"].any()


# ---- edge data: the tensor-core answer equals SIMT bit for bit, SIMT agrees with float64 --------------------------------
def edge_case(eng, X, Q, k, metric):
    pr = eng.exact_tc_probe(X, Q, k, metric)
    ks, ds = simt(eng, X, Q, k, metric)
    assert_equal_bits(pr["keys"], pr["dists"], ks, ds, "probe vs simt")
    assert_matches_float64(ks, ds, X, Q, metric, k)
    return pr


def report(name, metric, pr, X, Q):
    A, _ = approx_matrix(pr, len(X))
    D = d64(X, Q, metric)
    E = eps64(pr, metric, pr["qn"][:, None], pr["xn"][None, :])
    with np.errstate(all="ignore"):
        r = np.abs(A - D) / E
    r = r[np.isfinite(r)]
    print("MARGIN edge %s %s: max |approx - d64| / eps = %s, certified %d of %d" % (
        name, metric, "%.4f" % r.max() if r.size else "n/a", len(Q) - int(pr["unsafe"].sum()), len(Q)))
    return float(r.max()) if r.size else 0.0


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
def test_edge_exact_duplicates_beyond_the_list(eng, metric):
    """128 copies of query 0 fill row tile 0 (one row group): more zero-distance rows than a list keeps, so the dropped
    bound reaches the k-th upper bound and the query falls back; the answer is the lowest offsets."""
    X = structured(4000, 32, seed=40)
    Q = structured(8, 32, seed=41)
    X[:128] = Q[0]
    pr = edge_case(eng, X, Q, 10, metric)
    assert pr["KP"] < 128 and pr["unsafe"][0] == 1
    assert np.array_equal(pr["keys"][0], np.arange(10))
    assert report("duplicates", metric, pr, X, Q) <= 1.0


def test_edge_large_common_offset(eng):
    """1e3 + N(0, 1e-2): eps (relative to |q|^2 + |x|^2) dwarfs every distance, so more than kRrCap = 512 rows survive.
    k = 192 (KP = 256) with 3000 rows (one 128-row tile per group): no list drops anything, so the kRrCap branch alone makes
    the queries fall back."""
    k = 192
    rng = np.random.default_rng(42)
    X = (1e3 + 1e-2 * rng.standard_normal((3000, 32))).astype(np.float32)
    Q = (1e3 + 1e-2 * rng.standard_normal((16, 32))).astype(np.float32)
    pr = edge_case(eng, X, Q, k, "l2sq")
    assert pr["KP"] == 256 and pr["groups"] * 128 >= len(X)
    assert (pr["dropped_lb"] == np.inf).all()
    # survivors of the re-rank's bound test, recounted on the host: (approx - eps) <= k-th smallest (approx + eps)
    A, counts = approx_matrix(pr, len(X))
    assert (counts == 1).all()
    E = eps64(pr, "l2sq", pr["qn"][:, None], pr["xn"][None, :])
    kth_ub = np.sort(A + E, axis=1)[:, k - 1:k]
    survivors = (A - E <= kth_ub).sum(1)
    assert (survivors > 512).all(), survivors.min()
    assert pr["unsafe"].all()
    assert report("offset", "l2sq", pr, X, Q) <= 1.0


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
def test_edge_near_duplicates(eng, metric):
    rng = np.random.default_rng(43)
    X = structured(3000, 64, seed=44)
    Q = structured(8, 64, seed=45)
    X[100:140] = Q[1] * (1 + 1e-6 * rng.standard_normal((40, 64))).astype(np.float32)
    pr = edge_case(eng, X, Q, 20, metric)
    assert report("near-duplicates", metric, pr, X, Q) <= 1.0


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("scale", [-70, -40, 40, 62])
def test_edge_power_of_two_scaled(eng, metric, scale):
    """2^-70: squares and products are subnormal; 2^-40 and 2^40: normal; 2^62: norms overflow to +inf."""
    X = structured(3000, 32, seed=46) * np.float32(2.0 ** scale)
    Q = structured(8, 32, seed=47) * np.float32(2.0 ** scale)
    if metric == "cos" and scale == 62:
        # |x|^2 overflows fp32, so the fp32 metric is not the float64 one: only the two GPU paths are compared
        pr = eng.exact_tc_probe(X, Q, 10, metric)
        assert_equal_bits(pr["keys"], pr["dists"], *simt(eng, X, Q, 10, metric), "probe vs simt")
    else:
        pr = edge_case(eng, X, Q, 10, metric)
    if scale == 62:
        assert pr["unsafe"].all()  # non-finite approximations certify nothing
    else:
        assert report("scale 2^%d" % scale, metric, pr, X, Q) <= 1.0
    if scale in (-40, 40):
        assert not pr["unsafe"].any()


def test_edge_near_zero_query_against_wide_rows(eng):
    """|q| << |x| at d = 2048: the l2sq bound rests on the norms' and the exact sum's fp32 rounding alone."""
    X = structured(3000, 2048, seed=48)
    Q = structured(4, 2048, seed=49)
    Q[0] *= 1e-4
    Q[1] = 0
    pr = edge_case(eng, X, Q, 10, "l2sq")
    assert report("near-zero query d=2048", "l2sq", pr, X, Q) <= 1.0


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
def test_edge_nan_and_inf(eng, metric):
    """Rows and queries holding NaN or +-inf: NaN distances rank after everything, and a query whose filter saw a non-finite
    approximation is not certified."""
    X = structured(3000, 32, seed=50)
    Q = structured(6, 32, seed=51)
    X[5, 3] = np.nan
    X[17, 0] = np.inf
    X[40, :] = -np.inf
    X[41, 2] = np.inf
    X[41, 9] = -np.inf
    Q[1, 2] = np.nan
    Q[2, 0] = np.inf
    pr = edge_case(eng, X, Q, 10, metric)
    assert pr["unsafe"].all()
    # without the poisoned rows, the clean queries are certified again
    clean = np.ones(len(X), bool)
    clean[[5, 17, 40, 41]] = False
    pr = edge_case(eng, X[clean], Q[[0, 3, 4, 5]], 10, metric)
    assert not pr["unsafe"].any()


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("n,nq", [(5, 3), (20, 3), (1, 3), (3000, 1), (1, 1)])
def test_edge_few_rows_or_one_query(eng, metric, n, nq):
    X = structured(n, 40, seed=52)
    Q = structured(nq, 40, seed=53)
    pr = edge_case(eng, X, Q, 20, metric)
    assert not pr["unsafe"].any()


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("k", [1, 31, 32, 33, 149, 150, 192])
def test_edge_k(eng, metric, k):
    X = structured(5000, 48, seed=54)
    Q = structured(40, 48, seed=55)
    pr = edge_case(eng, X, Q, k, metric)
    assert not pr["unsafe"].any()


def test_simt_exact_search_past_the_block_count_growth(eng):
    """n > 1024 * 4096 rows: launch_exact grows rows_per_block so that at most 1024 blocks run (d = 8 stays on SIMT)."""
    n = 4096 * 1024 + 1000
    X = gaussian(n, 8, seed=60)
    Q = gaussian(8, 8, seed=61)
    ks, ds = eng.exact_search(X, Q, 10, "l2sq")
    X64 = X.astype(np.float64)
    for q in range(len(Q)):
        r = np.sum((X64 - Q[q].astype(np.float64)) ** 2, 1)
        order = np.lexsort((np.arange(n), r))[:10]
        assert np.allclose(ds[q], r[order], rtol=1e-5, atol=1e-6), q
        assert np.array_equal(ks[q].astype(np.int64), order) or np.allclose(r[ks[q].astype(np.int64)], r[order], rtol=1e-5), q
