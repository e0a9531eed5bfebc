"""The projected screen of the search beam (pscreen.cu, screen.cuh, DESIGN.md 4.1).

An f32 l2sq / cos index whose rows have most of their energy in a few directions keeps, instead of the int8 copy of every
dimension, a 64- or 128-byte record per row: k int8 codes of P x and two residual norms.  The screen rejects a candidate whose
lower bound lb >= radius without reading its row, so lb must never exceed the distance the search kernel computes, for ANY
basis P.  api.search_pscreen_probe returns both for every (query, row) pair, with the records, pre-pass and bound the search
uses; the remaining tests check that searches return exactly what they return without a screen, with the same counters."""
import numpy as np
import pytest

from test_gpu_search_screen import DIMS, KINDS, _data, _oracle_pair, _violations
from util import compare_results, structured

pytestmark = pytest.mark.gpu

KS = [16, 32, 48, 64, 96, 112]


def _pca(X, k):
    X64 = X.astype(np.float64)
    X64[~np.isfinite(X64)] = 0.0
    w, V = np.linalg.eigh(X64.T @ X64)
    P = np.zeros((k, X.shape[1]), np.float32)
    m = min(k, X.shape[1])
    P[:m] = V[:, ::-1][:, :m].T
    return P


def _bases(X, d, k, rng):
    """the rows' own basis, and adversarial ones: non-orthonormal, scaled by 2^+-20, rank-deficient, all zero"""
    own = _pca(X, k)
    rand = rng.standard_normal((k, d)).astype(np.float32)
    rank_def = np.repeat(rand[:1], k, axis=0) * np.arange(1, k + 1, dtype=np.float32)[:, None]
    return {"own": own, "random": rand, "big": own * np.float32(2.0**20), "small": rand * np.float32(2.0**-20),
            "rank_deficient": rank_def, "zero": np.zeros((k, d), np.float32)}


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("d", DIMS)
def test_pscreen_bound_below_kernel_distance(eng, metric, d):
    rng = np.random.default_rng(d)
    for i, kind in enumerate(KINDS):
        X, Q = _data(kind, 160, 24, d, seed=d)
        k = KS[(i + DIMS.index(d)) % len(KS)]  # every k at every NQ across the kinds
        for name, P in _bases(X, d, k, rng).items():
            lb, dist = eng.search_pscreen_probe(X, Q, metric, basis=P)
            bad = _violations(lb, dist)
            assert not bad.any(), (kind, name, k, int(bad.sum()), lb[bad][:4], dist[bad][:4])


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("d", [64, 320, 768])
def test_pscreen_engine_basis_below_kernel_distance(eng, metric, d):
    """the engine's own basis (moment matrix on the device, eigenvectors on the host) at every k"""
    for i, kind in enumerate(("structured", "zero_mean", "nonfinite")):
        X, Q = _data(kind, 400, 16, d, seed=7)
        for k in KS[i::3] if d > 320 else KS:  # every k at every d; all of them at every kind below d768
            lb, dist = eng.search_pscreen_probe(X, Q, metric, k=k)
            bad = _violations(lb, dist)
            assert not bad.any(), (kind, k, int(bad.sum()))


def test_pscreen_degenerate_rows_always_pass(eng):
    X, Q = _data("nonfinite", 40, 6, 96, seed=1)
    P = _pca(X, 16)
    for metric in ("l2sq", "cos"):
        lb, _ = eng.search_pscreen_probe(X, Q, metric, basis=P)
        for row in (3, 5, 9):
            assert not (lb[:, row] > -np.inf).any(), (metric, row)
        for q in (1, 2):
            assert not (lb[q] > -np.inf).any(), (metric, q)


def _pass_fraction(lb, dist, lo=64, hi=4000, rank=127):
    """share of candidates (distance ranks lo..hi, standing in for a beam's) that a screen at the rank-th distance keeps"""
    order = np.argsort(dist, axis=1)
    radius = np.take_along_axis(dist, order[:, rank:rank + 1], axis=1)
    cand = order[:, lo:hi]
    keep = ~(np.take_along_axis(lb, cand, axis=1) >= radius)
    return keep.mean()


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
def test_pscreen_as_tight_as_int8_screen(eng, metric):
    """On the benchmark's distribution (32-d latent + noise, d768) the projected screen keeps at most 1.5x (+0.5 points) the
    candidates the int8 screen keeps."""
    X = structured(20000, 768, seed=1234)
    Q = structured(40, 768, seed=42)
    lb8, dist = eng.search_screen_probe(X, Q, metric)
    lbp, distp = eng.search_pscreen_probe(X, Q, metric)
    assert np.array_equal(dist.view(np.uint32), distp.view(np.uint32))
    f8, fp = _pass_fraction(lb8, dist), _pass_fraction(lbp, dist)
    exact = _pass_fraction(dist, dist)
    assert exact <= fp <= 1.5 * f8 + 0.005, (exact, f8, fp)


def _knobs(g, Q, monkeypatch, knobs=("0", "1", "2"), ef=96):
    out = {}
    for knob in knobs:
        monkeypatch.setenv("LB200_SEARCH_SCREEN", knob)
        k, dd, c = g.search_batch(Q, 10, ef=ef)
        out[knob] = (k, dd, c, g.last_stats())
    return out


def _assert_same(out, ref="0"):
    k0, d0, c0, s0 = out[ref]
    for knob, (k, dd, c, s) in out.items():
        assert np.array_equal(k0, k), knob
        assert np.array_equal(d0.view(np.uint32), dd.view(np.uint32)), knob
        assert np.array_equal(c0, c), knob
        for f in ("computed_distances", "base_pops", "upper_hops", "limbo_overflows"):
            assert s0[f] == s[f], (knob, f)


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("kind", ["structured", "zero_mean", "huge_coord", "offset", "near_dup", "zeros", "nonfinite"])
def test_pscreen_knobs_bit_identical(eng, monkeypatch, metric, kind):
    """off, int8 and projected screens on one graph: the same keys, distance bits, counts and counters"""
    X, Q = _data(kind, 3000, 100, 320, seed=5)
    g = eng.Index(320, metric, "f32", M=16, efc=64, ef=64)
    g.add_batch(np.arange(len(X), dtype=np.uint64), X)
    out = _knobs(g, Q, monkeypatch)
    _assert_same(out)
    assert out["0"][3]["screen_kind"] == 0 and out["1"][3]["screen_kind"] == 1 and out["2"][3]["screen_kind"] == 2
    assert out["2"][3]["screen_dims"] in KS
    if kind == "structured":
        assert out["2"][3]["full_rows_read"] < out["0"][3]["full_rows_read"]
        assert out["2"][3]["algorithmic_bytes"] < out["1"][3]["algorithmic_bytes"]


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("d,ef", [(256, 64), (768, 128)])
def test_pscreen_search_matches_oracle(eng, port, monkeypatch, metric, d, ef):
    X = structured(3000, d, seed=11)
    Q = structured(200, d, seed=12)
    pidx, g = _oracle_pair(eng, port, X, metric, 16, ef)
    out = _knobs(g, Q, monkeypatch, ef=ef)
    _assert_same(out)
    gk, gd, gc, st = out["2"]
    pk, pd, pc, tot = pidx.search_batch(Q, 10)
    assert np.array_equal(gc.astype(np.int64), pc)
    assert np.allclose(gd, pd, rtol=1e-5, atol=1e-6), np.abs(gd - pd).max()
    exact, ok = compare_results(gk, gd, pk, pd)
    assert ok == len(Q), (exact, ok)
    assert exact >= 0.97 * len(Q), exact
    for f in ("computed_distances", "base_pops", "upper_hops"):
        if out["0"][3][f] == tot[f]:
            assert st[f] == tot[f], f
    assert st["full_rows_read"] < st["computed_distances"]


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
def test_pscreen_choice(eng, monkeypatch, metric):
    """automatic: structured rows give the projected screen, isotropic Gaussian rows and small indexes the int8 one"""
    monkeypatch.delenv("LB200_SEARCH_SCREEN", raising=False)
    rng = np.random.default_rng(3)
    cases = {"structured": (structured(20000, 320, seed=31), 2), "gaussian": (rng.standard_normal((20000, 320)).astype(np.float32), 1),
             "small": (structured(3000, 320, seed=32), 1)}
    Q = structured(64, 320, seed=33)
    for name, (X, want) in cases.items():
        g = eng.Index(320, metric, "f32", M=16, efc=64, ef=64)
        g.add_batch(np.arange(len(X), dtype=np.uint64), X)
        g.search_batch(Q, 10)
        st = g.last_stats()
        P, sec = g.screen_basis()
        assert st["screen_kind"] == want, (name, st)
        if want == 2:
            assert P is not None and len(P) == st["screen_dims"] and len(P) in KS, name
            assert len(P) <= 48  # a 32-d latent: one 64-byte record
        else:
            assert P is None and st["screen_dims"] == 320, name
            # forcing the projected screen for an experiment leaves the automatic mode on the int8 one it chose
            monkeypatch.setenv("LB200_SEARCH_SCREEN", "2")
            g.search_batch(Q, 10)
            assert g.last_stats()["screen_kind"] == 2, name
            monkeypatch.delenv("LB200_SEARCH_SCREEN")
            g.search_batch(Q, 10)
            assert g.last_stats()["screen_kind"] == 1, name


def test_pscreen_survives_growth_and_reload(eng, monkeypatch):
    """the basis is kept through growth; load_buffer chooses it again from the loaded rows, to the same bits every time"""
    X = structured(24000, 384, seed=21)
    Q = structured(64, 384, seed=22)
    g = eng.Index(384, "cos", "f32", M=16, efc=64, ef=64)
    g.add_batch(np.arange(17000, dtype=np.uint64), X[:17000])
    g.build()
    P0, _ = g.screen_basis()
    assert P0 is not None
    for lo in range(17000, 24000, 2500):  # several adds, each may grow the capacity
        g.add_batch(np.arange(lo, min(lo + 2500, 24000), dtype=np.uint64), X[lo:lo + 2500])
    g.build()
    P1, _ = g.screen_basis()
    assert np.array_equal(P0.view(np.uint32), P1.view(np.uint32))
    buf = g.save_buffer()
    hs = []
    for _ in range(2):
        h = eng.Index(384, "cos", "f32", M=16, efc=64, ef=64)
        h.load_buffer(buf)
        hs.append(h)
    Pa, _ = hs[0].screen_basis()
    Pb, _ = hs[1].screen_basis()
    assert Pa is not None and np.array_equal(Pa.view(np.uint32), Pb.view(np.uint32))
    ref = None
    for idx in (g, *hs):
        out = _knobs(idx, Q, monkeypatch, knobs=("0", "2"))
        _assert_same(out)
        assert out["2"][3]["full_rows_read"] < out["2"][3]["computed_distances"]
        monkeypatch.delenv("LB200_SEARCH_SCREEN")
        k, dd, c = idx.search_batch(Q, 10, ef=96)
        assert idx.last_stats()["screen_kind"] == 2
        if ref is None:
            ref = (k, dd.view(np.uint32))
        assert np.array_equal(k, ref[0]) and np.array_equal(dd.view(np.uint32), ref[1])
