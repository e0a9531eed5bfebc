"""The int8 screen of the search beam (screen.cuh, DESIGN.md 4.1).

An f32 l2sq / cos index keeps an int8 copy of its rows; once the level-0 top list is full, the search rejects a candidate
whose lower bound lb >= radius without reading its fp32 row.  That is only safe if lb never exceeds the distance the search
kernel itself computes, rounding included.  api.search_screen_probe returns both, from the device functions the search
uses, for every (query, row) pair; the remaining tests check that searches with the screen return exactly what the oracle
and the unscreened kernel return, with the same work counters."""
import numpy as np
import pytest

from util import build_port_index, compare_results, structured

pytestmark = pytest.mark.gpu

# every chunks-per-lane count NQ (1, 2, 3, 4, 6, 8, 12, 16) and ragged tails
DIMS = [1, 3, 4, 17, 64, 127, 128, 200, 256, 384, 385, 512, 700, 768, 1000, 1024, 1536, 2047, 2048]


def _data(kind, n, nq, d, seed):
    rng = np.random.default_rng(seed)
    if kind == "zero_mean":
        X, Q = rng.standard_normal((n, d)), rng.standard_normal((nq, d))
    elif kind == "positive":
        X, Q = rng.random((n, d)), rng.random((nq, d))
    elif kind == "structured":
        X, Q = structured(n, d, seed), structured(nq, d, seed + 1)
    elif kind == "huge_coord":  # one huge coordinate per row: a coarse scale for everything else
        X, Q = rng.standard_normal((n, d)), rng.standard_normal((nq, d))
        X[np.arange(n), rng.integers(0, d, n)] = 1e4
    elif kind == "offset":  # large common offset: distances are tiny next to the norms
        X, Q = 1000.0 + rng.standard_normal((n, d)) * 0.01, 1000.0 + rng.standard_normal((nq, d)) * 0.01
    elif kind == "near_dup":  # queries a rounding error away from rows
        X = rng.standard_normal((n, d))
        Q = X[rng.integers(0, n, nq)] * (1 + 1e-6 * rng.standard_normal((nq, d)))
    elif kind == "tiny":
        X, Q = rng.standard_normal((n, d)) * 2.0**-70, rng.standard_normal((nq, d)) * 2.0**-70
    elif kind == "huge":
        X, Q = rng.standard_normal((n, d)) * 2.0**62, rng.standard_normal((nq, d)) * 2.0**62
    elif kind == "zeros":  # zero rows and zero queries among ordinary ones
        X, Q = rng.standard_normal((n, d)), rng.standard_normal((nq, d))
        X[::7] = 0.0
        Q[::5] = 0.0
    elif kind == "int8_exact":  # rows the int8 codes represent exactly (r = 0): only the rounding terms keep the bound valid
        X = rng.integers(-127, 128, (n, d)).astype(np.float64)
        X[np.arange(n), rng.integers(0, d, n)] = 127.0
        Q = X[rng.integers(0, n, nq)] + rng.standard_normal((nq, d)) * 1e-3
    elif kind == "nonfinite":
        X, Q = rng.standard_normal((n, d)), rng.standard_normal((nq, d))
        X[3, 0], X[5, d // 2], X[9, d - 1] = np.nan, np.inf, -np.inf
        Q[1, 0], Q[2, d - 1] = np.nan, np.inf
    else:
        raise ValueError(kind)
    return X.astype(np.float32), Q.astype(np.float32)


def _violations(lb, d):
    """pairs where the bound is wrong: lb > d.  A NaN bound means 'keep'; a NaN distance is rejected by the walk anyway."""
    with np.errstate(invalid="ignore"):
        return ~np.isnan(lb) & ~np.isnan(d) & (lb > d)


KINDS = ["zero_mean", "positive", "structured", "huge_coord", "offset", "near_dup", "int8_exact", "tiny", "huge", "zeros",
         "nonfinite"]


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("d", DIMS)
def test_bound_below_kernel_distance(eng, metric, d):
    for kind in KINDS:
        X, Q = _data(kind, 160, 24, d, seed=d)
        lb, dist = eng.search_screen_probe(X, Q, metric)
        bad = _violations(lb, dist)
        assert not bad.any(), (kind, int(bad.sum()), lb[bad][:4], dist[bad][:4])


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
def test_bound_is_tight_on_continuous_data(eng, metric):
    """The screen only saves bytes if lb is close to d: on ordinary data the gap is a small fraction of the distances."""
    X, Q = _data("structured", 2000, 50, 768, seed=3)
    lb, dist = eng.search_screen_probe(X, Q, metric)
    gap = (dist - lb) / np.median(dist)
    assert (gap >= 0).all()
    assert np.median(gap) < 0.05, np.median(gap)


def test_degenerate_rows_always_pass(eng):
    X, Q = _data("nonfinite", 40, 6, 96, seed=1)
    X[7] = 0.0
    X[11] = 2.0**-148  # scale underflows to 0
    for metric in ("l2sq", "cos"):
        lb, _ = eng.search_screen_probe(X, Q, metric)
        for row in (3, 5, 9):
            assert not (lb[:, row] > -np.inf).any(), (metric, row)
        assert not (lb[:, 11] > -np.inf).any()
    lb, _ = eng.search_screen_probe(X, Q, "cos")
    assert not (lb[:, 7] > -np.inf).any()  # zero norm: cos_from_parts' special cases
    Q[0] = 0.0
    lb, _ = eng.search_screen_probe(X, Q, "cos")
    assert not (lb[0] > -np.inf).any()


def _oracle_pair(eng, port, X, metric, M, ef):
    pidx = build_port_index(port, X, metric, "f32", M=M, efc=128, ef=ef)
    g = eng.Index(X.shape[1], metric, "f32", M=M, efc=128, ef=ef)
    g.load_buffer(pidx.save_buffer())
    return pidx, g


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("d,ef", [(256, 64), (768, 128), (1024, 64)])
def test_screened_search_matches_oracle(eng, port, monkeypatch, metric, d, ef):
    """Screened search (the default at d >= 256) on an oracle-built graph: exactly the unscreened kernel's ids, distances
    and work counters, and the oracle's results within test_same_graph_same_ids' tolerance.  The GPU and the oracle sum
    distances in different orders, so a candidate within an ulp of the radius can be decided differently; the counters are
    required to equal the oracle's wherever the unscreened kernel's do."""
    monkeypatch.delenv("LB200_SEARCH_SCREEN", raising=False)
    X = structured(3000, d, seed=11)
    Q = structured(200, d, seed=12)
    pidx, g = _oracle_pair(eng, port, X, metric, 16, ef)
    gk, gd, gc = g.search_batch(Q, 10)
    st = g.last_stats()
    monkeypatch.setenv("LB200_SEARCH_SCREEN", "0")
    uk, ud, uc = g.search_batch(Q, 10)
    su = g.last_stats()
    pk, pd, pc, tot = pidx.search_batch(Q, 10)
    assert np.array_equal(gc.astype(np.int64), pc)
    assert np.allclose(gd, pd, rtol=1e-5, atol=1e-6), np.abs(gd - pd).max()
    exact, ok = compare_results(gk, gd, pk, pd)
    assert ok == len(Q), (exact, ok)
    assert exact >= 0.97 * len(Q), exact
    assert np.array_equal(gk, uk) and np.array_equal(gd.view(np.uint32), ud.view(np.uint32)) and np.array_equal(gc, uc)
    for f in ("computed_distances", "base_pops", "upper_hops"):
        assert st[f] == su[f], f
        if su[f] == tot[f]:
            assert st[f] == tot[f], f
    assert st["full_rows_read"] < st["computed_distances"]  # the screen ran (d >= 256: 1 KB rows)
    assert su["full_rows_read"] == su["computed_distances"]


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("kind", ["structured", "zero_mean", "huge_coord", "offset", "near_dup", "tiny", "huge", "zeros",
                                  "nonfinite"])
def test_screen_on_off_bit_identical(eng, monkeypatch, metric, kind):
    X, Q = _data(kind, 3000, 100, 320, seed=5)
    g = eng.Index(320, metric, "f32", M=16, efc=64, ef=64)
    g.add_batch(np.arange(len(X), dtype=np.uint64), X)
    out = {}
    for knob in ("0", "1"):
        monkeypatch.setenv("LB200_SEARCH_SCREEN", knob)
        k, dd, c = g.search_batch(Q, 10, ef=96)
        out[knob] = (k, dd, c, g.last_stats())
    k0, d0, c0, s0 = out["0"]
    k1, d1, c1, s1 = out["1"]
    assert np.array_equal(k0, k1)
    assert np.array_equal(d0.view(np.uint32), d1.view(np.uint32))
    assert np.array_equal(c0, c1)
    for f in ("computed_distances", "base_pops", "upper_hops", "limbo_overflows"):
        assert s0[f] == s1[f], f
    assert s0["full_rows_read"] == s0["computed_distances"]
    if kind in ("structured", "zero_mean"):
        assert s1["full_rows_read"] < s0["full_rows_read"]
        assert s1["algorithmic_bytes"] < s0["algorithmic_bytes"]


def test_screen_survives_growth_and_reload(eng, monkeypatch):
    """The companion is written for every producer of rows: added batches, capacity growth, and load_buffer."""
    X = structured(4000, 384, seed=21)
    Q = structured(64, 384, seed=22)
    g = eng.Index(384, "cos", "f32", M=16, efc=64, ef=64)
    for lo in range(0, 4000, 700):  # several adds, each may grow the capacity
        g.add_batch(np.arange(lo, min(lo + 700, 4000), dtype=np.uint64), X[lo:lo + 700])
    h = eng.Index(384, "cos", "f32", M=16, efc=64, ef=64)
    h.load_buffer(g.save_buffer())
    res = []
    for idx in (g, h):
        for knob in ("0", "1"):
            monkeypatch.setenv("LB200_SEARCH_SCREEN", knob)
            k, dd, c = idx.search_batch(Q, 10)
            res.append((k, dd.view(np.uint32), idx.last_stats()))
    for k, dd, st in res[1:]:
        assert np.array_equal(k, res[0][0]) and np.array_equal(dd, res[0][1])
        assert st["computed_distances"] == res[0][2]["computed_distances"]
    assert res[1][2]["full_rows_read"] < res[1][2]["computed_distances"]
    assert res[3][2]["full_rows_read"] < res[3][2]["computed_distances"]
