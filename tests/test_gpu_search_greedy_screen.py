"""The screen of the greedy descent (walk.cuh WalkerT::greedy, group.cu's owner; DESIGN.md 4.1).

A greedy pass over an upper-level list takes the first candidate, in stored order, whose distance is the minimum and strictly
below cur_d.  A candidate with lb >= cur_d has d >= cur_d and can never be taken, so screened searches reject it without
reading its row.  Graphs of small M have many levels, so the descent is a large share of the walk there; the searches must
return exactly what the unscreened search returns, with the same work counters, in both search kernels."""
import numpy as np
import pytest

from test_gpu_search_screen import _data, _oracle_pair
from util import compare_results, structured

pytestmark = pytest.mark.gpu

SAME = ("computed_distances", "base_pops", "upper_hops", "limbo_overflows")
KERNEL_SAME = SAME + ("full_rows_read", "screen_kind", "screen_dims", "algorithmic_bytes")


def _runs(g, Q, monkeypatch, k, ef, knobs=("0", "1", "2")):
    """(knob, kernel) -> keys, distance bits, counts, stats"""
    out = {}
    for knob in knobs:
        monkeypatch.setenv("LB200_SEARCH_SCREEN", knob)
        for kern in (1, 2):
            g.set_option("search_kernel", kern)
            keys, dists, counts = g.search_batch(Q, k, ef)
            out[(knob, kern)] = (keys, dists.view(np.uint32), counts, g.last_stats())
    g.set_option("search_kernel", 0)
    return out


def _assert_same(out, what):
    k0, d0, c0, s0 = out[("0", 1)]
    for (knob, kern), (k, d, c, s) in out.items():
        w = (what, knob, kern)
        assert s["search_kernel"] == kern, w
        assert np.array_equal(k0, k) and np.array_equal(d0, d) and np.array_equal(c0, c), w
        for f in SAME:
            assert s0[f] == s[f], (w, f, s0[f], s[f])
    for knob in ("0", "2"):  # the warp kernel runs the projected screen or none: the same rows read as the CTA kernel's
        s1, s2 = out[(knob, 1)][3], out[(knob, 2)][3]
        for f in KERNEL_SAME:
            assert s1[f] == s2[f], (what, knob, f, s1[f], s2[f])


def _index(eng, X, metric, M, ef):
    g = eng.Index(X.shape[1], metric, "f32", M=M, efc=64, ef=ef)
    g.reserve(len(X))
    g.add_batch(np.arange(1, len(X) + 1, dtype=np.uint64), X)
    g.build()
    return g


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("kind", ["structured", "zero_mean", "huge_coord", "near_dup", "zeros", "nonfinite"])
@pytest.mark.parametrize("d,M,n", [(320, 4, 6000), (768, 8, 3000), (320, 16, 8000)])
def test_descent_screen_changes_nothing(eng, monkeypatch, metric, kind, d, M, n):
    """off, int8 and projected screens in both kernels on one deep graph: the same keys, distance bits, counts and counters.
    (Fewer full rows than unscreened is asserted too, but the level-0 screen alone gives that; the descent's own rejects are
    isolated by test_descent_screened_when_level0_never_fills.)"""
    X, Q = _data(kind, n, 100, d, seed=d + M)
    g = _index(eng, X, metric, M, 64)
    for k, ef in ((10, 64), (1, 1)):
        out = _runs(g, Q, monkeypatch, k, ef)
        _assert_same(out, (k, ef))
        if kind == "structured":
            assert out[("2", 1)][3]["full_rows_read"] < out[("0", 1)][3]["full_rows_read"], (k, ef)
    g.close()


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
def test_descent_screened_when_level0_never_fills(eng, monkeypatch, metric):
    """ef above the number of rows: the level-0 top list never fills, so no level-0 round is screened and every row a
    screened search does not read is a descent candidate"""
    X, Q = structured(1200, 320, seed=51), structured(100, 320, seed=52)
    g = _index(eng, X, metric, 4, 1536)
    out = _runs(g, Q, monkeypatch, 10, 1536)
    _assert_same(out, "ef > n")
    assert out[("0", 1)][3]["full_rows_read"] == out[("0", 1)][3]["computed_distances"]
    for key in (("1", 1), ("2", 1), ("2", 2)):
        st = out[key][3]
        assert st["full_rows_read"] < st["computed_distances"], (key, st["full_rows_read"], st["computed_distances"])
    g.close()


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("d,M", [(320, 4), (768, 8)])
def test_descent_screen_matches_oracle(eng, port, monkeypatch, metric, d, M):
    """on an oracle-built deep graph the screened searches return the oracle's results, and its counters wherever the
    unscreened kernel's equal them (the two sum distances in different orders).  The full_rows_read check here holds through
    the level-0 screen alone."""
    X = structured(3000, d, seed=61)
    Q = structured(200, d, seed=62)
    pidx, g = _oracle_pair(eng, port, X, metric, M, 64)
    out = _runs(g, Q, monkeypatch, 10, 64)
    _assert_same(out, "oracle")
    pk, pd, pc, tot = pidx.search_batch(Q, 10)
    for key in (("1", 1), ("2", 1), ("2", 2)):
        gk, gd, gc, st = out[key]
        gd = gd.view(np.float32)
        assert np.array_equal(gc.astype(np.int64), pc), key
        assert np.allclose(gd, pd, rtol=1e-5, atol=1e-6), (key, np.abs(gd - pd).max())
        exact, ok = compare_results(gk, gd, pk, pd)
        assert ok == len(Q), (key, exact, ok)
        assert exact >= 0.97 * len(Q), (key, exact)
        for f in ("computed_distances", "base_pops", "upper_hops"):
            if out[("0", 1)][3][f] == tot[f]:
                assert st[f] == tot[f], (key, f)
        assert st["full_rows_read"] < st["computed_distances"], key
    g.close()
