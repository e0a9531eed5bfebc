"""The projected screen in the one-warp-per-query search kernel (csrc/group.cu, one rank; DESIGN.md 4.1).

The warp kernel's owner screens a level-0 round's candidates with the same records, pre-pass and bound as the one-CTA-per-query
kernel (PScreenEval), so on one graph both kernels must return the same keys, distance bits and counts and report the same
work: computed distances (screened candidates included), full rows read, screen kind and width, algorithmic bytes."""
import numpy as np
import pytest

from test_gpu_search_screen import _data
from util import structured

pytestmark = pytest.mark.gpu

FIELDS = ("computed_distances", "base_pops", "upper_hops", "limbo_overflows", "full_rows_read", "screen_kind", "screen_dims",
          "algorithmic_bytes")
PAIRS = ((10, 64), (10, 128), (100, 300), (1, 1))  # (k, ef)


def _both(g, Q, k, ef):
    out = []
    for kern in (1, 2):
        g.set_option("search_kernel", kern)
        keys, dists, counts = g.search_batch(Q, k, ef)
        out.append((keys, dists, counts, g.last_stats()))
    g.set_option("search_kernel", 0)
    return out


def _assert_same(out, what):
    (k1, d1, c1, s1), (k2, d2, c2, s2) = out
    assert s1["search_kernel"] == 1 and s2["search_kernel"] == 2, what
    assert np.array_equal(k1, k2), what
    assert np.array_equal(d1.view(np.uint32), d2.view(np.uint32)), what
    assert np.array_equal(c1, c2), what
    # the warp kernel screens with the projected screen only; where the CTA kernel ran the int8 one it reads every row
    fields = FIELDS if s1["screen_kind"] != 1 else FIELDS[:4]
    for f in fields:
        assert s1[f] == s2[f], (what, f, s1[f], s2[f])
    if s1["screen_kind"] == 1:
        assert s2["screen_kind"] == 0 and s2["full_rows_read"] == s2["computed_distances"], what
    assert s1["owner_cycles_produce"] == 0 and s2["owner_cycles_produce"] > 0, what
    if s2["screen_kind"] == 2 and s2["full_rows_read"] < s2["computed_distances"]:
        assert s2["owner_cycles_screen"] > 0, what
    return s2


def _index(eng, X, metric, M, ef=64):
    g = eng.Index(X.shape[1], metric, "f32", M=M, efc=64, ef=ef)
    g.reserve(len(X))
    g.add_batch(np.arange(1, len(X) + 1, dtype=np.uint64), X)
    g.build()
    return g


def _sweep(g, Q, monkeypatch, what):
    for screen in ("2", None):
        if screen is None:
            monkeypatch.delenv("LB200_SEARCH_SCREEN", raising=False)
        else:
            monkeypatch.setenv("LB200_SEARCH_SCREEN", screen)
        for k, ef in PAIRS:
            s2 = _assert_same(_both(g, Q, k, ef), (what, screen, k, ef))
            if screen == "2":
                assert s2["screen_kind"] == 2
    return s2


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("d,M", [(320, 16), (768, 32), (1536, 16), (320, 64)])  # NQ 3, 6, 12; M0 32, 64 (two halves), 128
def test_warp_screen_equals_cta_kernel(eng, monkeypatch, metric, d, M):
    X, Q = structured(3000, d, seed=d + M), structured(150, d, seed=d + M + 1)
    g = _index(eng, X, metric, M)
    _sweep(g, Q, monkeypatch, (d, M))
    monkeypatch.setenv("LB200_SEARCH_SCREEN", "2")
    g.set_option("search_kernel", 2)
    g.search_batch(Q, 10, 64)
    st = g.last_stats()
    assert st["full_rows_read"] < st["computed_distances"]  # the screen rejects candidates in the warp kernel too
    g.close()


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
def test_warp_screen_wide_records(eng, monkeypatch, metric):
    """an 80-dimensional latent needs k > 48: 128-byte records"""
    X, Q = structured(3000, 320, seed=3, latent=80), structured(150, 320, seed=4, latent=80)
    g = _index(eng, X, metric, 16)
    monkeypatch.setenv("LB200_SEARCH_SCREEN", "2")
    s2 = _assert_same(_both(g, Q, 10, 64), "wide")
    assert s2["screen_dims"] > 48, s2["screen_dims"]
    _sweep(g, Q, monkeypatch, "wide")
    g.close()


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("kind", ["structured", "zero_mean", "near_dup", "zeros", "nonfinite"])
def test_warp_screen_data_kinds(eng, monkeypatch, metric, kind):
    X, Q = _data(kind, 3000, 100, 320, seed=5)
    g = eng.Index(320, metric, "f32", M=16, efc=64, ef=64)
    g.add_batch(np.arange(len(X), dtype=np.uint64), X)
    monkeypatch.setenv("LB200_SEARCH_SCREEN", "2")
    for k, ef in ((10, 96), (1, 1)):
        _assert_same(_both(g, Q, k, ef), (kind, k, ef))
    g.close()


def test_warp_screen_touched_overflow_and_clean_bitmaps(eng, monkeypatch):
    """a beam that overflows a small un-visit log clears the whole bitmap; batches back to back start from clean bitmaps"""
    X = structured(3000, 320, seed=9)
    Q1, Q2 = structured(120, 320, seed=10), structured(120, 320, seed=11)
    g = _index(eng, X, "cos", 16)
    monkeypatch.setenv("LB200_SEARCH_SCREEN", "2")
    ref = _both(g, Q1, 10, 300)
    _assert_same(ref, "ref")
    g.set_option("touched_cap", 32)
    small = _both(g, Q1, 10, 300)
    _assert_same(small, "touched_cap")
    assert np.array_equal(small[1][0], ref[1][0]) and np.array_equal(small[1][1].view(np.uint32), ref[1][1].view(np.uint32))
    g.set_option("touched_cap", 16384)
    g.set_option("search_kernel", 2)
    a1 = g.search_batch(Q1, 10, 128)
    g.search_batch(Q2, 10, 128)
    a2 = g.search_batch(Q1, 10, 128)
    assert all(np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x, y.view(np.uint32) if y.dtype == np.float32 else y)
               for x, y in zip(a1, a2))
    g.close()


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
def test_automatic_choice_keeps_cta_kernel(eng, monkeypatch, metric):
    """unset, a projected-screen index runs one CTA per query for small and large batches alike (the warp kernel measured
    slower with the screen too, DESIGN.md 6); the warp kernel, forced, returns the same"""
    monkeypatch.delenv("LB200_SEARCH_SCREEN", raising=False)
    X = structured(20000, 320, seed=31)
    Q = structured(8192, 320, seed=33)  # >= 2 x 16 CTAs/SM x 132 SMs
    g = _index(eng, X, metric, 16)
    for nq in (64, 8192):
        keys, dists, _ = g.search_batch(Q[:nq], 10)
        st = g.last_stats()
        assert st["screen_kind"] == 2 and st["search_kernel"] == 1, (nq, st)
    g.set_option("search_kernel", 2)
    wk, wd, _ = g.search_batch(Q, 10)
    wst = g.last_stats()
    assert wst["search_kernel"] == 2
    assert np.array_equal(wk, keys) and np.array_equal(wd.view(np.uint32), dists.view(np.uint32))
    for f in FIELDS:
        assert wst[f] == st[f], f
    g.close()


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("screen", ["1", "2"])
def test_screened_round_visited_halves_change_nothing(eng, monkeypatch, metric, screen):
    """the CTA kernel's screened rounds with and without the one-trip 64-wide visited pass (flags bit 8, on by default): the
    same keys, distance bits, counts and counters"""
    X, Q = structured(3000, 320, seed=41), structured(150, 320, seed=42)
    g = _index(eng, X, metric, 32)  # M0 = 64
    monkeypatch.setenv("LB200_SEARCH_SCREEN", screen)
    out = []
    for flags in ("2", "10", None):
        if flags is None:
            monkeypatch.delenv("LB200_FLAGS", raising=False)
        else:
            monkeypatch.setenv("LB200_FLAGS", flags)
        for k, ef in PAIRS:
            keys, dists, counts = g.search_batch(Q, k, ef)
            st = g.last_stats()
            out.append((flags, k, ef, keys, dists.view(np.uint32), counts, tuple(st[f] for f in FIELDS)))
    ref = {(k, ef): o for o in out if o[0] == "2" for k, ef in [(o[1], o[2])]}
    for o in out:
        r = ref[(o[1], o[2])]
        assert all(np.array_equal(a, b) for a, b in zip(o[3:6], r[3:6])) and o[6] == r[6], (o[0], o[1], o[2])
    g.close()
