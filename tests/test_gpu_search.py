"""GPU parity: the CUDA search path (through the C ABI) against the oracle ON THE SAME GRAPH.

The graph is built by the CPU oracle (hnsw_oracle.c, itself pinned byte-for-byte against the
reference), serialised in the usearch/lantern file format and loaded with lb200_load_buffer --
exactly how Lantern's scan path hands an index to usearch (scan.c:99-110)."""
import numpy as np
import pytest

from util import build_port_index, compare_results, structured

pytestmark = pytest.mark.gpu


def _roundtrip(eng, port, X, Q, metric, quant, M, efc, ef, k, exact_ids=True):
    pidx = build_port_index(port, X, metric, quant, M=M, efc=efc, ef=ef)
    buf = pidx.save_buffer()
    dim = X.shape[1] * 8 if X.dtype == np.uint8 else X.shape[1]
    g = eng.Index(dim, metric, quant, M=M, efc=efc, ef=ef)
    g.load_buffer(buf)
    assert g.size() == len(X)
    gk, gd, gc = g.search_batch(Q, k)
    pk, pd, pc, tot = pidx.search_batch(Q, k)
    assert np.array_equal(gc.astype(np.int64), pc)
    st = g.last_stats()
    return gk, gd, pk, pd, st, tot, g, pidx


def test_small_world_cube(eng, port):
    cube = np.array([[0, 0, 0], [0, 0, 1], [0, 1, 0], [0, 1, 1], [1, 0, 0], [1, 0, 1], [1, 1, 0], [1, 1, 1]], np.float32)
    Q = np.array([[0, 1, 0]], np.float32)
    gk, gd, pk, pd, st, tot, g, p = _roundtrip(eng, port, cube, Q, "l2sq", "f32", 2, 128, 4, 8)
    assert np.array_equal(gd[0], np.array([0, 1, 1, 1, 2, 2, 2, 3], np.float32))
    assert np.array_equal(np.sort(gk[0]), np.arange(1, 9))
    assert gk[0][0] == 3  # vertex 010


@pytest.mark.parametrize("metric,quant,d", [("l2sq", "f32", 64), ("cos", "f32", 96), ("l2sq", "f32", 768), ("cos", "f32", 100),
                                            ("l2sq", "f16", 128), ("cos", "f16", 72), ("l2sq", "i8", 128), ("cos", "i8", 80),
                                            ("l2sq", "f32", 3), ("l2sq", "f32", 1536)])
def test_same_graph_same_ids(eng, port, metric, quant, d):
    n = 3000 if d <= 768 else 1500
    X = structured(n, d, seed=7)
    Q = structured(200, d, seed=8)
    if quant == "i8":
        X, Q = X * 0.3, Q * 0.3
    gk, gd, pk, pd, st, tot, g, p = _roundtrip(eng, port, X, Q, metric, quant, 16, 128, 64, 10)
    assert np.allclose(gd, pd, rtol=1e-5, atol=1e-6), np.abs(gd - pd).max()
    exact, ok = compare_results(gk, gd, pk, pd)
    assert ok == len(Q), (exact, ok)
    assert exact >= 0.97 * len(Q), exact
    # work counters are the reference's own (index.hpp:2726): identical decisions -> identical counts
    if exact == len(Q):
        assert st["computed_distances"] == tot["computed_distances"]
        assert st["base_pops"] == tot["base_pops"]
        assert st["upper_hops"] == tot["upper_hops"]


def test_integer_data_ties(eng, port):
    """Integer-valued vectors: every fp32 sum is exact whatever the order, but exact distance TIES are frequent;
    only the order in which equal-distance candidates leave the queue may differ (SURVEY App. A.7)."""
    rng = np.random.default_rng(3)
    X = rng.integers(-8, 9, (4000, 48)).astype(np.float32)
    Q = rng.integers(-8, 9, (300, 48)).astype(np.float32)
    gk, gd, pk, pd, st, tot, g, p = _roundtrip(eng, port, X, Q, "l2sq", "f32", 8, 64, 40, 10)
    assert np.array_equal(gd[:, 0], pd[:, 0])
    assert np.mean(gd == pd) > 0.98
    exact, ok = compare_results(gk, gd, pk, pd)
    assert exact >= 0.9 * len(Q)


def test_hamming_bits(eng, port):
    rng = np.random.default_rng(5)
    protos = rng.integers(0, 256, (16, 96), dtype=np.uint8)
    def gen(n, seed):
        r = np.random.default_rng(seed)
        base = protos[r.integers(0, 16, n)]
        flips = (r.random((n, 96 * 8)) < 0.1)
        return base ^ np.packbits(flips, axis=1)
    X, Q = gen(3000, 1), gen(100, 2)
    gk, gd, pk, pd, st, tot, g, p = _roundtrip(eng, port, X, Q, "hamming", "b1", 16, 128, 64, 10)
    # heavy ties: against the reference's heap order only the distance profile is comparable ...
    assert np.array_equal(gd[:, 0], pd[:, 0])
    assert np.mean(gd == pd) > 0.98
    # ... but against the oracle run with the engine's own tie order (hnsw_oracle.c beam_engine_order) the ids are
    # IDENTICAL: exact distance ties are the only reason ids ever differ from the reference
    p.set_engine_order(True)
    ek, ed, _, etot = p.search_batch(Q, 10)
    assert np.array_equal(gk, ek) and np.array_equal(gd, ed)
    assert st["computed_distances"] == etot["computed_distances"]
    assert st["limbo_overflows"] == 0  # the 64-entry tie buffer never overflowed: no expansion of the reference was skipped


def test_k_larger_than_ef_and_small_index(eng, port):
    X = structured(50, 32, seed=1)
    Q = structured(20, 32, seed=2)
    gk, gd, pk, pd, st, tot, g, p = _roundtrip(eng, port, X, Q, "l2sq", "f32", 4, 16, 8, 40)  # expansion = max(ef,k)
    exact, ok = compare_results(gk, gd, pk, pd)
    assert ok == len(Q)
    k1, d1 = g.search(Q[0], 5, ef=100)  # single-query entry point, ef honoured
    k2, d2, _ = p.search(Q[0], 5, ef=100)
    assert np.array_equal(k1, k2)


def test_exhaustive_ef_matches_brute_force(eng, port):
    """ef -> infinity: graph search with ef >= N equals brute force (bit-exact ids) on a connected graph."""
    X = structured(1200, 40, seed=11)
    Q = structured(50, 40, seed=12)
    pidx = build_port_index(port, X, "l2sq", "f32", M=16, efc=128, ef=1200)
    g = eng.Index(40, "l2sq", "f32", M=16, efc=128, ef=1200)
    g.load_buffer(pidx.save_buffer())
    gk, gd, _ = g.search_batch(Q, 10)
    bk, bd = eng.exact_search(X, Q, 10, "l2sq")
    assert np.array_equal(gk, bk + 1)  # keys are offset+1
    assert np.allclose(gd, bd, rtol=1e-5)


def test_save_load_roundtrip_bytes(eng, port):
    X = structured(700, 24, seed=21)
    pidx = build_port_index(port, X, "cos", "f32", M=6, efc=40, ef=20)
    buf = pidx.save_buffer()
    g = eng.Index(24, "cos", "f32", M=6, efc=40, ef=20)
    g.load_buffer(buf)
    out = g.save_buffer()
    assert len(out) == len(buf) and np.array_equal(out, buf)


def test_continue_search_streaming(eng, port):
    """scan.c:240-292: first k = init_k, then continue_search with doubled k; no key may be returned twice and the
    concatenation must be ascending and equal to one big search."""
    import ctypes as C
    X = structured(1500, 24, seed=31)
    pidx = build_port_index(port, X, "l2sq", "f32", M=8, efc=64, ef=64)
    g = eng.Index(24, "l2sq", "f32", M=8, efc=64, ef=64)
    g.load_buffer(pidx.save_buffer())
    q = structured(1, 24, seed=32)[0]
    L = eng.lib()
    got_k, got_d = [], []
    k = 10
    cont = False
    for _ in range(4):
        keys, dists = np.zeros(k, np.uint64), np.zeros(k, np.float32)
        err = C.c_char_p()
        n = L.lb200_search_ef(g.h, q.ctypes.data, 1, k, 0, cont, keys.ctypes.data, dists.ctypes.data, C.byref(err))
        assert not err.value
        got_k += list(keys[:n]); got_d += list(dists[:n])
        cont, k = True, k * 2
    assert len(got_k) == 10 + 20 + 40 + 80 and len(set(got_k)) == len(got_k)  # never a row twice
    # each call's slice is ascending; across calls a wider beam may surface closer rows later (approximate search)
    pos = 0
    for n in (10, 20, 40, 80):
        assert all(a <= b for a, b in zip(got_d[pos:pos + n], got_d[pos + 1:pos + n]))
        pos += n
    allk, alld = g.search(q, 150, ef=150)
    assert len(set(allk) & set(got_k)) >= 140  # the stream covers (nearly) the same 150 rows as one wide search
    # a different query cannot be "continued"
    err = C.c_char_p()
    other = structured(1, 24, seed=33)[0]
    L.lb200_search_ef(g.h, other.ctypes.data, 1, 5, 0, True, keys.ctypes.data, dists.ctypes.data, C.byref(err))
    assert err.value and b"continue_search" in err.value


def test_wide_beam_touched_list_overflow_and_large_k(eng, port):
    """A beam that visits more nodes than the per-CTA un-visit log holds exercises the full-bitmap clear; k = 500 the
    large top list."""
    rng = np.random.default_rng(41)
    X = rng.standard_normal((30000, 8)).astype(np.float32)
    Q = rng.standard_normal((24, 8)).astype(np.float32)
    pidx = build_port_index(port, X, "l2sq", "f32", M=8, efc=32, ef=32)
    g = eng.Index(8, "l2sq", "f32", M=8, efc=32, ef=32)
    g.load_buffer(pidx.save_buffer())
    g.set_option("touched_cap", 1024)
    for rep in range(2):  # second pass: the bitmaps must have been cleaned by the first
        gk, gd, gc = g.search_batch(Q, 500, ef=4000)
        st = g.last_stats()
        assert st["computed_distances"] / len(Q) > 1024  # the overflow path really ran
        pk, pd, pc, _ = pidx.search_batch(Q, 500, ef=4000)
        assert np.array_equal(gc.astype(np.int64), pc) and np.allclose(gd, pd, rtol=1e-5, atol=1e-6)
        assert np.mean(gk == pk) > 0.995
    gk2, gd2, _ = g.search_batch(Q, 10)  # and a normal search afterwards still agrees with the oracle
    pk2, pd2, _, _ = pidx.search_batch(Q, 10)
    assert np.array_equal(gk2, pk2)


def test_high_connectivity_graph(eng, port):
    X = structured(1500, 24, seed=51)
    Q = structured(50, 24, seed=52)
    pidx = build_port_index(port, X, "cos", "f32", M=64, efc=96, ef=80)  # M0 = 128: adjacency spans several 32-id chunks
    g = eng.Index(24, "cos", "f32", M=64, efc=96, ef=80)
    g.load_buffer(pidx.save_buffer())
    gk, gd, _ = g.search_batch(Q, 20)
    pk, pd, _, _ = pidx.search_batch(Q, 20)
    assert np.allclose(gd, pd, rtol=1e-5, atol=1e-6) and np.mean(gk == pk) > 0.99


@pytest.mark.parametrize("metric,quant,d", [("l2sq", "f32", 64), ("cos", "f32", 768), ("hamming", "b1", 6144), ("cos", "i8", 80), ("l2sq", "f16", 128)])
def test_warp_per_query_kernel_equals_cta_kernel(eng, metric, quant, d):
    """The one-warp-per-query search kernel (csrc/group.cu with one rank; the narrow-row path and the multi-GPU kernel) against
    the one-CTA-per-query kernel (csrc/search.cu) on the same graph: same ids, bit-identical distances, same work counters."""
    rng = np.random.default_rng(4)
    n = 4000
    if quant == "b1":
        protos = rng.integers(0, 256, (16, d // 8), dtype=np.uint8)
        X = protos[rng.integers(0, 16, n)] ^ np.packbits(rng.random((n, d)) < 0.1, axis=1)
        Q = protos[rng.integers(0, 16, 200)] ^ np.packbits(rng.random((200, d)) < 0.1, axis=1)
    else:
        X, Q = structured(n, d, seed=7), structured(200, d, seed=8)
        if quant == "i8":
            X, Q = X * 0.3, Q * 0.3
    g = eng.Index(d, metric, quant, M=16, efc=64, ef=48)
    g.reserve(n)
    g.add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
    g.build()
    for k, ef in ((10, 48), (100, 300), (1, 1)):
        g.set_option("search_kernel", 1)
        k1, d1, c1 = g.search_batch(Q, k, ef)
        s1 = g.last_stats()
        g.set_option("search_kernel", 2)
        k2, d2, c2 = g.search_batch(Q, k, ef)
        s2 = g.last_stats()
        assert np.array_equal(k1, k2) and np.array_equal(d1.view(np.uint32), d2.view(np.uint32)) and np.array_equal(c1, c2)
        assert (s1["computed_distances"], s1["base_pops"], s1["upper_hops"]) == (s2["computed_distances"], s2["base_pops"], s2["upper_hops"])
