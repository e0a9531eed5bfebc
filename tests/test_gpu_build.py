"""GPU parity of the build path (lb200_add* + lb200_build) against the oracle."""
import os

import numpy as np
import pytest

from util import build_port_index, describe_file_difference, recall, structured

pytestmark = pytest.mark.gpu

CUBE = np.array([[0, 0, 0], [0, 0, 1], [0, 1, 0], [0, 1, 1], [1, 0, 0], [1, 0, 1], [1, 1, 0], [1, 1, 1]], np.float32)


def test_small_world_through_add(eng):
    """BASELINE config 1 (small_world 8 x d3, M=2, ef=4) through the reference-facing calls only."""
    g = eng.Index(3, "l2sq", "f32", M=2, efc=128, ef=4)
    g.reserve(8)
    for i, v in enumerate(CUBE):
        g.add(100 + i, v)
    assert g.size() == 8
    k, d = g.search(np.array([0, 1, 0], np.float32), 8)
    assert np.array_equal(d, np.array([0, 1, 1, 1, 2, 2, 2, 3], np.float32))
    assert k[0] == 102 and set(k[1:4]) == {100, 103, 106} and set(k[4:7]) == {101, 104, 107} and k[7] == 105
    k1, d1 = g.search(np.array([0, 1, 0], np.float32), 1)
    assert k1[0] == 102 and d1[0] == 0


@pytest.mark.parametrize("metric,d,M,efc", [("l2sq", 48, 8, 64), ("l2sq", 24, 6, 40), ("cos", 32, 16, 128)])
def test_exact_order_build_is_byte_identical(eng, port, metric, d, M, efc):
    """build_batch=1 == the reference's sequential insertion with the engine's tie order (the oracle's engine-order
    switch, set before adding): same level draws, same lists, same file bytes (integer-valued vectors: fp32 sums are
    order independent; exact ties are frequent and must break identically in the beam, the sorted-list and the heuristic
    code paths)."""
    rng = np.random.default_rng(17)
    n = 1200
    X = rng.integers(-8, 9, (n, d)).astype(np.float32)
    pidx = port.PortIndex(d, metric, "f32", M=M, efc=efc, ef=32)
    pidx.set_engine_order(True)
    pidx.reserve(n)
    for i in range(n):
        pidx.add(i + 1, X[i])
    g = eng.Index(d, metric, "f32", M=M, efc=efc, ef=32)
    g.set_option("build_batch", 1)
    g.reserve(n)
    g.add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
    g.build()
    gb, pb = g.save_buffer(), pidx.save_buffer()
    assert np.array_equal(gb, pb), describe_file_difference(gb, pb, M, d * 4, X, metric, "f32", d, port)


@pytest.mark.parametrize("metric,d,M,efc,batch,lim", [("l2sq", 16, 8, 64, 64, 300), ("l2sq", 48, 8, 64, 64, 8),
                                                      ("cos", 32, 16, 128, 256, 8)])
def test_batched_build_follows_the_cpu_model(eng, port, metric, d, M, efc, batch, lim):
    """The DEFAULT (batched, two-phase) build against its CPU specification, oracle ora_add_batch_engine in the engine's
    tie order: same batch schedule (build_batch / build_ratio), same phase-1 searches against the pre-batch graph, same
    stable request order in phase 2.  Integer coordinates: every distance is an exact fp32 integer (< 2^24) whatever the
    summation order.  In [-300, 300] at d=16 exact ties are rare; in [-8, 8] they are everywhere, and the engine expands
    equal-distance candidates in its own order (DESIGN.md 4.1), which the model reproduces.  The files must be identical."""
    rng = np.random.default_rng(19)
    n = 3000
    X = rng.integers(-lim, lim + 1, (n, d)).astype(np.float32)
    keys = np.arange(1, n + 1, dtype=np.uint64)
    p = port.PortIndex(d, metric, "f32", M=M, efc=efc, ef=32)
    p.set_engine_order(True)
    p.reserve(n)
    p.add_batch_engine(keys, X, batch, 64)
    g = eng.Index(d, metric, "f32", M=M, efc=efc, ef=32)
    g.set_option("build_batch", batch)
    g.set_option("build_ratio", 64)
    g.reserve(n)
    g.add_batch(keys, X)
    g.build()
    gb, pb = g.save_buffer(), p.save_buffer()
    assert np.array_equal(gb, pb), describe_file_difference(gb, pb, M, d * 4, X, metric, "f32", d, port)


def test_batched_build_recall_matches_reference_graph(eng, port):
    """Default (batched) GPU build vs the oracle's sequential build on the same data: recall@10 at the same ef
    within the north_star's +-0.5% window (the reference's own multi-threaded builds vary by about that much)."""
    n, d = 20000, 64
    X = structured(n, d, seed=3)
    Q = structured(500, d, seed=4)
    truth, _ = eng.exact_search(X, Q, 10, "l2sq")
    pidx = build_port_index(port, X, "l2sq", "f32", M=16, efc=128, ef=64)
    pk, _, _, _ = pidx.search_batch(Q, 10)
    r_ref = recall(pk - 1, truth)
    g = eng.Index(d, "l2sq", "f32", M=16, efc=128, ef=64)
    g.reserve(n)
    g.add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
    g.build()
    gk, _, _ = g.search_batch(Q, 10)
    r_gpu = recall(gk - 1, truth)
    print("recall@10 reference-built %.4f  gpu-built %.4f" % (r_ref, r_gpu))
    assert r_gpu >= r_ref - 0.005
    # the GPU-built file loads into the oracle and gives the same answers there (same-graph parity, other direction)
    p2 = port.PortIndex(d, "l2sq", "f32", M=16, efc=128, ef=64)
    p2.reserve(n)
    p2.load_buffer(g.save_buffer())
    k2, d2, _, _ = p2.search_batch(Q[:100], 10)
    assert np.mean(k2 == gk[:100]) > 0.99


def test_incremental_add_after_build(eng, port):
    X = structured(3000, 32, seed=9)
    g = eng.Index(32, "l2sq", "f32", M=8, efc=64, ef=48)
    g.reserve(3000)
    g.add_batch(np.arange(1, 2001, dtype=np.uint64), X[:2000])
    k, d = g.search(X[5], 1)  # triggers the build
    assert k[0] == 6 and d[0] == 0
    g.add_batch(np.arange(2001, 3001, dtype=np.uint64), X[2000:])
    k, d = g.search(X[2500], 1)
    assert k[0] == 2501 and d[0] == 0
    assert g.size() == 3000


def test_hamming_build(eng):
    rng = np.random.default_rng(5)
    protos = rng.integers(0, 256, (16, 96), dtype=np.uint8)
    base = protos[rng.integers(0, 16, 4000)]
    X = base ^ np.packbits(rng.random((4000, 768)) < 0.1, axis=1)
    g = eng.Index(768, "hamming", "b1", M=16, efc=128, ef=64)
    g.reserve(4000)
    g.add_batch(np.arange(1, 4001, dtype=np.uint64), X)
    g.build()
    Q = X[:200]
    gk, gd, _ = g.search_batch(Q, 10)
    truth, td = eng.exact_search(X, Q, 10, "hamming", "b1")
    assert np.array_equal(gd[:, 0], np.zeros(200, np.float32))
    assert np.mean(gd <= td + 1e-6) > 0.9  # distance profile close to exact


@pytest.mark.parametrize("quant,scale", [("f16", 1.0), ("i8", 0.3)])
def test_scalar_quantised_builds(eng, port, quant, scale):
    """quant_bits=16 / 8 storage: the GPU build works in the storage domain like the reference (f32 in, cast on add)."""
    n, d = 6000, 48
    X = structured(n, d, seed=13) * scale
    Q = structured(200, d, seed=14) * scale
    g = eng.Index(d, "cos", quant, M=16, efc=64, ef=64)
    g.reserve(n)
    g.add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
    g.build()
    gk, gd, _ = g.search_batch(Q, 10)
    # ground truth in the same storage domain
    cx, cq = eng.cast(X, quant), eng.cast(Q, quant)
    tk, td = eng.exact_search(cx, cq, 10, "cos", quant, d)
    assert recall(gk - 1, tk) > 0.9
    # the GPU-built file loads into the oracle and gives (nearly) the same answers there
    p = port.PortIndex(d, "cos", quant, M=16, efc=64, ef=64)
    p.reserve(n)
    p.load_buffer(g.save_buffer())
    pk, pd, _, _ = p.search_batch(Q[:60], 10)
    assert np.mean(pk == gk[:60]) > 0.97 and np.allclose(pd, gd[:60], rtol=1e-4, atol=1e-5)


def test_malformed_index_files_are_rejected(eng, port):
    X = structured(300, 16, seed=2)
    pidx = build_port_index(port, X, "l2sq", "f32", M=4, efc=32, ef=16)
    buf = pidx.save_buffer().copy()
    g = eng.Index(16, "l2sq", "f32", M=4, efc=32, ef=16)
    bad = buf.copy(); bad[112:118] = 255  # entry slot far out of range
    with pytest.raises(eng.EngineError, match="entry slot"):
        g.load_buffer(bad)
    bad = buf.copy(); bad[104] = 9  # max_level that no node has
    with pytest.raises(eng.EngineError, match="max_level|level"):
        g.load_buffer(bad)
    with pytest.raises(eng.EngineError, match="truncated"):
        g.load_buffer(buf[:len(buf) // 2])
    g.load_buffer(buf)  # the intact file still loads afterwards
    assert g.size() == 300


def test_row_at_a_time_adds_are_staged(eng):
    """usearch_add from a heap scan (build.c:128): one row per call; rows reach the GPU in blocks, size() counts them."""
    X = structured(5000, 16, seed=61)
    g = eng.Index(16, "l2sq", "f32", M=8, efc=32, ef=32)
    g.reserve(5000)
    for i in range(5000):
        g.add(i + 1, X[i])
    assert g.size() == 5000
    k, d = g.search(X[4999], 1)  # the last, still host-staged row must be findable: search flushes and builds
    assert k[0] == 5000 and d[0] == 0
    buf = g.save_buffer()
    g2 = eng.Index(16, "l2sq", "f32", M=8, efc=32, ef=32)
    g2.load_buffer(buf)
    assert g2.size() == 5000
