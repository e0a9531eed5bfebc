"""The plain-C restatement against the compiled reference itself (skipped where oracle/_ref is absent)."""
import struct

import numpy as np
import pytest


def trim(buf, stored_bytes=None):
    """The reference's save_buffer may leave slack after the last node; pq nodes carry `num_subvectors` code bytes instead
    of the header's vector_size_bytes."""
    n, M, M0 = struct.unpack_from("<QQQ", buf, 80)
    vsz, = struct.unpack_from("<Q", buf, 120)
    if stored_bytes is not None:
        vsz = stored_bytes
    off, b = 136, bytes(buf)
    for _ in range(n):
        lvl, = struct.unpack_from("<h", b, off + 8)
        off += 10 + 4 + 6 * M0 + lvl * (4 + 6 * M) + vsz
    return np.array(buf[:off])


@pytest.mark.parametrize("n,d,M,efc,ef,metric", [(1500, 32, 16, 128, 64, "l2sq"), (2000, 24, 6, 40, 20, "l2sq"), (1200, 48, 16, 96, 50, "cos")])
def test_build_and_search_byte_exact_on_integer_data(port, ref, n, d, M, efc, ef, metric):
    rng = np.random.default_rng(n)
    X = rng.integers(-8, 9, (n, d)).astype(np.float32)
    Q = rng.integers(-8, 9, (150, d)).astype(np.float32)
    r = ref.RefIndex(d, metric, M=M, efc=efc, ef=ef)
    p = port.PortIndex(d, metric, M=M, efc=efc, ef=ef)
    r.reserve(n), p.reserve(n)
    for i in range(n):
        r.add(i + 1, X[i]), p.add(i + 1, X[i])
    assert np.array_equal(trim(r.save_buffer()), p.save_buffer())
    for q in Q:
        rk, rd = r.search(q, 10)
        pk, pd, st = p.search(q, 10)
        assert np.array_equal(rk, pk) and np.array_equal(rd, pd)


def test_counters_match_reference(port, ref):
    """computed_distances / visited_members (index.hpp:2726-2727) -- the quantity the roofline's algorithmic bytes use."""
    import ctypes as C
    rng = np.random.default_rng(5)
    X = rng.integers(-8, 9, (2000, 32)).astype(np.float32)
    r = ref.RefIndex(32, "l2sq", M=16, efc=128, ef=64)
    p = port.PortIndex(32, "l2sq", M=16, efc=128, ef=64)
    r.reserve(2000), p.reserve(2000)
    for i in range(2000):
        r.add(i + 1, X[i]), p.add(i + 1, X[i])
    L = ref.lib()
    for q in rng.integers(-8, 9, (50, 32)).astype(np.float32):
        keys, dists = np.zeros(10, np.uint64), np.zeros(10, np.float32)
        comp, vis = C.c_uint64(), C.c_uint64()
        L.refx_search_stats(r.h, q.ctypes.data, 10, keys.ctypes.data, dists.ctypes.data, C.byref(comp), C.byref(vis))
        pk, pd, st = p.search(q, 10)
        assert st.computed_distances == comp.value and st.visited_members == vis.value


def test_float_data_ids_and_tolerance(port, ref):
    rng = np.random.default_rng(11)
    X = rng.standard_normal((1500, 64)).astype(np.float32)
    r = ref.RefIndex(64, "cos", M=16, efc=128, ef=64)
    r.reserve(1500)
    for i in range(1500):
        r.add(i + 1, X[i])
    p = port.PortIndex(64, "cos", M=16, efc=128, ef=64)
    p.reserve(1500)
    p.load_buffer(trim(r.save_buffer()))  # same graph, the reference's own bytes
    same = 0
    for q in rng.standard_normal((200, 64)).astype(np.float32):
        rk, rd = r.search(q, 10)
        pk, pd, _ = p.search(q, 10)
        assert np.allclose(rd, pd, rtol=1e-5, atol=1e-6)
        same += np.array_equal(rk, pk)
    assert same >= 198


def test_pq_128_centroid_quirk(port, ref):
    """codebook_t::compress never picks centroids >= 128 (signed char loop, lantern_storage.hpp:123)."""
    rng = np.random.default_rng(2)
    d, nsub, ncent = 16, 4, 256
    cb = rng.standard_normal((ncent, d)).astype(np.float32)
    X = rng.standard_normal((300, d)).astype(np.float32)
    r = ref.RefIndex(d, "l2sq", M=8, efc=32, ef=300, pq=True, num_centroids=ncent, num_subvectors=nsub, codebook=cb)
    r.reserve(300)
    for i in range(300):
        r.add(i + 1, X[i])
    codes = port.pq_compress(cb, X, nsub, compat128=True)
    assert codes.max() < 128
    dec = port.pq_decompress(cb, codes)
    q = rng.standard_normal(d).astype(np.float32)
    rk, rd = r.search(q, 300)  # ef = N -> (almost) every node, distances = raw query vs decoded candidate
    mine = ((dec[rk.astype(int) - 1] - q) ** 2).sum(1)
    assert np.allclose(mine, rd, rtol=1e-5, atol=1e-6)
    full = port.pq_compress(cb, X, nsub, compat128=False)
    assert (full >= 128).any()


def test_engine_tie_order_mode_equals_reference_without_ties(port):
    """The oracle's model of the CUDA engine's queue discipline is the reference's algorithm whenever distances are distinct
    (ids AND work counters identical); with exact ties only equal-distance order may differ (same distance profile)."""
    import sys, os
    sys.path.insert(0, os.path.dirname(__file__))
    from util import build_port_index, structured
    X, Q = structured(2500, 24, seed=3), structured(150, 24, seed=4)
    p = build_port_index(port, X, "cos", "f32", M=12, efc=64, ef=40)
    k1, d1, c1, t1 = p.search_batch(Q, 10)
    p.set_engine_order(True)
    k2, d2, c2, t2 = p.search_batch(Q, 10)
    assert np.array_equal(k1, k2) and np.array_equal(d1, d2) and t1 == t2
    rng = np.random.default_rng(9)
    Xi = rng.integers(-3, 4, (2000, 12)).astype(np.float32)  # integer data: ties everywhere
    Qi = rng.integers(-3, 4, (100, 12)).astype(np.float32)
    p = build_port_index(port, Xi, "l2sq", "f32", M=8, efc=48, ef=24)
    k1, d1, _, _ = p.search_batch(Qi, 10)
    p.set_engine_order(True)
    k2, d2, _, _ = p.search_batch(Qi, 10)
    assert np.mean(d1 == d2) > 0.97


def test_property_port_equals_reference_on_random_small_configs(port, ref):
    """Property test (hypothesis): for random (N, d, M, ef_construction, ef, metric) and integer-valued data the
    restatement and the compiled reference write the same index file and return the same ids and distances."""
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=20, deadline=None)
    @given(n=st.integers(2, 300), d=st.integers(1, 20), M=st.sampled_from([2, 3, 4, 8, 16]), efc=st.integers(4, 64),
           ef=st.integers(1, 48), metric=st.sampled_from(["l2sq", "cos"]), seed=st.integers(0, 10_000))
    def check(n, d, M, efc, ef, metric, seed):
        rng = np.random.default_rng(seed)
        X = rng.integers(-5, 6, (n, d)).astype(np.float32)
        r = ref.RefIndex(d, metric, M=M, efc=efc, ef=ef)
        p = port.PortIndex(d, metric, M=M, efc=efc, ef=ef)
        r.reserve(n), p.reserve(n)
        for i in range(n):
            r.add(i + 1, X[i]), p.add(i + 1, X[i])
        assert np.array_equal(trim(r.save_buffer()), p.save_buffer())
        for q in rng.integers(-5, 6, (10, d)).astype(np.float32):
            k = int(rng.integers(1, 12))
            rk, rd = r.search(q, k)
            pk, pd, _ = p.search(q, k)
            assert np.array_equal(rk, pk) and np.array_equal(rd, pd)

    check()


def test_property_scalar_kinds_bits_and_pq(port, ref):
    """Same property for the storage variants: f16 / i8 scalar quantisation (f32 in, cast on add), packed bits with the
    hamming metric, and pq storage with a random codebook (stored side decoded, value side raw)."""
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=20, deadline=None)
    @given(n=st.integers(2, 200), sub=st.integers(1, 6), M=st.sampled_from([2, 4, 8]), efc=st.integers(4, 48),
           ef=st.integers(1, 32), variant=st.sampled_from(["f16", "i8", "b1", "pq"]), metric=st.sampled_from(["l2sq", "cos"]),
           seed=st.integers(0, 10_000))
    def check(n, sub, M, efc, ef, variant, metric, seed):
        rng = np.random.default_rng(seed)
        kw, quant, d = {}, "f32", 4 * sub
        if variant == "b1":
            metric, quant, d = "hamming", "b1", 32 * sub
            X = rng.integers(0, 256, (n, d // 8), dtype=np.uint8)
            Q = rng.integers(0, 256, (8, d // 8), dtype=np.uint8)
        else:
            # small multiples of 1/4: exact in f16, and |x| * 100 stays an integer below the i8 clamp for the small ones
            X = (rng.integers(-4, 5, (n, d)) / 4.0).astype(np.float32)
            Q = (rng.integers(-4, 5, (8, d)) / 4.0).astype(np.float32)
            if variant == "pq":
                ncent = int(rng.integers(2, 9))
                kw = dict(pq=True, num_centroids=ncent, num_subvectors=sub,
                          codebook=(rng.integers(-4, 5, (ncent, d)) / 4.0).astype(np.float32))
            else:
                quant = variant
        r = ref.RefIndex(d, metric, quant, M=M, efc=efc, ef=ef, **kw)
        p = port.PortIndex(d, metric, quant, M=M, efc=efc, ef=ef, **kw)
        r.reserve(n), p.reserve(n)
        for i in range(n):
            r.add(i + 1, X[i]), p.add(i + 1, X[i])
        assert np.array_equal(trim(r.save_buffer(), sub if variant == "pq" else None), p.save_buffer())
        for q in Q:
            k = int(rng.integers(1, 10))
            rk, rd = r.search(q, k)
            pk, pd, _ = p.search(q, k)
            assert np.array_equal(rk, pk) and np.array_equal(rd, pd)

    check()


@pytest.mark.parametrize("metric,quant", [("l2sq", "f32"), ("cos", "f32"), ("hamming", "b1")])
def test_batched_build_model_with_batches_of_one_is_sequential_insertion(port, metric, quant):
    """ora_add_batch_engine models the CUDA engine's two-phase batched build on top of the reference procedures
    (hnsw_oracle.c).  With batch_cap = 1 it must BE the reference's sequential insertion: byte-identical index file."""
    rng = np.random.default_rng(23)
    n = 1500
    if quant == "b1":
        X, dim = rng.integers(0, 256, (n, 24), dtype=np.uint8), 192
    else:
        X, dim = rng.integers(-8, 9, (n, 24)).astype(np.float32), 24
    keys = np.arange(1, n + 1, dtype=np.uint64)
    a = port.PortIndex(dim, metric, quant, M=8, efc=48, ef=32)
    a.reserve(n)
    for k, v in zip(keys, X):
        a.add(int(k), v)
    b = port.PortIndex(dim, metric, quant, M=8, efc=48, ef=32)
    b.reserve(n)
    b.add_batch_engine(keys[:700], X[:700], 1)   # two calls: the level generator carries over like in ora_add
    b.add_batch_engine(keys[700:], X[700:], 1)
    assert np.array_equal(a.save_buffer(), b.save_buffer())


def _model_file(port, X, dim, metric, quant, M, efc, batch, engine_order):
    keys = np.arange(1, len(X) + 1, dtype=np.uint64)
    p = port.PortIndex(dim, metric, quant, M=M, efc=efc, ef=32)
    p.set_engine_order(engine_order)
    p.reserve(len(X))
    p.add_batch_engine(keys, X, batch, 64)
    return p.save_buffer()


@pytest.mark.parametrize("batch", [1, 64])
@pytest.mark.parametrize("M", [4, 16])
@pytest.mark.parametrize("metric", ["l2sq", "cos"])
def test_engine_order_build_equals_heap_order_without_ties(port, metric, M, batch):
    """On float data without exact distance ties the engine's tie order (set before adding: it then governs the insertion
    beams too) changes nothing: the same file, byte for byte, as the reference's heap order."""
    from util import structured
    X = structured(1500, 24, seed=31)
    a = _model_file(port, X, 24, metric, "f32", M, 64, batch, False)
    b = _model_file(port, X, 24, metric, "f32", M, 64, batch, True)
    assert np.array_equal(a, b)


@pytest.mark.parametrize("batch", [1, 64])
def test_engine_order_reaches_the_insertion_beam(port, batch):
    """Clustered hamming data, where exact ties are everywhere: the two orders build different graphs (about 30 % of the
    lists differ), so the switch really reaches search_to_insert and not only the search."""
    from util import adjacency_lists, hamming_rows
    X = hamming_rows(2000, 768, seed=1)
    a = _model_file(port, X, 768, "hamming", "b1", 16, 128, batch, False)
    b = _model_file(port, X, 768, "hamming", "b1", 16, 128, batch, True)
    la, _ = adjacency_lists(a, 16, 96)
    lb, _ = adjacency_lists(b, 16, 96)
    assert sum(la[k] != lb[k] for k in la) > 0.1 * len(la)


@pytest.mark.parametrize("metric,quant", [("l2sq", "f32"), ("cos", "f32"), ("hamming", "b1")])
def test_engine_order_batches_of_one_are_sequential_insertion(port, metric, quant):
    """In the engine's tie order too, the batched-build model with batch_cap = 1 is add() node after node."""
    from util import hamming_rows
    n = 1500
    if quant == "b1":
        X, dim = hamming_rows(n, 192, seed=2), 192
    else:
        X, dim = np.random.default_rng(37).integers(-8, 9, (n, 24)).astype(np.float32), 24
    a = port.PortIndex(dim, metric, quant, M=8, efc=48, ef=32)
    a.set_engine_order(True)
    a.reserve(n)
    for k, v in enumerate(X):
        a.add(k + 1, v)
    assert np.array_equal(a.save_buffer(), _model_file(port, X, dim, metric, quant, 8, 48, 1, True))


def test_batched_build_model_is_deterministic_and_as_good_as_sequential(port):
    rng = np.random.default_rng(29)
    n, d = 4000, 24
    X = rng.integers(-8, 9, (n, d)).astype(np.float32)
    Q = rng.integers(-8, 9, (300, d)).astype(np.float32)
    keys = np.arange(1, n + 1, dtype=np.uint64)
    truth, _ = port.exact_search(X, Q, 10)

    def rec(idx):
        k, _, _, _ = idx.search_batch(Q, 10)
        return float(np.mean([len(set(a.tolist()) & set((t + 1).tolist())) / 10.0 for a, t in zip(k, truth)]))

    seq = port.PortIndex(d, "l2sq", "f32", M=8, efc=48, ef=32)
    seq.reserve(n)
    for k, v in zip(keys, X):
        seq.add(int(k), v)
    files = []
    for _ in range(2):
        b = port.PortIndex(d, "l2sq", "f32", M=8, efc=48, ef=32)
        b.reserve(n)
        b.add_batch_engine(keys, X, 64, 64)
        files.append(b.save_buffer())
    assert np.array_equal(files[0], files[1])
    assert len(files[0]) == len(seq.save_buffer())  # same level draws -> same file size
    assert abs(rec(b) - rec(seq)) < 0.02
    # every link of the batched graph points to a node that exists on that level (what lb200_load_buffer verifies)
    for slot in range(0, n, 97):
        for level in range(b.level(slot) + 1):
            for nb in b.neighbors(slot, level):
                assert b.level(int(nb)) >= level


@pytest.mark.parametrize("metric,scale", [("l2sq", 3.0), ("l2sq", 8.0), ("cos", 3.0)])
def test_kmeans_restatement_equals_the_reference(ref, port, metric, scale):
    """PQ codebook training: the UNMODIFIED reference k-means (lantern_hnsw/src/hnsw/product_quantization.c compiled against
    the stand-in postgres.h of oracle/pg_shim/, PRNG scripted so that both sides start from the same rows) against the
    plain-C restatement ora_kmeans -- bit for bit, for 1, 3 and up to 25 Lloyd rounds, which pins row (f4) of SURVEY 8."""
    if not ref.pq_available():
        pytest.skip("oracle/_ref/liboracle_refpq.so not built")
    rng = np.random.default_rng(6)
    n, d, nsub, ncent = 3000, 24, 4, 16
    centers = rng.standard_normal((ncent, d)).astype(np.float32) * scale
    X = (centers[rng.integers(0, ncent, n)] + rng.standard_normal((n, d))).astype(np.float32)
    init = np.stack([rng.choice(n, ncent, replace=False) for _ in range(nsub)]).astype(np.uint32)
    seen_rounds = set()
    for it in (1, 3, 25):
        rcb = ref.ref_kmeans(X, nsub, ncent, init, metric, it)
        pcb, rounds = port.kmeans(X, nsub, ncent, init, metric, it)
        assert np.array_equal(rcb.view(np.uint32), pcb.view(np.uint32)), np.abs(rcb - pcb).max()
        seen_rounds.add(rounds)
    if metric == "l2sq":
        assert max(seen_rounds) > 3  # the stop rule (mean centre shift <= 0.1) was exercised beyond the early rounds
    # the hnsw_pq_index.sql fixture geometry: k == n, every init is a permutation, one round moves nothing
    Xc = np.repeat((np.arange(10) * 0.1).astype(np.float32)[:, None], 16, axis=1)
    perm = np.stack([rng.permutation(10) for _ in range(4)]).astype(np.uint32)
    assert np.array_equal(ref.ref_kmeans(Xc, 4, 10, perm, "l2sq", 20), port.kmeans(Xc, 4, 10, perm, "l2sq", 20)[0])
