"""Every row width the kernels are compiled for, against float64.

Each row-distance kernel is instantiated per distance mode, scalar kind and NQ, the number of 16-byte query chunks a lane
keeps in registers (walk.cuh pick_nq: NQ in {1, 2, 3, 4, 6, 8, 12, 16}, rows up to 512 NQ bytes).  width_table lists, for each
(kind, metric), dimension counts that reach every NQ: the widest row of each NQ, the narrowest one (the previous widest plus
one element, which opens a new register pass and leaves a ragged tail), d = 1 and 3, and one more ragged row at NQ = 16.

The GPU tests run the search kernels (one CTA per query, one warp per query, at both ends of their ring depths), the
batched build, the row-sharded group, the screened f32 walkers, the exhaustive search and the pair distances at those
widths, and check every distance against util.reference64: float64 on the storage-domain rows with an a-priori bound on
the fp32 kernels' rounding.  Ids are compared tie-aware.
"""
import os

import numpy as np
import pytest

from util import (check_distances, check_topk, chunk_passes, compare_results, describe_file_difference, hamming_rows,
                  make_rows, reference64, row_bytes, structured)

NQ_OPTS = (1, 2, 3, 4, 6, 8, 12, 16)
PAIRS = [("f32", "l2sq"), ("f32", "cos"), ("f16", "l2sq"), ("f16", "cos"), ("i8", "l2sq"), ("i8", "cos"), ("b1", "hamming")]
PER_BYTE = {"f32": 0.25, "f16": 0.5, "i8": 1, "b1": 8}  # elements (bits for b1) per byte
REFUSED = "wider than 8192 bytes"
K = 10


def pick_nq(rb):
    """walk.cuh pick_nq: the register passes a row of `rb` padded bytes needs, rounded up to a compiled NQ; -1 past 8192."""
    need = chunk_passes(rb)
    return next((o for o in NQ_OPTS if o >= need), -1)


def widest(quant, nq):
    return int(512 * nq * PER_BYTE[quant])


def width_table(quant):
    dims = {1, 3, widest(quant, 16) - 1}
    for i, nq in enumerate(NQ_OPTS):
        dims.add(widest(quant, nq))
        if i:
            dims.add(widest(quant, NQ_OPTS[i - 1]) + 1)
    return sorted(dims)


def first_refused(quant):
    return widest(quant, 16) + 1


def case_ids(pairs_dims):
    return ["%s-%s-d%d" % c for c in pairs_dims]


ALL = [(q, m, d) for q, m in PAIRS for d in width_table(q)]
WIDEST = [(q, m, widest(q, nq)) for q, m in PAIRS for nq in NQ_OPTS]


def test_width_table():
    """CPU: the table reaches every NQ for every (kind, metric), with ragged rows, and the first width past 8192 bytes is
    one the engine refuses."""
    assert width_table("f32") == [1, 3, 128, 129, 256, 257, 384, 385, 512, 513, 768, 769, 1024, 1025, 1536, 1537, 2047, 2048]
    ragged = {"f32": lambda d: d % 4 == 1, "f16": lambda d: d % 2 == 1, "i8": lambda d: d % 16 == 1, "b1": lambda d: d % 8 == 1}
    for quant, metric in PAIRS:
        table = width_table(quant)
        by_nq = {}
        for d in table:
            rb = row_bytes(quant, d)
            by_nq.setdefault(pick_nq(rb), []).append((d, rb))
        assert sorted(by_nq) == list(NQ_OPTS), (quant, metric, sorted(by_nq))
        for i, nq in enumerate(NQ_OPTS):
            rbs = [rb for _, rb in by_nq[nq]]
            assert max(rbs) == 512 * nq, (quant, nq)
            if i:
                assert min(rbs) == 512 * NQ_OPTS[i - 1] + 16, (quant, nq)
            assert any(ragged[quant](d) for d, _ in by_nq[nq]), (quant, nq)
        assert pick_nq(row_bytes(quant, first_refused(quant))) == -1
    assert [first_refused(q) for q in ("f32", "f16", "i8", "b1")] == [2049, 4097, 8193, 65537]


@pytest.mark.parametrize("quant,metric", [p for p in PAIRS if p[0] in ("f32", "f16")], ids=["%s-%s" % p for p in PAIRS[:4]])
def test_reference_bound_is_tight(port, quant, metric):
    """CPU: on continuous data the median bound is below 1e-5 of the distance at every width, so a kernel that is wrong by
    more than rounding cannot hide inside it."""
    for dims in (3, widest(quant, 1), widest(quant, 16)):
        X, Q, S, QS = search_data(port, quant, dims, 300, 8, seed=dims)
        D, B = reference64(QS, S, metric, quant)
        assert np.median(B / D) < 1e-5, (dims, np.median(B / D))
        # the nearest rows too; under cos relative to 1, the scale at which 1 - ab / (|a| |b|) is rounded
        top = np.argsort(D, 1)[:, :K]
        scale = np.take_along_axis(D, top, 1) if metric == "l2sq" else 1.0
        assert np.median(np.take_along_axis(B, top, 1) / scale) < 1e-5, dims


# ---- data ---------------------------------------------------------------------------------------------------------------
def search_data(port, quant, dims, n, nq, seed):
    """(rows, queries) as passed to the engine and the oracle, and the same in the storage domain."""
    if quant == "b1":
        X, Q = hamming_rows(n, dims, seed), hamming_rows(nq, dims, seed + 1)
        return X, Q, X, Q
    X, Q = structured(n, dims, seed), structured(nq, dims, seed + 1)
    if quant == "i8":
        X, Q = X * 0.3, Q * 0.3
    if quant == "f32":
        return X, Q, X, Q
    return X, Q, port.cast_f32(X, quant), port.cast_f32(Q, quant)


def sizes(rb):
    """(rows, queries): fewer rows past 2 KB, where the CPU oracle's graph build is slow."""
    return (1200, 64) if rb <= 2048 else (500, 64)


class env:
    """Engine environment knobs for one block (the engine reads them at each call)."""

    def __init__(self, **kv):
        self.kv, self.old = kv, {}

    def __enter__(self):
        for k, v in self.kv.items():
            self.old[k] = os.environ.get(k)
            os.environ[k] = str(v)

    def __exit__(self, *a):
        for k, v in self.old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


@pytest.fixture(autouse=True)
def no_screen():
    """The plain walkers unless a test asks for a screen."""
    with env(LB200_SEARCH_SCREEN=0):
        yield


def returned_reference(QS, S, keys, metric, quant):
    """float64 distances and bounds of the returned ids (keys are offsets + 1)."""
    D, B = reference64(QS, S, metric, quant)
    ids = keys.astype(np.int64) - 1
    return np.take_along_axis(D, ids, 1), np.take_along_axis(B, ids, 1)


# ---- the search kernels on the oracle's graph ------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("quant,metric,dims", ALL, ids=case_ids(ALL))
def test_search_same_graph(eng, port, quant, metric, dims):
    """The oracle's graph: both search kernels, at both ends of their ring depths, give the oracle's ids and work counters
    and bit-identical distances within the float64 bound.  Then ef >= n on the same (connected) graph: the CTA kernel's
    top-k is the float64 brute force, and the warp kernel agrees bit for bit or refuses the ef by name."""
    rb = row_bytes(quant, dims)
    n, nq = sizes(rb)
    X, Q, S, QS = search_data(port, quant, dims, n, nq, seed=dims)
    M, efc, ef = 16, 32, 32
    p = port.PortIndex(dims, metric, quant, M=M, efc=efc, ef=ef)
    p.reserve(n)
    for i in range(n):
        p.add(i + 1, X[i])
    g = eng.Index(dims, metric, quant, M=M, efc=efc, ef=ef)
    g.load_buffer(p.save_buffer())
    p.set_engine_order(True)  # the engine's order among equal distances (b1 and tiny rows are full of ties)
    pk, pd, pc, tot = p.search_batch(Q, K)

    variants = [("cta", 1, {}), ("cta-2warps", 1, {"LB200_SEARCH_WARPS": 2}), ("cta-ring4", 1, {"LB200_RING_BYTES": 1}),
                ("cta-ring16", 1, {"LB200_RING_BYTES": 16 * rb}), ("warp", 2, {}),
                ("warp-ring1", 2, {"LB200_GROUP_RING_SLOTS": 1}), ("warp-ring8", 2, {"LB200_GROUP_RING_SLOTS": 8})]
    runs = {}
    for name, kernel, kv in variants:
        g.set_option("search_kernel", kernel)
        with env(**kv):
            try:
                gk, gd, gc = g.search_batch(Q, K)
            except eng.EngineError as e:  # a ring deeper than shared memory holds: refused by name, nothing left broken
                assert name.endswith(("ring16", "ring8")) and "kernel does not fit on an SM" in str(e), (name, str(e))
                continue
        st = g.last_stats()
        assert st["search_kernel"] == kernel, name
        runs[name] = (gk, gd, gc, st)

    gk, gd, gc, st = runs["cta"]
    assert np.array_equal(gc.astype(np.int64), pc)
    exact, ok = compare_results(gk, gd, pk, pd)
    assert ok == nq, (exact, ok)
    assert exact >= 0.97 * nq, exact
    Dr, Br = returned_reference(QS, S, gk, metric, quant)
    check_distances(gd, Dr, Br, "cta")
    for name, (k2, d2, c2, s2) in runs.items():
        assert np.array_equal(k2, gk) and np.array_equal(d2.view(np.uint32), gd.view(np.uint32)), name
        assert np.array_equal(c2, gc), name
        if exact == nq:
            assert (s2["computed_distances"], s2["base_pops"], s2["upper_hops"]) == (
                tot["computed_distances"], tot["base_pops"], tot["upper_hops"]), name

    g.set_option("search_kernel", 1)
    xk, xd, _ = g.search_batch(Q, K, ef=n)
    D, B = reference64(QS, S, metric, quant)
    check_topk(xk.astype(np.int64) - 1, xd, D, B, K, "cta ef=n")
    g.set_option("search_kernel", 2)
    try:
        wk, wd, _ = g.search_batch(Q, K, ef=n)
    except eng.EngineError as e:
        assert "warp search: kernel does not fit on an SM" in str(e), str(e)
    else:
        assert np.array_equal(wk, xk) and np.array_equal(wd.view(np.uint32), xd.view(np.uint32))


# ---- the batched build, byte for byte against its CPU model ----------------------------------------------------------
BUILD = [(q, m, d) for q, m in PAIRS for d in [3] + [widest(q, nq) for nq in NQ_OPTS]]


def exact_rows_spec(quant, metric, dims):
    """The largest value range whose fp32 distances are exact at this width (util.make_rows)."""
    if quant == "b1":
        return ("bits",)
    lim = 2 ** 24 - 1
    r = int(np.sqrt(lim / dims) / 2) if metric == "l2sq" else int(np.sqrt(lim / dims))
    while (dims * (2 * r) ** 2 if metric == "l2sq" else dims * r * r) >= 2 ** 24:
        r -= 1
    if quant == "i8":
        r = min(r, 100)
        return ("i8", r / 100 + 0.005)
    return ("int0" if metric == "cos" else "int", min(r, 100 if quant == "f32" else 2048))


@pytest.mark.gpu
@pytest.mark.parametrize("batch", [1, 64])
@pytest.mark.parametrize("quant,metric,dims", BUILD, ids=case_ids(BUILD))
def test_build_equals_cpu_model(eng, port, quant, metric, dims, batch):
    n = 300 if row_bytes(quant, dims) <= 2048 else 200
    X, S = make_rows(port, quant, metric, dims, exact_rows_spec(quant, metric, dims), n, seed=dims + batch)
    keys = np.arange(1, n + 1, dtype=np.uint64) * 3
    M, efc = 8, 32
    p = port.PortIndex(dims, metric, quant, M=M, efc=efc, ef=16)
    p.set_engine_order(True)
    p.reserve(n)
    p.add_batch_engine(keys, X, batch, 16)
    g = eng.Index(dims, metric, quant, M=M, efc=efc, ef=16)
    g.set_option("build_batch", batch)
    g.set_option("build_ratio", 16)
    g.reserve(n)
    g.add_batch(keys, X)
    g.build()
    gb, pb = g.save_buffer(), p.save_buffer()
    assert np.array_equal(gb, pb), describe_file_difference(gb, pb, M, S.shape[1] * S.itemsize, S, metric, quant, dims, port)


# ---- the row-sharded group -------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("quant,metric,dims", WIDEST, ids=case_ids(WIDEST))
def test_group_index_two_ranks(eng, port, quant, metric, dims):
    n, nq = sizes(row_bytes(quant, dims))
    X, Q, S, QS = search_data(port, quant, dims, n, nq, seed=dims + 3)
    keys = np.arange(1, n + 1, dtype=np.uint64)
    one = eng.Index(dims, metric, quant, M=8, efc=48, ef=32)
    one.set_option("build_batch", 64)
    one.reserve(n)
    one.add_batch(keys, X)
    one.build()
    one.set_option("search_kernel", 2)
    ok_, od, oc = one.search_batch(Q, K)
    grp = eng.Group.local([r % eng.device_count() for r in range(2)])  # one device may hold both ranks
    try:
        grp.index_init(n, dims, metric, quant, M=8, efc=48, ef=32)
        grp.index_set_option("build_batch", 64)
        grp.index_add_batch(keys, X)
        grp.index_build()
        gk, gd, gc = grp.search_batch(Q, K)
    finally:
        grp.close()
    assert np.array_equal(gk, ok_) and np.array_equal(gd.view(np.uint32), od.view(np.uint32)) and np.array_equal(gc, oc)
    D, B = returned_reference(QS, S, gk, metric, quant)
    check_distances(gd, D, B, "group")


# ---- the screened f32 walkers ----------------------------------------------------------------------------------------
SCREENED = [("f32", m, 128 * nq) for m in ("l2sq", "cos") for nq in (1, 3, 4, 12, 16)]


@pytest.mark.gpu
@pytest.mark.parametrize("quant,metric,dims", SCREENED, ids=case_ids(SCREENED))
def test_screened_walkers_bit_identical(eng, port, quant, metric, dims):
    n, nq = sizes(row_bytes(quant, dims))
    X, Q, S, QS = search_data(port, quant, dims, n, nq, seed=dims + 5)
    g = eng.Index(dims, metric, quant, M=8, efc=48, ef=32)
    g.reserve(n)
    g.add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
    g.build()
    runs = {}
    for kernel in (1, 2):
        g.set_option("search_kernel", kernel)
        for screen in (0, 1, 2):
            if kernel == 2 and screen == 1:
                continue  # the warp kernel screens with the projected screen only
            with env(LB200_SEARCH_SCREEN=screen):
                runs[(kernel, screen)] = g.search_batch(Q, K)
            st = g.last_stats()
            assert st["screen_kind"] == screen, (kernel, screen, st["screen_kind"])
    bk, bd, bc = runs[(1, 0)]
    for key, (k2, d2, c2) in runs.items():
        assert np.array_equal(k2, bk) and np.array_equal(d2.view(np.uint32), bd.view(np.uint32)) and np.array_equal(c2, bc), key
    D, B = returned_reference(QS, S, bk, metric, quant)
    check_distances(bd, D, B, "screen")


# ---- exhaustive search and pair distances ----------------------------------------------------------------------------
WIDE = {"f32": [4096, 7200, 7201, 8192, 16384]}
WIDE["f16"] = [2 * d for d in WIDE["f32"]]
WIDE["i8"] = [4 * d for d in WIDE["f32"]]
EXACT = ALL + [(q, m, d) for q, m in PAIRS if q in WIDE for d in WIDE[q]] + [("b1", "hamming", 8 * 4 * 7201)]


def exact_data(quant, dims, n, nq, seed):
    """Storage-domain rows and queries, passed to the engine in their own kind."""
    rng = np.random.default_rng(seed)
    if quant == "b1":
        return hamming_rows(n, dims, seed), hamming_rows(nq, dims, seed + 1)
    X, Q = structured(n, dims, seed), structured(nq, dims, seed + 1)
    if quant == "f16":
        return X.astype(np.float16).view(np.uint16), Q.astype(np.float16).view(np.uint16)
    if quant == "i8":
        return (rng.integers(-128, 128, (n, dims)).astype(np.int8), rng.integers(-128, 128, (nq, dims)).astype(np.int8))
    return X, Q


@pytest.mark.gpu
@pytest.mark.parametrize("quant,metric,dims", EXACT, ids=case_ids(EXACT))
def test_exact_search_and_pair_distance(eng, quant, metric, dims):
    n = 1061 if row_bytes(quant, dims) <= 8192 else 101  # not multiples of 32; past 8192 bytes k = 1024 exceeds n
    S, QS = exact_data(quant, dims, n, 9, seed=dims)
    D, B = reference64(QS, S, metric, quant)
    modes = ["simt", "tc"] if quant == "f32" else ["simt"]
    for mode in modes:
        with env(LB200_EXACT=mode):
            for nq in (1, 9):
                for k in (1, 33, 1024):
                    keys, dists = eng.exact_search(S, QS[:nq], k, metric, quant, dims)
                    check_topk(keys, dists, D[:nq], B[:nq], k, "%s nq%d k%d" % (mode, nq, k))
    # pair distances: query i against row i
    m = min(n, 300)
    pairs = eng.distance_batch(np.repeat(QS, m // len(QS) + 1, 0)[:m], S[:m], metric, quant, dims)
    Dp, Bp = reference64(np.repeat(QS, m // len(QS) + 1, 0)[:m], S[:m], metric, quant)
    check_distances(pairs, np.diag(Dp), np.diag(Bp), "distance_batch")


@pytest.mark.gpu
def test_exact_search_600000_queries(eng):
    """More query tiles than a grid's y dimension holds (65535 x 8 queries)."""
    rng = np.random.default_rng(2)
    X = rng.integers(-3, 4, (64, 4)).astype(np.float32)
    Q = rng.integers(-3, 4, (600000, 4)).astype(np.float32)
    keys, dists = eng.exact_search(X, Q, 1, "l2sq")
    want = np.empty(len(Q), np.int64)
    wd = np.empty(len(Q), np.float32)
    for s in range(0, len(Q), 50000):  # integer data: exact distances, ties by lower offset
        d = ((Q[s:s + 50000, None, :] - X[None, :, :]) ** 2).sum(-1)
        want[s:s + 50000] = d.argmin(1)
        wd[s:s + 50000] = d.min(1)
    assert np.array_equal(keys[:, 0].astype(np.int64), want) and np.array_equal(dists[:, 0], wd)


# ---- refusals --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("quant,metric", PAIRS, ids=["%s-%s" % p for p in PAIRS])
def test_first_width_past_8192_bytes_is_refused(eng, port, quant, metric):
    dims = first_refused(quant)
    with pytest.raises(eng.EngineError, match=REFUSED):
        eng.Index(dims, metric, quant, M=8, efc=16, ef=16)
    rng = np.random.default_rng(0)
    X = hamming_rows(20, dims, 1) if quant == "b1" else rng.standard_normal((20, dims)).astype(np.float32)
    p = port.PortIndex(dims, metric, quant, M=8, efc=16, ef=16)
    p.reserve(len(X))
    for i in range(len(X)):
        p.add(i + 1, X[i])
    buf = p.save_buffer()
    for form in (lambda grp: grp.index_load_buffer(buf, 0, dims, metric, quant, M=8, efc=16, ef=16),
                 lambda grp: grp.index_init(100, dims, metric, quant, M=8, efc=16, ef=16),
                 lambda grp: grp.load_buffer(buf, dims, metric, quant, M=8, efc=16, ef=16)):
        grp = eng.Group.local([0])
        try:
            with pytest.raises(eng.EngineError, match=REFUSED):
                form(grp)
        finally:
            grp.close()
    # a correct index on the same device afterwards
    d_ok = widest(quant, 16)
    Xo = hamming_rows(300, d_ok, 2) if quant == "b1" else rng.standard_normal((300, d_ok)).astype(np.float32)
    g = eng.Index(d_ok, metric, quant, M=8, efc=32, ef=32)
    g.reserve(300)
    g.add_batch(np.arange(1, 301, dtype=np.uint64), Xo)
    g.build()
    gk, gd, _ = g.search_batch(Xo[:5], 1, ef=300)
    assert np.array_equal(gk[:, 0], np.arange(1, 6))
    assert (np.abs(gd[:, 0]) <= (1e-6 if metric == "cos" else 0)).all(), gd[:, 0]


# ---- edge values -----------------------------------------------------------------------------------------------------
EDGE = [(q, m, d) for q, m in PAIRS for d in (1, widest(q, 16))] + [("b1", "hamming", 4097), ("b1", "hamming", 65535)]
# i8 at the widest exact-search rows: 255^2 d passes 2^31 past 33025 dimensions; 131071 is the widest i8 row accepted
EDGE += [("i8", "l2sq", 65536), ("i8", "cos", 65536), ("i8", "l2sq", 131071)]


def edge_rows(quant, metric, dims, n, seed):
    """Storage-domain rows holding each kind's extreme values."""
    rng = np.random.default_rng(seed)
    if quant == "b1":  # bits past `dims` set in the last byte of every other row: usearch counts them, so must the kernels
        X = hamming_rows(n, dims, seed)
        if dims % 8:
            X[::2, -1] |= np.uint8((1 << (8 - dims % 8)) - 1)
        return X
    if quant == "f16":
        vals = np.array([65504, -65504, 2.0 ** -24, -(2.0 ** -24), 3 * 2.0 ** -20, 2.0 ** -14, 1.0, -0.5, 0.0], np.float16)
        X = rng.choice(vals, (n, dims)).astype(np.float16).view(np.uint16)
    elif quant == "i8":
        X = rng.choice(np.array([-128, 127, -1, 1, 0, 100, -100], np.int8), (n, dims))
    else:
        X = rng.choice(np.array([3.0e4, -3.0e4, 1e-3, -2.5, 1.0, 0.0], np.float32), (n, dims))
    if quant == "i8":
        X[3], X[5] = -128, 127  # all -128 against all 127: the largest i8 distance of the width
    if metric == "cos":
        X[:3] = 0  # zero rows: the zero-norm table
    return X


@pytest.mark.gpu
@pytest.mark.parametrize("quant,metric,dims", EDGE, ids=case_ids(EDGE))
def test_edge_values(eng, quant, metric, dims):
    n = 97
    S = edge_rows(quant, metric, dims, n, seed=dims)
    QS = S[[0, 5, 6, 50, 96]].copy()
    if metric == "cos":
        QS[0] = 0  # a zero query
    D, B = reference64(QS, S, metric, quant)
    keys, dists = eng.exact_search(S, QS, 33, metric, quant, dims)
    check_topk(keys, dists, D, B, 33, "exact")
    pd = eng.distance_batch(np.repeat(QS, 20, 0)[:n], S, metric, quant, dims)
    Dp, Bp = reference64(np.repeat(QS, 20, 0)[:n], S, metric, quant)
    check_distances(pd, np.diag(Dp), np.diag(Bp), "distance_batch")
    if quant == "i8":
        far = eng.distance_batch(S[[3, 5]], S[[5, 3]], metric, quant, dims)  # -128 against 127 and back
        Df, Bf = reference64(S[[3, 5]], S[[5, 3]], metric, quant)
        check_distances(far, np.diag(Df), np.diag(Bf), "-128 against 127")
        if dims == 131071:  # one more and the int32 dot products could wrap: refused by name
            wide = np.zeros((2, dims + 1), np.int8)
            with pytest.raises(eng.EngineError, match="i8 rows wider than 131071 dimensions"):
                eng.exact_search(wide, wide, 1, metric, quant, dims + 1)
            with pytest.raises(eng.EngineError, match="i8 rows wider than 131071 dimensions"):
                eng.distance_batch(wide, wide, metric, quant, dims + 1)
        elif dims <= 8192:  # the index takes i8 rows and queries only as f32 values to cast: i8 queries are refused by name
            g = eng.Index(dims, metric, quant, M=16, efc=64, ef=n)
            keys, dists = np.zeros((len(QS), 10), np.uint64), np.zeros((len(QS), 10), np.float32)
            with pytest.raises(eng.EngineError, match="vectors must be passed as f32"):
                g.search_batch_raw(QS.ctypes.data, len(QS), QS.strides[0], "i8", 10, 0, keys.ctypes.data, dists.ctypes.data, 0)
    else:
        # the index path: f16 rows arrive as f32 values (the cast is exact for f16 values), b1 as packed bytes
        In = S.view(np.float16).astype(np.float32) if quant == "f16" else S
        Iq = QS.view(np.float16).astype(np.float32) if quant == "f16" else QS
        g = eng.Index(dims, metric, quant, M=16, efc=64, ef=n)
        g.reserve(n)
        g.add_batch(np.arange(1, n + 1, dtype=np.uint64), In)
        g.build()
        for kernel in (1, 2):
            g.set_option("search_kernel", kernel)
            gk, gd, _ = g.search_batch(Iq, 10, ef=n)
            check_topk(gk.astype(np.int64) - 1, gd, D, B, 10, "index kernel %d" % kernel)
