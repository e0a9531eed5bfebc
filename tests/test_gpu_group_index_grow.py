"""GPU tests of a group index that is opened from an index file (lb200_group_index_load[_buffer]) and grown past its capacity
(lb200_group_index_reserve), csrc/group.cu.  A loaded group index holds exactly what a one-GPU index holds after
lb200_load_buffer, so the same adds and builds give the same file, byte for byte; a reserve moves rows between ranks and
changes nothing a search or a save can see.  "Identical search" means keys, distance bits and counts.

As in tests/test_gpu_group_index.py, rank r runs on device r % device_count(), so every case also runs on a box with one GPU."""
import numpy as np
import pytest

from test_golden import G
from test_gpu_group_index import EF, EFC, KINDS, M, _data, _devices, _one_gpu_index, _row_bytes, _stats
from util import structured

pytestmark = pytest.mark.gpu


def _same(a, b):
    (ka, da, ca), (kb, db, cb) = a, b
    return np.array_equal(ka, kb) and np.array_equal(da.view(np.uint32), db.view(np.uint32)) and np.array_equal(ca, cb)


def _check_ranges(grp, ranks, capacity, rb):
    for r in range(ranks):
        info = grp.rank_info(r)
        lo, hi = capacity * r // ranks, capacity * (r + 1) // ranks
        assert (info["rank"], info["world"], info["rows_begin"], info["rows_end"]) == (r, ranks, lo, hi)
        assert info["bytes_rows"] == (hi - lo) * rb


_F0 = {}


def _f0(eng, metric, quant, d, rows):
    """(file F0 of the first n0 rows, built on one GPU; all n0 + n1 rows)"""
    key = (metric, quant, d, rows)
    if key not in _F0:
        n0, n1 = (700, 500) if d < 768 else (400, 300)
        X = _data(quant, d, n0 + n1, rows, metric, seed=11)
        g = _one_gpu_index(eng, metric, quant, d, 64, n0)
        g.add_batch(np.arange(1, n0 + 1, dtype=np.uint64), X[:n0])
        g.build()
        _F0[key] = (g.save_buffer(), X, n0)
        g.close()
    return _F0[key]


def _chunks(a, b):
    """[a, b) in pieces of 1, ~1/3, 7 and the rest"""
    n = b - a
    cuts = [a, a + 1, a + n // 3, a + n // 3 + 7, b]
    return list(zip(cuts[:-1], cuts[1:]))


@pytest.mark.parametrize("build_batch", [64, 1])
@pytest.mark.parametrize("ranks", [1, 2, 4, 8])
@pytest.mark.parametrize("metric,quant,d,rows", KINDS)
def test_load_then_extend_equals_one_gpu(eng, metric, quant, d, rows, ranks, build_batch):
    F0, X, n0 = _f0(eng, metric, quant, d, rows)
    n = len(X)
    capacity = n + 13  # not a multiple of 2, 4 or 8
    keys = np.arange(1, n + 1, dtype=np.uint64)
    one = eng.Index(d, metric, quant, M=M, efc=EFC, ef=EF)
    one.set_option("build_batch", build_batch)
    one.load_buffer(F0)
    one.reserve(capacity)
    grp = eng.Group.local(_devices(eng, ranks))
    grp.index_load_buffer(F0, capacity, d, metric, quant, M=M, efc=EFC, ef=EF, max_batch=256)
    grp.index_set_option("build_batch", build_batch)
    assert grp.index_size() == n0
    _check_ranges(grp, ranks, capacity, _row_bytes(quant, d))
    for a, b in _chunks(n0, n):  # straddling the ranges
        one.add_batch(keys[a:b], X[a:b])
        grp.index_add_batch(keys[a:b], X[a:b])
    one.build()
    grp.index_build()
    assert grp.index_size() == one.size() == n
    assert _stats(grp.index_last_build_stats()) == _stats(one.last_build_stats())
    f = grp.index_save_buffer()
    ref = one.save_buffer()
    assert len(f) == len(ref)
    assert np.array_equal(f, ref), int(np.count_nonzero(f != ref))
    _check_ranges(grp, ranks, capacity, _row_bytes(quant, d))
    grp.close()
    one.close()


@pytest.mark.parametrize("ranks", [2, 4])
def test_loaded_index_searches_like_the_file(eng, ranks, tmp_path):
    """capacity 0 (= the file's rows) and 3 n0, where the trailing ranks hold no rows; the path variant maps the file"""
    metric, quant, d = "cos", "f32", 96
    F0, X, n0 = _f0(eng, metric, quant, d, "structured")
    Q = structured(300, d, seed=77)
    one = eng.Index(d, metric, quant, M=M, efc=EFC, ef=EF)
    one.load_buffer(F0)
    loaded = eng.Group.local(_devices(eng, ranks))
    loaded.load_buffer(F0, d, metric, quant, M=M, efc=EFC, ef=EF, max_batch=512)
    path = str(tmp_path / "f0.usearch")
    F0.tofile(path)
    for capacity, from_path in ((0, False), (3 * n0, False), (3 * n0, True)):
        grp = eng.Group.local(_devices(eng, ranks))
        if from_path:
            grp.index_load(path, capacity, d, metric, quant, M=M, efc=EFC, ef=EF, max_batch=512)
        else:
            grp.index_load_buffer(F0, capacity, d, metric, quant, M=M, efc=EFC, ef=EF, max_batch=512)
        C = capacity or n0
        _check_ranges(grp, ranks, C, _row_bytes(quant, d))
        if capacity:
            assert [r for r in range(ranks) if grp.rank_info(r)["rows_begin"] >= n0], "some rank should hold no rows"
        for ef in (16, 64):
            r1 = one.search_batch(Q, 10, ef)
            assert _same(grp.search_batch(Q, 10, ef), r1), (capacity, ef)
            assert _same(loaded.search_batch(Q, 10, ef), r1), (capacity, ef)
        assert np.array_equal(grp.index_save_buffer(), F0)  # nothing pending: the file comes back unchanged
        grp.close()
    loaded.close()
    one.close()


# reference-written files (tests/golden/make_golden.py): name, metric, d, M, efc, ef
GOLDEN = [("rand_l2", "l2sq", 16, 8, 48, 24), ("rand_cos", "cos", 12, 6, 40, 20)]


@pytest.mark.parametrize("ranks", [2, 4])
@pytest.mark.parametrize("case", GOLDEN, ids=[c[0] for c in GOLDEN])
def test_reference_written_files(eng, case, ranks):
    name, metric, d, m, efc, ef = case
    F, X, Q = G[name + "_file"], G[name + "_X"], G[name + "_Q"]
    n0 = len(X)
    one = eng.Index(d, metric, "f32", M=m, efc=efc, ef=ef)
    one.load_buffer(F)
    loaded = eng.Group.local(_devices(eng, ranks))
    loaded.load_buffer(F, d, metric, "f32", M=m, efc=efc, ef=ef, max_batch=64)
    grp = eng.Group.local(_devices(eng, ranks))
    n1 = 301
    capacity = n0 + n1 + 3
    grp.index_load_buffer(F, capacity, d, metric, "f32", M=m, efc=efc, ef=ef, max_batch=64)
    for e in (16, 64):
        r1 = one.search_batch(Q, 10, e)
        assert _same(grp.search_batch(Q, 10, e), r1), e
        assert _same(loaded.search_batch(Q, 10, e), r1), e
    # then extended, as one GPU extends it
    Y = structured(n1, d, seed=41)
    keys = np.arange(5000, 5000 + n1, dtype=np.uint64)
    one.reserve(capacity)
    for s in (one, grp):
        (s.set_option if s is one else s.index_set_option)("build_batch", 64)
    for a, b in _chunks(0, n1):
        one.add_batch(keys[a:b], Y[a:b])
        grp.index_add_batch(keys[a:b], Y[a:b])
    one.build()
    grp.index_build()
    assert grp.index_size() == one.size() == n0 + n1
    assert _stats(grp.index_last_build_stats()) == _stats(one.last_build_stats())
    assert np.array_equal(grp.index_save_buffer(), one.save_buffer())
    assert _same(grp.search_batch(Q, 10, 32), one.search_batch(Q, 10, 32))
    grp.close()
    loaded.close()
    one.close()


def _pair(eng, ranks, metric, quant, d, capacity, max_batch=512):
    one = _one_gpu_index(eng, metric, quant, d, 64, capacity)
    grp = eng.Group.local(_devices(eng, ranks))
    grp.index_init(capacity, d, metric, quant, M=M, efc=EFC, ef=EF, max_batch=max_batch)
    grp.index_set_option("build_batch", 64)
    return one, grp


@pytest.mark.parametrize("ranks", [2, 4])
def test_reserve_moves_rows_and_changes_nothing_else(eng, ranks):
    metric, quant, d = "l2sq", "f32", 48
    C, extra, max_batch = 1001, 1700, 512
    X, Q = _data(quant, d, C + extra, seed=21), structured(max_batch, d, seed=23)
    keys = np.arange(1, C + extra + 1, dtype=np.uint64)
    rb = _row_bytes(quant, d)
    one, grp = _pair(eng, ranks, metric, quant, d, C, max_batch)
    for add, build in ((one.add_batch, one.build), (grp.index_add_batch, grp.index_build)):
        add(keys[:C], X[:C])  # to the capacity
        build()
    before = grp.search_batch(Q[:100], 10, 32)
    graph_bytes = grp.rank_info(0)["bytes_graph"]
    # at or below the capacity: nothing happens
    for c in (C, C - 10, 0):
        grp.index_reserve(c)
        _check_ranges(grp, ranks, C, rb)
    C2 = 3 * C + 5  # rows cross more than one range boundary
    grp.index_reserve(C2)
    one.reserve(C2)
    _check_ranges(grp, ranks, C2, rb)
    assert grp.rank_info(0)["bytes_graph"] > graph_bytes
    assert grp.index_size() == C
    assert _same(grp.search_batch(Q[:100], 10, 32), before)
    for a, b in _chunks(C, C + extra):  # past the old capacity
        one.add_batch(keys[a:b], X[a:b])
        grp.index_add_batch(keys[a:b], X[a:b])
    one.build()
    grp.index_build()
    assert _stats(grp.index_last_build_stats()) == _stats(one.last_build_stats())
    assert np.array_equal(grp.index_save_buffer(), one.save_buffer())
    # the group's full batch once n has passed the old capacity: the owners' bitmaps were resized
    assert _same(grp.search_batch(Q, 10, 64), one.search_batch(Q, 10, 64))
    grp.close()
    one.close()


def test_reserve_between_add_and_build_moves_pending_rows(eng):
    metric, quant, d, ranks = "cos", "f32", 96, 4
    C, n = 1003, 2600
    X, Q = _data(quant, d, n, seed=29), structured(200, d, seed=31)
    keys = np.arange(1, n + 1, dtype=np.uint64)
    one, grp = _pair(eng, ranks, metric, quant, d, C)
    for add, build, reserve in ((one.add_batch, one.build, one.reserve), (grp.index_add_batch, grp.index_build, grp.index_reserve)):
        add(keys[:600], X[:600])
        build()
        add(keys[600:1000], X[600:1000])  # pending across the reserve
        reserve(2 * C + 1)
        add(keys[1000:2000], X[1000:2000])
        reserve(n)
        add(keys[2000:], X[2000:])
        build()
    assert grp.index_size() == one.size() == n
    assert _stats(grp.index_last_build_stats()) == _stats(one.last_build_stats())
    assert np.array_equal(grp.index_save_buffer(), one.save_buffer())
    assert _same(grp.search_batch(Q, 10, 48), one.search_batch(Q, 10, 48))
    _check_ranges(grp, ranks, n, _row_bytes(quant, d))
    grp.close()
    one.close()


@pytest.mark.parametrize("ranks", [2, 4])
def test_growth_by_doubling_as_the_external_indexer_does(eng, ranks):
    """lantern_cli's external indexer reserves an estimate, then doubles the capacity whenever the rows received reach it"""
    metric, quant, d, n, chunk = "l2sq", "f32", 64, 5200, 300
    X = _data(quant, d, n, seed=37)
    keys = np.arange(1, n + 1, dtype=np.uint64)
    one, grp = _pair(eng, ranks, metric, quant, d, 1000)
    for add, build, reserve in ((one.add_batch, one.build, one.reserve), (grp.index_add_batch, grp.index_build, grp.index_reserve)):
        capacity, received = 1000, 0
        for i, a in enumerate(range(0, n, chunk)):
            b = min(a + chunk, n)
            if b > capacity:  # (row by row: at received == capacity)
                received_at = max(a, capacity)
                add(keys[a:received_at], X[a:received_at])
                while b > capacity:
                    capacity *= 2
                    reserve(capacity)
                add(keys[received_at:b], X[received_at:b])
            else:
                add(keys[a:b], X[a:b])
            received = b
            if i % 4 == 3:
                build()
        build()
    assert received == n and capacity == 8000
    assert grp.index_size() == one.size() == n
    assert np.array_equal(grp.index_save_buffer(), one.save_buffer())
    _check_ranges(grp, ranks, 8000, _row_bytes(quant, d))
    grp.close()
    one.close()


def test_empty_file(eng):
    metric, quant, d = "l2sq", "f32", 32
    empty = eng.Index(d, metric, quant, M=M, efc=EFC, ef=EF).save_buffer()
    X = _data(quant, d, 500, seed=43)
    keys = np.arange(1, 501, dtype=np.uint64)
    grp = eng.Group.local(_devices(eng, 2))
    with pytest.raises(eng.EngineError, match="capacity"):
        grp.index_load_buffer(empty, 0, d, metric, quant, M=M, efc=EFC, ef=EF)
    grp.index_load_buffer(empty, 1, d, metric, quant, M=M, efc=EFC, ef=EF, max_batch=64)
    assert grp.index_size() == 0
    grp.index_reserve(500)
    grp.index_set_option("build_batch", 64)
    grp.index_add_batch(keys, X)
    grp.index_build()
    one = _one_gpu_index(eng, metric, quant, d, 64, 1)
    one.load_buffer(empty)
    one.reserve(500)
    one.add_batch(keys, X)
    one.build()
    assert np.array_equal(grp.index_save_buffer(), one.save_buffer())
    grp.close()
    one.close()


def test_refusals_leave_the_group_usable(eng):
    metric, quant, d = "cos", "f32", 96
    F0, X, n0 = _f0(eng, metric, quant, d, "structured")
    calls = []

    def allgather(send):
        calls.append(len(send))
        raise AssertionError("a refused index_load must not communicate")

    multi = eng.Group.ranked(0, 2, allgather)
    with pytest.raises(eng.EngineError, match="lb200_group_create_local"):
        multi.index_load_buffer(F0, 0, d, metric, quant, M=M, efc=EFC, ef=EF)
    assert not calls
    multi.close()

    def one_gpu_error(dim, met):
        g = eng.Index(dim, met, quant, M=M, efc=EFC, ef=EF)
        with pytest.raises(eng.EngineError) as e:
            g.load_buffer(F0)
        g.close()
        return str(e.value)

    for accept in ("load", "init"):
        grp = eng.Group.local(_devices(eng, 2))
        with pytest.raises(eng.EngineError, match="lb200_group_index_init"):
            grp.index_reserve(5000)
        with pytest.raises(eng.EngineError, match="pq"):
            grp.index_load_buffer(F0, 0, d, metric, quant, M=M, efc=EFC, ef=EF, pq=True)
        for dim, met in ((d + 1, metric), (d, "l2sq")):
            with pytest.raises(eng.EngineError) as e:
                grp.index_load_buffer(F0, 0, dim, met, quant, M=M, efc=EFC, ef=EF)
            assert str(e.value) == one_gpu_error(dim, met)
        with pytest.raises(eng.EngineError, match="truncated"):
            grp.index_load_buffer(F0[:-10], 0, d, metric, quant, M=M, efc=EFC, ef=EF)
        for capacity in (n0 - 1, 2**31 - 1, 2**32):
            with pytest.raises(eng.EngineError, match="capacity"):
                grp.index_load_buffer(F0, capacity, d, metric, quant, M=M, efc=EFC, ef=EF)
        if accept == "load":
            grp.index_load_buffer(F0, 0, d, metric, quant, M=M, efc=EFC, ef=EF, max_batch=256)
            assert grp.index_size() == n0
            assert np.array_equal(grp.index_save_buffer(), F0)
        else:
            grp.index_init(n0, d, metric, quant, M=M, efc=EFC, ef=EF, max_batch=256)
            assert grp.index_size() == 0
        # a second formation of any kind
        msg = "one lb200_group_distribute, lb200_group_load or lb200_group_index_init"
        with pytest.raises(eng.EngineError, match=msg):
            grp.index_load_buffer(F0, 0, d, metric, quant, M=M, efc=EFC, ef=EF)
        with pytest.raises(eng.EngineError, match=msg):
            grp.index_init(n0, d, metric, quant, M=M, efc=EFC, ef=EF)
        with pytest.raises(eng.EngineError, match="already"):
            grp.load_buffer(F0, d, metric, quant, M=M, efc=EFC, ef=EF)
        grp.close()

    # a group formed by lb200_group_load holds no index of its own to reserve
    loaded = eng.Group.local(_devices(eng, 2))
    loaded.load_buffer(F0, d, metric, quant, M=M, efc=EFC, ef=EF, max_batch=64)
    with pytest.raises(eng.EngineError, match="lb200_group_index_init"):
        loaded.index_reserve(5000)
    loaded.close()


@pytest.mark.parametrize("ranks", [2, 3])
def test_reserve_no_device_can_hold_is_refused_and_changes_nothing(eng, ranks):
    """2^31 - 2 rows of d768 f32 is ~6.6 TB of rows: an ordinary allocation failure, named by rank and category"""
    metric, quant, d = "l2sq", "f32", 768
    F0, X, n0 = _f0(eng, metric, quant, d, "structured")
    Q = structured(100, d, seed=47)
    grp = eng.Group.local(_devices(eng, ranks))
    grp.index_load_buffer(F0, n0 + 50, d, metric, quant, M=M, efc=EFC, ef=EF, max_batch=128)
    grp.index_set_option("build_batch", 64)
    grp.index_add_batch(np.arange(n0 + 1, n0 + 51, dtype=np.uint64), X[n0:n0 + 50])
    before = grp.search_batch(Q, 10, 48)  # (builds the added rows)
    saved = grp.index_save_buffer()
    info = [grp.rank_info(r) for r in range(ranks)]
    with pytest.raises(eng.EngineError, match=r"rank \d+ \(device \d+\): no room for its rows"):
        grp.index_reserve(2**31 - 2)
    assert [grp.rank_info(r) for r in range(ranks)] == info
    assert _same(grp.search_batch(Q, 10, 48), before)
    assert np.array_equal(grp.index_save_buffer(), saved)
    # and a reserve that fits still works afterwards
    grp.index_reserve(3 * n0)
    _check_ranges(grp, ranks, 3 * n0, _row_bytes(quant, d))
    assert _same(grp.search_batch(Q, 10, 48), before)
    assert np.array_equal(grp.index_save_buffer(), saved)
    grp.close()
