"""GPU tests of the group's own index (lb200_group_index_*, csrc/group.cu + csrc/build.cu): an index built straight into the
row-sharded layout, where rank r holds only the rows of its capacity range and the build's walks read every other row from
the rank that holds it.  The result must be the index lb200_build makes on one GPU with the same rows and batch cap -- the
same file, byte for byte, the same size and build counters -- and the group must search it as a one-GPU index loaded from
that file searches it.

As in tests/test_gpu_group_build.py, rank r runs on device r % device_count(), so every case also runs on a box with one GPU;
rows of other ranks are then still read through the peer path (16-byte loads instead of bulk copies)."""
import os

import numpy as np
import pytest

from util import exact_int_rows, structured

pytestmark = pytest.mark.gpu

# (metric, quant, d, rows): rows "structured" = low-rank float data; "exact" = integer rows whose distances are exact in fp32,
# full of exact ties (tests/test_gpu_build_model.py)
KINDS = [("cos", "f32", 96, "structured"), ("l2sq", "f32", 768, "structured"), ("hamming", "b1", 512, "structured"),
         ("l2sq", "f16", 72, "structured"), ("cos", "i8", 64, "structured"), ("l2sq", "f32", 48, "exact")]
M, EFC, EF = 16, 64, 48


def _data(quant, d, n, rows="structured", metric="l2sq", seed=5):
    if rows == "exact":
        return exact_int_rows(np.random.default_rng(seed), n, d, 8, metric)
    X = structured(n, d, seed=seed)
    if quant == "b1":
        return np.packbits(X > 0, axis=1)
    if quant == "i8":
        return X * 0.3
    return X


def _row_bytes(quant, d):
    raw = {"f32": 4 * d, "f16": 2 * d, "i8": d, "b1": (d + 7) // 8}[quant]
    return (raw + 15) // 16 * 16


def _devices(eng, ranks):
    ndev = eng.device_count()
    return [r % ndev for r in range(ranks)]


def _one_gpu_index(eng, metric, quant, d, build_batch, capacity):
    g = eng.Index(d, metric, quant, M=M, efc=EFC, ef=EF)
    g.set_option("build_batch", build_batch)
    g.reserve(capacity)
    return g


def _group_index(eng, ranks, metric, quant, d, build_batch, capacity, max_batch=512):
    grp = eng.Group.local(_devices(eng, ranks))
    grp.index_init(capacity, d, metric, quant, M=M, efc=EFC, ef=EF, max_batch=max_batch)
    grp.index_set_option("build_batch", build_batch)
    return grp


def _stats(s):
    return s["vectors"], s["computed_distances"]


_ONE_GPU = {}


def _one_gpu(eng, metric, quant, d, rows, n, build_batch):
    key = (metric, quant, d, rows, n, build_batch)
    if key not in _ONE_GPU:
        X = _data(quant, d, n, rows, metric)
        g = _one_gpu_index(eng, metric, quant, d, build_batch, n)
        g.add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
        g.build()
        _ONE_GPU[key] = (g.save_buffer(), _stats(g.last_build_stats()), g.size())
        g.close()
    return _ONE_GPU[key]


@pytest.mark.parametrize("build_batch", [64, 1])
@pytest.mark.parametrize("ranks", [1, 2, 4, 8])
@pytest.mark.parametrize("metric,quant,d,rows", KINDS)
def test_group_index_file_equals_one_gpu_build(eng, metric, quant, d, rows, ranks, build_batch):
    n = 1500 if d < 768 else 800
    capacity = n + 37  # the ranges do not end where the rows do
    ref_file, ref_stats, ref_size = _one_gpu(eng, metric, quant, d, rows, n, build_batch)
    X = _data(quant, d, n, rows, metric)
    keys = np.arange(1, n + 1, dtype=np.uint64)
    grp = _group_index(eng, ranks, metric, quant, d, build_batch, capacity)
    for a, b in ((0, 1), (1, n // 3), (n // 3, n // 3 + 7), (n // 3 + 7, n)):  # several chunks, straddling the ranges
        grp.index_add_batch(keys[a:b], X[a:b])
    assert grp.index_size() == n
    grp.index_build()
    assert grp.index_size() == ref_size == n
    assert _stats(grp.index_last_build_stats()) == ref_stats
    f = grp.index_save_buffer()
    assert len(f) == len(ref_file)
    assert np.array_equal(f, ref_file), int(np.count_nonzero(f != ref_file))
    # no rank holds all rows: each keeps exactly its capacity range
    rb = _row_bytes(quant, d)
    for r in range(ranks):
        info = grp.rank_info(r)
        lo, hi = capacity * r // ranks, capacity * (r + 1) // ranks
        assert (info["rank"], info["world"], info["rows_begin"], info["rows_end"]) == (r, ranks, lo, hi)
        assert info["bytes_rows"] == (hi - lo) * rb
    grp.close()


@pytest.mark.parametrize("ranks", [2, 4])
def test_group_index_incremental_builds_and_searches(eng, ranks):
    """add, build, search, add (partly host-staged in small chunks), build, save: the one-GPU index given the same sequence."""
    metric, quant, d, n = "l2sq", "f32", 48, 3000
    X, Q = _data(quant, d, n, seed=9), structured(100, d, seed=19)
    keys = np.arange(1, n + 1, dtype=np.uint64)
    one = _one_gpu_index(eng, metric, quant, d, 64, n)
    grp = _group_index(eng, ranks, metric, quant, d, 64, n + 100)
    out = []
    for add, search, build in ((one.add_batch, one.search_batch, one.build),
                               (grp.index_add_batch, grp.search_batch, grp.index_build)):
        add(keys[: n // 2], X[: n // 2])
        build()
        first = search(Q, 10, 32)
        for a in range(n // 2, n, 250):
            add(keys[a:a + 250], X[a:a + 250])
        build()
        out.append(first)
    (k1, d1, c1), (kg, dg, cg) = out
    assert np.array_equal(kg, k1) and np.array_equal(dg.view(np.uint32), d1.view(np.uint32)) and np.array_equal(cg, c1)
    assert grp.index_size() == one.size() == n
    assert _stats(grp.index_last_build_stats()) == _stats(one.last_build_stats())
    assert np.array_equal(grp.index_save_buffer(), one.save_buffer())
    grp.close()
    one.close()


@pytest.mark.parametrize("ranks,capacity_factor", [(2, 1), (4, 3)])
def test_group_index_search_equals_one_gpu_search_of_its_file(eng, ranks, capacity_factor):
    """The built group answers as a one-GPU index loaded from its file; at capacity ~3n the last ranks hold no rows yet (and
    the search is what builds the pending rows)."""
    metric, quant, d, n = "cos", "f32", 96, 4000
    X, Q = _data(quant, d, n), structured(300, d, seed=77)
    capacity = capacity_factor * n + 11
    grp = _group_index(eng, ranks, metric, quant, d, 64, capacity)
    grp.index_add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
    kg1, dg1, cg1 = grp.search_batch(Q, 10, 16)  # builds the pending rows first
    assert grp.index_size() == n
    one = eng.Index(d, metric, quant, M=M, efc=EFC, ef=EF)
    one.load_buffer(grp.index_save_buffer())
    for ef, (kg, dg, cg) in ((16, (kg1, dg1, cg1)), (64, grp.search_batch(Q, 10, 64))):
        k1, d1, c1 = one.search_batch(Q, 10, ef)
        assert np.array_equal(kg, k1), ef
        assert np.array_equal(dg.view(np.uint32), d1.view(np.uint32)), ef
        assert np.array_equal(cg, c1), ef
    if capacity_factor > 1:
        empty = [r for r in range(ranks) if grp.rank_info(r)["rows_begin"] >= n]
        assert empty, "some rank should hold no rows yet"
    grp.close()
    one.close()


def test_group_index_save_paths_agree_and_load_everywhere(eng, tmp_path):
    metric, quant, d, n = "l2sq", "f32", 64, 3000
    X, Q = _data(quant, d, n, seed=3), structured(200, d, seed=31)
    grp = _group_index(eng, 4, metric, quant, d, 64, n)
    grp.index_add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
    path = str(tmp_path / "group.usearch")
    grp.index_save(path)  # builds first
    buf = grp.index_save_buffer()
    assert np.array_equal(np.fromfile(path, np.uint8), buf)
    one = eng.Index(d, metric, quant, M=M, efc=EFC, ef=EF)
    one.load(path)
    loaded = eng.Group.local(_devices(eng, 2))
    loaded.load(path, d, metric, quant, M=M, efc=EFC, ef=EF, max_batch=512)
    k1, d1, c1 = one.search_batch(Q, 10, 40)
    for g in (loaded, grp):
        kg, dg, cg = g.search_batch(Q, 10, 40)
        assert np.array_equal(kg, k1) and np.array_equal(dg.view(np.uint32), d1.view(np.uint32)) and np.array_equal(cg, c1)
    loaded.close()
    grp.close()
    one.close()


def test_group_index_refusals_leave_the_group_usable(eng):
    metric, quant, d, n = "l2sq", "f32", 32, 2000
    X = _data(quant, d, n)
    keys = np.arange(1, n + 1, dtype=np.uint64)
    calls = []

    def allgather(send):
        calls.append(len(send))
        raise AssertionError("a refused index_init must not communicate")

    multi = eng.Group.ranked(0, 2, allgather)
    with pytest.raises(eng.EngineError, match="lb200_group_create_local"):
        multi.index_init(n, d, metric, quant)
    assert not calls
    multi.close()

    grp = eng.Group.local(_devices(eng, 2))
    with pytest.raises(eng.EngineError, match="pq"):
        grp.index_init(n, d, metric, quant, pq=True)
    with pytest.raises(eng.EngineError, match="lb200_group_index_init"):
        grp.index_add_batch(keys[:10], X[:10])
    grp.index_init(n, d, metric, quant, M=M, efc=EFC, ef=EF, max_batch=256)  # the refusals above left it free
    grp.index_set_option("build_batch", 64)
    with pytest.raises(eng.EngineError, match="one lb200_group_distribute, lb200_group_load or lb200_group_index_init"):
        grp.index_init(n, d, metric, quant)
    one = _one_gpu_index(eng, metric, quant, d, 64, n)
    with pytest.raises(eng.EngineError, match="already"):
        grp.distribute(one)
    with pytest.raises(eng.EngineError, match="already"):
        grp.load_buffer(np.zeros(200, np.uint8), d, metric, quant)
    with pytest.raises(eng.EngineError, match="unknown option"):
        grp.index_set_option("search_kernel", 2)

    grp.index_add_batch(keys[: n - 100], X[: n - 100])
    with pytest.raises(eng.EngineError, match="capacity"):
        grp.index_add_batch(np.append(keys[n - 100:], n + 1), np.concatenate([X[n - 100:], X[:1]]))  # one row past it
    bad = keys[n - 100:].copy()
    bad[5] = np.iinfo(np.uint64).max
    with pytest.raises(eng.EngineError, match="UINT64_MAX"):
        grp.index_add_batch(bad, X[n - 100:])
    assert grp.index_size() == n - 100  # nothing was added by the refusals
    grp.index_add_batch(keys[n - 100:], X[n - 100:])
    grp.index_build()
    one.add_batch(keys, X)
    one.build()
    assert np.array_equal(grp.index_save_buffer(), one.save_buffer())
    grp.close()
    one.close()
