"""GPU tests of the group build (lb200_group_build, csrc/build.cu + csrc/group.cu): the ranks of a single-process group share
every batch of the insertion, each on its own replica of the graph, and the result must be the graph lb200_build makes on one
GPU with the same batch cap -- the same file, byte for byte, and the same work counters.

As in tests/test_gpu_group.py, several ranks may share one physical device (devices = [r % ndev ...]), so every case also runs
on a box with a single GPU; the replicas, the write-through stores and the cross-rank barriers are exercised all the same."""
import os
import socket
import subprocess
import time

import numpy as np
import pytest

from test_golden import LATTICE, PQ_CODEBOOK, int_bits
from test_gpu_server import session
from util import recall, structured

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SERVER = os.path.join(ROOT, "lantern_b200", "lb200_index_server")

KINDS = [("cos", "f32", 96), ("l2sq", "f32", 768), ("hamming", "b1", 512), ("l2sq", "f16", 72), ("cos", "i8", 64),
         ("l2sq", "pq", 32)]


def _data(quant, d, n, seed=5):
    X = structured(n, d, seed=seed)
    if quant == "b1":
        return np.packbits(X > 0, axis=1)
    if quant == "i8":
        return X * 0.3
    return X


def _index(eng, metric, quant, d, build_batch=None, M=16, efc=64, ef=48, capacity=0):
    if quant == "pq":
        cb = np.random.default_rng(11).standard_normal((64, d)).astype(np.float32)
        g = eng.Index(d, metric, "f32", M=M, efc=efc, ef=ef, pq=True, num_centroids=64, num_subvectors=8, codebook=cb)
    else:
        g = eng.Index(d, metric, quant, M=M, efc=efc, ef=ef)
    if build_batch is not None:
        g.set_option("build_batch", build_batch)
    if capacity:
        g.reserve(capacity)
    return g


def _devices(eng, ranks):
    ndev = eng.device_count()
    return [r % ndev for r in range(ranks)]  # several ranks per device when the box has fewer GPUs


def _stats(g):
    s = g.last_build_stats()
    return s["vectors"], s["computed_distances"]


_ONE_GPU = {}


def _one_gpu(eng, metric, quant, d, n, build_batch):
    """File and build counters of the one-GPU build of the same rows (shared by the rank counts)."""
    key = (metric, quant, d, n, build_batch)
    if key not in _ONE_GPU:
        X = _data(quant, d, n)
        g = _index(eng, metric, quant, d, build_batch, capacity=n)
        g.add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
        g.build()
        _ONE_GPU[key] = (g.save_buffer(), _stats(g), g.size())
        g.close()
    return _ONE_GPU[key]


@pytest.mark.parametrize("build_batch", [64, 1])
@pytest.mark.parametrize("ranks", [1, 2, 4, 8])
@pytest.mark.parametrize("metric,quant,d", KINDS)
def test_group_build_file_equals_one_gpu_build(eng, metric, quant, d, ranks, build_batch):
    n = 6000 if d < 768 else 3000
    ref_file, ref_stats, ref_size = _one_gpu(eng, metric, quant, d, n, build_batch)
    X = _data(quant, d, n)
    g = _index(eng, metric, quant, d, build_batch, capacity=n)
    g.add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
    grp = eng.Group.local(_devices(eng, ranks))
    grp.build(g, root=0)
    assert g.size() == ref_size == n
    assert _stats(g) == ref_stats
    f = g.save_buffer()
    assert len(f) == len(ref_file)
    assert np.array_equal(f, ref_file), int(np.count_nonzero(f != ref_file))
    grp.close()
    g.close()


def test_group_build_incremental_on_a_non_zero_root(eng):
    """First half built on one GPU, second half (a batch plus staged single rows) built by a group whose rank 1 holds the index."""
    metric, quant, d, n = "l2sq", "f32", 48, 5000
    X = _data(quant, d, n + 40, seed=9)
    keys = np.arange(1, n + 41, dtype=np.uint64)

    def grow(g, build_second):
        g.add_batch(keys[: n // 2], X[: n // 2])
        g.build()
        g.add_batch(keys[n // 2: n], X[n // 2: n])
        for i in range(n, n + 40):  # staged on the host, flushed by the build
            g.add(keys[i], X[i])
        build_second(g)
        return g

    one = grow(_index(eng, metric, quant, d, 64, capacity=n + 40), lambda g: g.build())
    ndev = eng.device_count()
    grp = eng.Group.local([1 % ndev, 0])  # rank 1 is device 0, where the index lives
    two = grow(_index(eng, metric, quant, d, 64, capacity=n + 40), lambda g: grp.build(g, root=1))
    assert two.size() == one.size() == n + 40
    assert _stats(two) == _stats(one)
    assert np.array_equal(two.save_buffer(), one.save_buffer())
    grp.close()


@pytest.mark.parametrize("ranks", [2, 4])
def test_group_build_then_distribute_and_search(eng, ranks):
    metric, quant, d, n = "cos", "f32", 96, 6000
    X, Q = _data(quant, d, n), structured(300, d, seed=77)
    one = _index(eng, metric, quant, d, 64, capacity=n)
    one.add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
    one.build()
    k1, d1, c1 = one.search_batch(Q, 10, 48)
    g = _index(eng, metric, quant, d, 64, capacity=n)
    g.add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
    grp = eng.Group.local(_devices(eng, ranks))
    grp.build(g, root=0)
    grp.distribute(g, root=0, max_batch=512)
    kg, dg, cg = grp.search_batch(Q, 10, 48)
    assert np.array_equal(kg, k1)
    assert np.array_equal(dg.view(np.uint32), d1.view(np.uint32))
    assert np.array_equal(cg, c1)
    grp.close()


def test_group_build_default_cap_keeps_recall(eng):
    """Default settings: the group's batches are up to 8x larger than one GPU's; recall must not suffer for it."""
    d, n = 32, 100_000
    X, Q = structured(n, d, seed=21), structured(1000, d, seed=22)
    truth, _ = eng.exact_search(X, Q, 10, "l2sq")
    rec = []
    for build in ("one", "group"):
        g = eng.Index(d, "l2sq", "f32", M=16, efc=128, ef=64)
        g.reserve(n)
        g.add_batch(np.arange(n, dtype=np.uint64), X)
        if build == "one":
            g.build()
        else:
            grp = eng.Group.local(_devices(eng, 8))
            grp.build(g)
            grp.close()
        assert g.size() == n
        k, _, _ = g.search_batch(Q, 10, 64)
        rec.append(recall(k, truth))
        g.close()
    assert rec[1] >= rec[0] - 0.005, rec


def test_group_build_refusals(eng):
    d, n = 32, 2000
    X = _data("f32", d, n)
    g = _index(eng, "l2sq", "f32", d, 64, capacity=n)
    g.add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
    calls = []

    def allgather(send):
        calls.append(len(send))
        raise AssertionError("a refused build must not communicate")

    multi = eng.Group.ranked(0, 2, allgather)  # lb200_group_create: one process per GPU
    with pytest.raises(eng.EngineError, match="lb200_group_create_local"):
        multi.build(g)
    assert not calls
    multi.close()
    grp = eng.Group.local(_devices(eng, 2))
    for root in (-1, 2):
        with pytest.raises(eng.EngineError, match="root"):
            grp.build(g, root=root)
    assert g.size() == n  # nothing was inserted or dropped by the refusals
    single = eng.Group.ranked(0, 1, allgather)  # a world-1 lb200_group_create group holds its only rank: accepted
    single.build(g)
    assert not calls
    built = g.save_buffer()
    one = _index(eng, "l2sq", "f32", d, 64, capacity=n)
    one.add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
    one.build()
    assert np.array_equal(built, one.save_buffer())
    grp.build(g)  # nothing pending: no-op
    assert np.array_equal(g.save_buffer(), built)
    single.close()
    if eng.device_count() >= 2:
        other = eng.Group.local([1, 0])
        g.add_batch(np.array([n + 1], np.uint64), X[:1])
        with pytest.raises(eng.EngineError, match="device"):
            other.build(g, root=0)  # the index lives on device 0, rank 0 is device 1
        other.close()
    grp.close()


def _start_server(port, *extra):
    p = subprocess.Popen([SERVER, "--port", str(port), "--quiet", *extra])
    for _ in range(100):
        try:
            socket.create_connection(("127.0.0.1", port), timeout=0.2).close()
            break
        except OSError:
            time.sleep(0.1)
    return p


def test_index_server_builds_on_a_device_group(eng):
    """The 14-point lattice conversations of tests/test_gpu_server.py against `--devices`: the same file bytes."""
    ndev = eng.device_count()
    devices = "0,1" if ndev >= 2 else "0,0"
    servers = [_start_server(7994), _start_server(7995, "--devices", devices)]
    try:
        files = []
        for port in (7994, 7995):
            out = []
            rows = [(i, v.astype(np.float32).tobytes()) for i, v in enumerate(LATTICE)]
            out.append(session(port, (0, 3, 1, 3, 12, 64, 32, 0, 0, 14, 32), rows))
            bits = int_bits(LATTICE)
            out.append(session(port, (0, 8, 5, 96, 12, 64, 32, 0, 0, 14, 1), [(i, bits[i].tobytes()) for i in range(14)]))
            Xp = (LATTICE * 0.1).astype(np.float32)
            out.append(session(port, (1, 3, 1, 3, 12, 64, 32, 4, 3, 14, 32), [(i, v.tobytes()) for i, v in enumerate(Xp)],
                               codebook=PQ_CODEBOOK))
            R = np.random.default_rng(1).standard_normal((300, 8)).astype(np.float32)
            out.append(session(port, (0, 3, 1, 8, 8, 32, 16, 0, 0, 10, 32), [(i + 1, v.tobytes()) for i, v in enumerate(R)]))
            files.append(out)
        for (c1, f1), (c2, f2) in zip(*files):
            assert c1 == c2 and isinstance(f1, np.ndarray) and np.array_equal(f1, f2)
    finally:
        for p in servers:
            p.terminate()
            p.wait(timeout=10)
