"""GPU tests of a row-sharded group formed straight from an index file (lb200_group_load / lb200_group_load_buffer): every
rank reads its own rows and the graph from the file bytes, so no GPU ever holds the whole index.  A loaded group answers
exactly as a one-GPU index that loaded the same bytes (ids, distance bits, counts, work counters), gets the row ranges a
distributed group gets, refuses every file Index.load_buffer refuses with the same message, and still takes a correct load
after a refusal.  Ranks share a device when the box has fewer GPUs, as in test_gpu_group.py."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

from test_golden import CUBE, LATTICE, G
from test_gpu_group import _index

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NQ_MAX = 512


def _devices(eng, ranks):
    ndev = eng.device_count()
    return [r % ndev for r in range(ranks)]


def _row_bytes(quant, d):
    vec = {"f32": 4 * d, "f16": 2 * d, "i8": d, "b1": (d + 7) // 8}[quant]
    return (vec + 15) // 16 * 16


def _same(a, b):
    (ka, da, ca), (kb, db, cb) = a, b
    return np.array_equal(ka, kb) and np.array_equal(da.view(np.uint32), db.view(np.uint32)) and np.array_equal(ca, cb)


CASES = [("cos", "f32", 96), ("l2sq", "f32", 768), ("hamming", "b1", 512), ("l2sq", "f16", 72), ("l2sq", "i8", 64)]


@functools.lru_cache(maxsize=None)
def _built(metric, quant, d):
    """(index built on one GPU, its queries, its file bytes): one build per case for the whole module"""
    from lantern_b200 import api
    g, X, Q = _index(api, metric, quant, d, 6000 if d < 768 else 3000)
    return g, len(X), Q, g.save_buffer()


@pytest.mark.parametrize("ranks", [1, 2, 4, 8])
@pytest.mark.parametrize("metric,quant,d", CASES)
def test_loaded_group_equals_one_gpu(eng, ranks, metric, quant, d):
    g, n, Q, buf = _built(metric, quant, d)
    k, ef = 10, 48
    one = g.search_batch(Q, k, ef)
    st1 = g.last_stats()
    grp = eng.Group.local(_devices(eng, ranks))
    grp.load_buffer(buf, d, metric, quant, M=16, efc=64, ef=ef, max_batch=NQ_MAX)
    for rep in range(2):  # the second batch reuses the mailboxes with new flags
        assert _same(grp.search_batch(Q, k, ef), one)
    stats = [grp.last_stats(r) for r in range(ranks)]
    assert sum(s["owner_computed_distances"] for s in stats) == st1["computed_distances"]
    assert sum(s["local_rows_evaluated"] for s in stats) == st1["computed_distances"] - len(Q)
    assert sum(s["rows_held"] for s in stats) == n
    info = [grp.rank_info(r) for r in range(ranks)]
    assert [i["rows_begin"] for i in info] == [0] + [i["rows_end"] for i in info[:-1]] and info[-1]["rows_end"] == n
    assert all(i["bytes_rows"] == (i["rows_end"] - i["rows_begin"]) * _row_bytes(quant, d) for i in info)
    assert len({i["bytes_graph"] for i in info}) == 1
    grp.close()


# index files written by the reference (tests/golden/make_golden.py): name, metric, quant, rows, M, efc, ef, queries, k
GOLDEN = [("cube_l2sq_file", "l2sq", "f32", CUBE, 2, 128, 4, CUBE, 8),
          ("cube_cos_file", "cos", "f32", CUBE, 2, 128, 4, CUBE, 8),
          ("lattice_f32_file", "l2sq", "f32", LATTICE, 12, 64, 32, LATTICE, 5),
          ("lattice_f16_file", "l2sq", "f16", LATTICE, 12, 64, 32, LATTICE, 5),
          ("lattice_i8_file", "l2sq", "i8", LATTICE * 0.25, 12, 64, 32, LATTICE * 0.25, 5),
          ("rand_l2_file", "l2sq", "f32", G["rand_l2_X"], 8, 48, 24, G["rand_l2_Q"], 10),
          ("rand_cos_file", "cos", "f32", G["rand_cos_X"], 6, 40, 20, G["rand_cos_Q"], 10)]


@pytest.mark.parametrize("ranks", [2, 8])
@pytest.mark.parametrize("case", GOLDEN, ids=[c[0] for c in GOLDEN])
def test_reference_written_files(eng, case, ranks):
    """The 8-row cube on 8 ranks leaves some ranks an empty range."""
    name, metric, quant, X, M, efc, ef, Q, k = case
    buf, d = G[name], X.shape[1]
    g = eng.Index(d, metric, quant, M=M, efc=efc, ef=ef)
    g.load_buffer(buf)
    one = g.search_batch(Q, k)
    grp = eng.Group.local(_devices(eng, ranks))
    grp.load_buffer(buf, d, metric, quant, M=M, efc=efc, ef=ef, max_batch=64)
    assert _same(grp.search_batch(Q, k), one)
    assert sum(grp.rank_info(r)["rows_end"] - grp.rank_info(r)["rows_begin"] for r in range(ranks)) == len(X)
    grp.close()


@pytest.mark.parametrize("M", [32, 48])
def test_planted_duplicate_ids(eng, M):
    """Lists with repeated ids, as refine_'s stale padding leaves them (test_gpu_group.py::test_group_wide_lists)."""
    g, X, Q = _index(eng, "cos", "f32", 64, 5000, M=M, efc=96, ef=64)
    buf = g.save_buffer().copy()
    off, planted = 136, 0
    for i in range(len(X)):
        lvl = int(np.frombuffer(buf, np.int16, 1, off + 8)[0])
        base = off + 10
        cnt = int(np.frombuffer(buf, np.uint32, 1, base)[0])
        if i % 7 == 0 and cnt >= 40:
            ids = buf[base + 4: base + 4 + 6 * cnt].reshape(cnt, 6)
            ids[cnt - 1] = ids[2]
            ids[5] = ids[4]
            planted += 1
        off = base + 4 + 12 * M + lvl * (4 + 6 * M) + 64 * 4
    assert planted > 50
    g2 = eng.Index(64, "cos", "f32", M=M, efc=96, ef=64)
    g2.load_buffer(buf)
    one = g2.search_batch(Q, 10, 64)
    total = g2.last_stats()["computed_distances"]
    for ranks in (2, 3):
        grp = eng.Group.local(_devices(eng, ranks))
        grp.load_buffer(buf, 64, "cos", "f32", M=M, efc=96, ef=64, max_batch=NQ_MAX)
        assert _same(grp.search_batch(Q, 10, 64), one)
        assert sum(grp.last_stats(r)["owner_computed_distances"] for r in range(ranks)) == total
        grp.close()


@pytest.mark.parametrize("ranks", [2, 3, 8])
def test_ranges_and_bytes_match_distribute(eng, ranks):
    g, n, Q, buf = _built("l2sq", "f32", 768)
    src = eng.Index(768, "l2sq", "f32", M=16, efc=64, ef=48)
    src.load_buffer(buf)
    dist = eng.Group.local(_devices(eng, ranks))
    dist.distribute(src, root=0, max_batch=NQ_MAX)
    load = eng.Group.local(_devices(eng, ranks))
    load.load_buffer(buf, 768, "l2sq", "f32", M=16, efc=64, ef=48, max_batch=NQ_MAX)
    a = [dist.rank_info(r) for r in range(ranks)]
    b = [load.rank_info(r) for r in range(ranks)]
    assert a == b  # same ranges, and the same bytes in every category
    assert b[0]["rows_begin"] == 0 and b[-1]["rows_end"] == n
    assert all(x["rows_end"] == y["rows_begin"] for x, y in zip(b, b[1:]))
    assert all(i["bytes_rows"] == (i["rows_end"] - i["rows_begin"]) * 768 * 4 for i in b)
    assert len({i["bytes_graph"] for i in b}) == 1 and all(i["rank"] == r and i["world"] == ranks for r, i in enumerate(b))
    assert _same(load.search_batch(Q, 10, 48), dist.search_batch(Q, 10, 48))
    dist.close(), load.close()


def _tapes(buf, M, stored):
    """(offset, level) of every node tape of a lantern-storage file"""
    n = int(np.frombuffer(buf, np.uint64, 1, 80)[0])
    out, off = [], 136
    for _ in range(n):
        lvl = int(np.frombuffer(buf, np.int16, 1, off + 8)[0])
        out.append((off, lvl))
        off += 10 + 4 + 12 * M + lvl * (4 + 6 * M) + stored
    return out


def _put_id(buf, at, v):
    buf[at: at + 6] = np.frombuffer(int(v).to_bytes(6, "little"), np.uint8)


def test_refusals_then_a_correct_load(eng):
    d, M = 32, 8
    g, X, Q = _index(eng, "l2sq", "f32", d, 1500, M=M, efc=32, ef=16)
    good = g.save_buffer()
    n = len(X)
    opts = dict(M=M, efc=32, ef=16)
    tapes = _tapes(good, M, 4 * d)
    bad = {}
    b = good.copy()
    b[0] = ord("x")
    bad["bad magic"] = b
    for cut in (100, 136 + 5, 136 + 10 + 7, len(good) // 2, len(good) - 1):
        bad["truncated at %d" % cut] = good[:cut].copy()
    b = good.copy()
    _put_id(b, tapes[3][0] + 10 + 4, n + 5)
    bad["slot out of range"] = b
    b = good.copy()
    b[112:120] = np.frombuffer(np.uint64(n + 1).tobytes(), np.uint8)
    bad["entry slot out of range"] = b
    up = next(i for i, (off, lvl) in enumerate(tapes) if lvl >= 1 and
              int(np.frombuffer(good, np.uint32, 1, off + 10 + 4 + 12 * M)[0]) > 0)
    flat = next(i for i, (off, lvl) in enumerate(tapes) if lvl == 0)
    b = good.copy()
    _put_id(b, tapes[up][0] + 10 + 4 + 12 * M + 4, flat)
    bad["link to a node missing on its level"] = b
    cases = [(name, buf, d, "l2sq", opts) for name, buf in bad.items()]
    cases += [("metric", good, d, "cos", opts), ("dims", good, d + 1, "l2sq", opts),
              ("connectivity", good, d, "l2sq", dict(opts, M=12))]
    # a PQ file: refused as distribute refuses PQ indexes, and with plain options as Index.load_buffer refuses it
    cb = np.random.default_rng(4).standard_normal((16, d)).astype(np.float32)
    pq = eng.Index(d, "l2sq", "f32", M=M, efc=32, ef=16, pq=True, num_centroids=16, num_subvectors=4, codebook=cb)
    pq.reserve(300)
    pq.add_batch(np.arange(300, dtype=np.uint64), X[:300])
    pq.build()
    pq_file = pq.save_buffer()
    cases.append(("pq file, plain options", pq_file, d, "l2sq", opts))

    grp = eng.Group.local(_devices(eng, 2))
    with pytest.raises(eng.EngineError, match="distribute"):
        grp.search_batch(Q, 5)  # nothing loaded yet
    with pytest.raises(eng.EngineError, match="load"):
        grp.rank_info(0)
    for name, buf, dim, metric, o in cases:
        with pytest.raises(eng.EngineError) as want:
            eng.Index(dim, metric, "f32", **o).load_buffer(buf)
        with pytest.raises(eng.EngineError) as got:
            grp.load_buffer(buf, dim, metric, "f32", max_batch=NQ_MAX, **o)
        assert str(got.value) == str(want.value), name
    with pytest.raises(eng.EngineError, match="pq indexes are not supported"):
        grp.load_buffer(pq_file, d, "l2sq", "f32", pq=True, max_batch=NQ_MAX, **opts)
    # after every refusal the group still takes a correct load, and answers as one GPU does
    grp.load_buffer(good, d, "l2sq", "f32", max_batch=NQ_MAX, **opts)
    assert _same(grp.search_batch(Q, 10), g.search_batch(Q, 10))
    with pytest.raises(eng.EngineError, match="already distributed"):
        grp.load_buffer(good, d, "l2sq", "f32", max_batch=NQ_MAX, **opts)
    grp.close()
    grp = eng.Group.local(_devices(eng, 2))
    grp.distribute(g, root=0, max_batch=NQ_MAX)
    with pytest.raises(eng.EngineError, match="already distributed"):
        grp.load_buffer(good, d, "l2sq", "f32", max_batch=NQ_MAX, **opts)
    grp.close()


def test_load_from_path(eng, tmp_path):
    g, n, Q, buf = _built("cos", "f32", 96)
    path = str(tmp_path / "idx.usearch")
    g.save(path)
    grp = eng.Group.local(_devices(eng, 4))
    with pytest.raises(eng.EngineError, match="Can't open file"):
        grp.load(str(tmp_path / "missing.usearch"), 96, "cos", "f32", M=16, efc=64, ef=48)
    grp.load(path, 96, "cos", "f32", M=16, efc=64, ef=48, root=1, max_batch=NQ_MAX)
    assert _same(grp.search_batch(Q, 10, 48), g.search_batch(Q, 10, 48))
    grp.close()


def _multi_process(eng, tmp_path, world, mode, port):
    d, n = 128, 8000
    files = []
    for seed in (21, 31):  # same options and size, different rows and graph
        g, X, Q = _index(eng, "cos", "f32", d, n, M=16, efc=64, ef=64, seed=seed)
        path = str(tmp_path / ("idx_%d.usearch" % seed))
        g.save(path)
        files.append(path)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "group_load_rank.py"), files[0], files[1], mode]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=dict(os.environ, MASTER_ADDR="127.0.0.1"))
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    assert out.stdout.count("group load rank ok") == world, out.stdout
    assert out.stdout.count("different file refused") == world, out.stdout


def test_group_load_multi_process(eng, tmp_path):
    """One process per GPU (torchrun): every rank maps the same file, keeps its own range and searches collectively; a rank
    given a different file fails the call on every rank."""
    if eng.device_count() < 2:
        pytest.skip("needs two CUDA devices (processes cannot run kernels concurrently on one GPU)")
    _multi_process(eng, tmp_path, min(4, eng.device_count()), "search", 29743)


def test_group_load_multi_process_exchanges(eng, tmp_path):
    """The load's exchanges between processes (file check, mailbox handles over CUDA IPC, the mapped tick) need no kernel of
    the group: two processes may share one device.  Ranges equal a single-process group's; a different file fails everywhere."""
    _multi_process(eng, tmp_path, 2, "load", 29745)
