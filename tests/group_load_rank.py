"""One rank of tests/test_gpu_group_load.py (launched by torchrun with two index files of the same options and a mode): every
rank loads the first file into a multi-process group; mode "search" checks the collective search against the rank's own
one-GPU search of the same file, mode "load" (ranks may share a device: no kernel of the group runs) checks the ranges against
those of a single-process group.  Then a group whose last rank is given the second file must fail on every rank."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from lantern_b200 import api  # noqa: E402
from util import structured  # noqa: E402

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
dist.init_process_group("gloo")
torch.cuda.set_device(local % torch.cuda.device_count())
path, other, mode = sys.argv[1], sys.argv[2], sys.argv[3]


def allgather(send):
    outs = [None] * world
    dist.all_gather_object(outs, send)
    return b"".join(outs)


d, nq, k, ef = 128, 256, 10, 64
opts = dict(metric="cos", quant="f32", M=16, efc=64, ef=ef)
Q = structured(nq, d, seed=12)
idx = api.Index(d, "cos", "f32", M=16, efc=64, ef=ef)
idx.load(path)
k1, d1, c1 = idx.search_batch(Q, k, ef)
total = idx.last_stats()["computed_distances"]
n = idx.size()
idx.close()

grp = api.Group.ranked(rank, world, allgather)
grp.load(path, d, root=0, max_batch=nq, **opts)
info = grp.rank_info()
ranges = [None] * world
dist.all_gather_object(ranges, (info["rows_begin"], info["rows_end"]))
assert [r[0] for r in ranges] == [0] + [r[1] for r in ranges[:-1]] and ranges[-1][1] == n, ranges
assert info["bytes_rows"] == (info["rows_end"] - info["rows_begin"]) * d * 4 and info["rank"] == rank and info["world"] == world
if mode == "search":
    keys, dists, counts = grp.search_batch(Q if rank == 0 else None, k, ef, nq=nq, dim_bytes=d * 4, kind="f32")
    assert np.array_equal(keys, k1) and np.array_equal(dists.view(np.uint32), d1.view(np.uint32)), float(np.mean(keys == k1))
    assert np.array_equal(counts, c1)
    st = grp.last_stats()
    evals = [None] * world
    dist.all_gather_object(evals, (st["owner_computed_distances"], st["local_rows_evaluated"]))
    assert sum(e[0] for e in evals) == total and sum(e[1] for e in evals) == total - nq, (evals, total)
    assert 0 < st["rows_held"] < n
else:
    one = api.Group.local([torch.cuda.current_device()] * world)
    one.load(path, d, root=0, max_batch=nq, **opts)
    assert info == one.rank_info(rank), (info, one.rank_info(rank))
    one.close()
print("group load rank ok %d/%d: rows [%d, %d)" % (rank, world, info["rows_begin"], info["rows_end"]))
grp.close()

grp = api.Group.ranked(rank, world, allgather)
try:
    grp.load(other if rank == world - 1 else path, d, root=0, max_batch=nq, **opts)
    refused = False
except api.EngineError as e:
    refused = "different index files" in str(e)
assert refused
print("different file refused %d/%d" % (rank, world))
grp.close()
dist.destroy_process_group()
