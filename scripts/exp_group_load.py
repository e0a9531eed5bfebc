"""Experiment: a row-sharded group formed straight from an index file (lb200_group_load) against the same group formed by
loading the file on device 0 and distributing it (lb200_group_distribute).  Writes a cfg3s-sized file once (1M x d768 f32
cosine, M=32), then for each group size G: per-device free memory (cudaMemGetInfo) before and after each path, load time,
lb200_group_rank_info bytes, search queries/s of both paths in the same run (alternated), and whether their outputs are
identical.  Meant for a box with >= 2 GPUs; with fewer devices than ranks, ranks share devices (a rehearsal: the memory figures
are then per physical device, and the rates are not multi-GPU rates).
    python scripts/exp_group_load.py [G list, default 2,4,8] [n, default 1000000] [file directory, default a temporary one]"""
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from lantern_b200 import api  # noqa: E402

sizes = [int(x) for x in (sys.argv[1] if len(sys.argv) > 1 else "2,4,8").split(",")]
n = int(sys.argv[2]) if len(sys.argv) > 2 else 1_000_000
tmp = tempfile.TemporaryDirectory(dir=sys.argv[3] if len(sys.argv) > 3 else None)
dim, metric, M, efc, ef, B, k, reps = 768, "cos", 32, 128, 128, 4096, 10, 5
opts = dict(metric=metric, quant="f32", M=M, efc=efc, ef=ef)
ndev = api.device_count()
if ndev < 1:
    raise SystemExit("no CUDA device")
for d in range(ndev):
    torch.cuda.set_device(d)
    torch.zeros(1, device="cuda")  # the torch context on every device before any memory figure is taken
torch.cuda.set_device(0)
props = torch.cuda.get_device_properties(0)
print("devices: %d x %s" % (ndev, props.name), flush=True)
try:
    print(subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                         text=True, timeout=60).stdout.strip(), flush=True)
except (OSError, subprocess.SubprocessError) as e:
    print("nvidia-smi unavailable:", e)

dev = torch.device("cuda", 0)
path = os.path.join(tmp.name, "cfg3s.usearch")
t0 = time.perf_counter()
X = bench.structured_torch(n, dim, 42, dev)
g = api.Index(dim, **opts)
g.reserve(n)
g.add_batch_device(np.arange(1, n + 1, dtype=np.uint64), X.data_ptr(), n, dim * 4, "f32")
g.build()
g.save(path)
Q = bench.structured_torch(B, dim, 43, dev).cpu().numpy()
del X
g.close()
torch.cuda.synchronize()
torch.cuda.empty_cache()
print("file: %d rows, %.2f GB, written in %.1f s" % (n, os.path.getsize(path) / 1e9, time.perf_counter() - t0), flush=True)


def free_mb(devs):
    return [torch.cuda.mem_get_info(d)[0] / 1e6 for d in sorted(set(devs))]


def used(before, after):
    return " ".join("%.0f" % (b - a) for b, a in zip(before, after))


for G in sizes:
    devs = [r % ndev for r in range(G)]
    shared = " (ranks share devices)" if G > ndev else ""
    print("== G = %d on devices %s%s" % (G, sorted(set(devs)), shared), flush=True)
    m0 = free_mb(devs)
    t0 = time.perf_counter()
    gl = api.Group.local(devs)
    gl.load(path, dim, root=0, max_batch=B, **opts)
    t_load = time.perf_counter() - t0
    m1 = free_mb(devs)
    for r in range(G):
        i = gl.rank_info(r)
        print("  load rank %d: rows [%d, %d)  MB rows %.0f graph %.0f scratch %.0f mailbox %.0f" % (
            r, i["rows_begin"], i["rows_end"], i["bytes_rows"] / 1e6, i["bytes_graph"] / 1e6, i["bytes_scratch"] / 1e6,
            i["bytes_mailbox"] / 1e6), flush=True)
    print("  load: %.1f s; device MB taken per device %s" % (t_load, used(m0, m1)), flush=True)
    t0 = time.perf_counter()
    torch.cuda.set_device(0)
    src = api.Index(dim, **opts)
    src.load(path)
    gd = api.Group.local(devs)
    gd.distribute(src, root=0, max_batch=B)
    t_dist = time.perf_counter() - t0
    m2 = free_mb(devs)
    print("  lb200_load on device 0 + distribute: %.1f s; device MB taken per device %s (the source index stays resident)" % (
        t_dist, used(m1, m2)), flush=True)
    ol, od = gl.search_batch(Q, k, ef), gd.search_batch(Q, k, ef)  # warm-up of both, and the outputs compared
    same = all(np.array_equal(a.view(np.uint32) if a.dtype == np.float32 else a, b.view(np.uint32) if b.dtype == np.float32 else b)
               for a, b in zip(ol, od))
    tl, td = [], []
    for rep in range(reps):  # alternated
        for grp, acc in ((gl, tl), (gd, td)):
            t0 = time.perf_counter()
            grp.search_batch(Q, k, ef)
            acc.append(time.perf_counter() - t0)
    print("  search %d queries: loaded group %.0f q/s, distributed group %.0f q/s (median of %d, host buffers in/out); "
          "identical keys, distance bits and counts: %s" % (B, B / np.median(tl), B / np.median(td), reps, same), flush=True)
    gl.close(), gd.close(), src.close()
    torch.cuda.synchronize()
tmp.cleanup()
