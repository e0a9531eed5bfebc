"""Dev experiment: the group build (lb200_group_build) on 1, 2, 4 and 8 GPUs of one box (needs GPUs).

Builds a workload's corpus (bench.py's generator and seeds) with default settings on G GPUs for each G in GPUS that the box
has, timing each build with the host clock around a synchronised call.  Prints wall seconds, vectors/s, the speedup over
one GPU, the batch count and cap of the schedule, and the summed computed_distances.  Then:
  - same graph: the largest group and one GPU build with the same explicit build_batch (= that group's default cap) and
    the two files are compared by SHA-256;
  - recall@10 at the workload's ef of the default largest-group graph and the default one-GPU graph, against exhaustive
    ground truth (lb200_exact_search_device).
The per-GPU default cap is one node per resident insert CTA: CAP1 (default 1056 = 8 CTAs x 132 SMs at d768).
With GPUS=1 only the existing one-GPU API is used, so the same run also works against an older library; HASH=1 adds the
SHA-256 of every default build's file.
usage: python scripts/exp_group_build.py [workload] ; env GPUS (default 1,2,4,8), HASH, OUT (directory for the JSON)"""
import hashlib, json, math, os, subprocess, sys, time
sys.path.insert(0, '.')
import numpy as np, torch
import bench
from lantern_b200 import api

wl_name = sys.argv[1] if len(sys.argv) > 1 else "cfg3s"
wl = bench.WORKLOADS[wl_name]
n, dim, k, ef, M = wl["n"], wl["dim"], wl["k"], wl["ef"], wl["M"]
ndev = api.device_count()
gpus = [g for g in (int(x) for x in os.environ.get("GPUS", "1,2,4,8").split(",")) if g <= ndev]
cap1 = int(os.environ.get("CAP1", "1056"))
dev = torch.device("cuda", 0)
X = bench.structured_torch(n, dim, bench.SEED_CORPUS, dev)
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()


def schedule(cap, ratio=64):
    """Batch count of the build schedule (csrc/build.cu plan_batches), from the same level generator."""
    state, top, visible, pos, batches = 1, -1, 0, 0, 0
    levels = np.empty(n, np.int32)
    inv = 1.0 / math.log(M)
    Rr = 2147483646.0
    for i in range(n):
        state = state * 16807 % 2147483647
        a = state - 1
        state = state * 16807 % 2147483647
        u = (a + (state - 1) * Rr) / (Rr * Rr)
        u = min(u, math.nextafter(1.0, 0.0))
        levels[i] = int(-math.log(u) * inv)
    top, visible, pos = int(levels[0]), 1, 1
    while pos < n:
        bsz = 1
        if levels[pos] <= top:
            bsz = min(n - pos, cap, max(1, visible // ratio))
            above = np.nonzero(levels[pos + 1: pos + bsz] > top)[0]
            if len(above):
                bsz = int(above[0]) + 1
        if levels[pos] > top:
            top = int(levels[pos])
        visible += bsz
        pos += bsz
        batches += 1
    return batches


def build(G, build_batch=0, save=False):
    idx = api.Index(dim, wl["metric"], "f32", M=M, efc=wl["efc"], ef=ef)
    idx.reserve(n)
    if build_batch:
        idx.set_option("build_batch", build_batch)
    idx.add_batch_device(np.arange(1, n + 1, dtype=np.uint64), X.data_ptr(), n, dim * 4, "f32")
    torch.cuda.synchronize()
    t = time.perf_counter()
    if G == 1:
        idx.build()
    else:
        grp = api.Group.local(list(range(G)))
        grp.build(idx)
        grp.close()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t
    st = idx.last_build_stats()
    digest = hashlib.sha256(idx.save_buffer().tobytes()).hexdigest() if save else None
    return idx, wall, st, digest


out = {"workload": wl_name, "n": n, "gpus_on_box": ndev, "cards": smi, "builds": {}}
base = None
for G in gpus:
    idx, wall, st, digest = build(G, save=os.environ.get("HASH") == "1")
    idx.close()
    base = base or wall
    cap = G * cap1
    row = {"wall_s": wall, "vectors_per_s": n / wall, "speedup": base / wall, "cap": cap, "batches": schedule(cap),
           "computed_distances": st["computed_distances"], "device_ms": st["device_ms"], "sha256": digest}
    out["builds"][G] = row
    print(G, "GPU", json.dumps(row), flush=True)
if len(gpus) > 1:
    G = gpus[-1]
    a, _, _, ha = build(G, G * cap1, save=True)
    a.close()
    b, _, _, hb = build(1, G * cap1, save=True)
    b.close()
    out["same_graph"] = {"gpus": G, "build_batch": G * cap1, "sha256_group": ha, "sha256_one": hb, "identical": ha == hb}
    print(json.dumps(out["same_graph"]), flush=True)
    nq = 4096
    Q = bench.structured_torch(nq, dim, bench.SEED_QUERY, dev)
    tk = torch.empty((nq, k), dtype=torch.int64, device=dev)
    td = torch.empty((nq, k), dtype=torch.float32, device=dev)
    api.exact_search_device(X.data_ptr(), n, dim * 4, Q.data_ptr(), nq, dim * 4, k, tk.data_ptr(), td.data_ptr(), wl["metric"], "f32", dim)
    torch.cuda.synchronize()
    truth = tk.cpu().numpy().astype(np.uint64) + 1
    rec = {}
    for g in (1, G):
        idx, _, _, _ = build(g)
        keys, _, _ = idx.search_batch(Q.cpu().numpy(), k, ef)
        rec[g] = float(np.mean([len(set(a.tolist()) & set(b.tolist())) / k for a, b in zip(keys, truth)]))
        idx.close()
    out["recall_at_10"] = {"one_gpu": rec[1], "group": rec[G], "gate_holds": rec[G] >= rec[1] - 0.005}
    print(json.dumps(out["recall_at_10"]), flush=True)
print(json.dumps(out))
if os.environ.get("OUT"):
    os.makedirs(os.environ["OUT"], exist_ok=True)
    with open(os.path.join(os.environ["OUT"], "exp_group_build_%s.json" % wl_name), "w") as f:
        json.dump(out, f, indent=1)
