"""Dev experiment: a group's own row-sharded index (lb200_group_index_*) against lb200_build (needs a GPU).

Builds a workload's corpus (bench.py's generator and seeds; default cfg3s = 1M x d768 cos, M=32) once with lb200_build on one
GPU and once per G in GPUS with lb200_group_index_init / _add_batch / _build on a single-process group whose rank r runs on
device r % device_count(), all with the same explicit build_batch (BATCH, default 1056 = the one-GPU default cap at d768).
Prints, per build: wall seconds (host clock around a synchronised call; the group's time excludes adding the rows), the
rank_info bytes of every rank (rows, graph, scratch, mailbox), and whether the saved file is identical to the one-GPU file
(SHA-256).  It also records the card, its power limit, and whether ranks shared a device: rates of ranks that share one
device are not multi-GPU rates.
usage: python scripts/exp_group_index.py [workload] ; env GPUS (default 1,2,4,8), BATCH, N (rows, default the workload's),
OUT (directory for the JSON)"""
import hashlib, json, os, subprocess, sys, time
sys.path.insert(0, '.')
import numpy as np, torch
import bench
from lantern_b200 import api

wl_name = sys.argv[1] if len(sys.argv) > 1 else "cfg3s"
wl = bench.WORKLOADS[wl_name]
n = int(os.environ.get("N", wl["n"]))
dim, ef, M, metric = wl["dim"], wl["ef"], wl["M"], wl["metric"]
batch = int(os.environ.get("BATCH", "1056"))
gpus = [int(x) for x in os.environ.get("GPUS", "1,2,4,8").split(",")]
ndev = api.device_count()
X = bench.structured_torch(n, dim, bench.SEED_CORPUS, torch.device("cuda", 0)).cpu().numpy()
keys = np.arange(1, n + 1, dtype=np.uint64)
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip().splitlines()


def sha(buf):
    return hashlib.sha256(np.ascontiguousarray(buf).tobytes()).hexdigest()


out = {"workload": wl_name, "n": n, "build_batch": batch, "gpus_on_box": ndev, "cards": smi, "builds": {}}
one = api.Index(dim, metric, "f32", M=M, efc=wl["efc"], ef=ef)
one.reserve(n)
one.set_option("build_batch", batch)
one.add_batch(keys, X)
torch.cuda.synchronize()
t = time.perf_counter()
one.build()
torch.cuda.synchronize()
ref = sha(one.save_buffer())
out["one_gpu"] = {"wall_s": time.perf_counter() - t, "computed_distances": one.last_build_stats()["computed_distances"],
                  "sha256": ref}
one.close()
print("lb200_build", json.dumps(out["one_gpu"]), flush=True)
for G in gpus:
    devices = [r % ndev for r in range(G)]
    grp = api.Group.local(devices)
    grp.index_init(n, dim, metric, "f32", M=M, efc=wl["efc"], ef=ef, max_batch=wl["batch"])
    grp.index_set_option("build_batch", batch)
    grp.index_add_batch(keys, X)
    torch.cuda.synchronize()
    t = time.perf_counter()
    grp.index_build()
    wall = time.perf_counter() - t
    h = sha(grp.index_save_buffer())
    row = {"wall_s": wall, "shared_device": len(set(devices)) < G, "devices": devices,
           "computed_distances": grp.index_last_build_stats()["computed_distances"],
           "rank_info": [grp.rank_info(r) for r in range(G)], "identical_to_one_gpu": h == ref}
    grp.close()
    out["builds"][G] = row
    print(G, "ranks", json.dumps(row), flush=True)
print(json.dumps(out))
if os.environ.get("OUT"):
    os.makedirs(os.environ["OUT"], exist_ok=True)
    with open(os.path.join(os.environ["OUT"], "exp_group_index_%s.json" % wl_name), "w") as f:
        json.dump(out, f, indent=1)
