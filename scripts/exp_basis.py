"""Dev experiment: time of the projected screen's basis choice per row width (needs a GPU).

For each width, builds an f32 cos index of N rows (bench.py's structured generator, or DATA=gauss for isotropic Gaussian rows)
and prints the automatic choice (k, or none = int8 screen) and the host time it took (Index.screen_basis), which covers the
moment matrix, the top eigenvectors, the residual energies and the records; and the same for load_buffer of the saved index.
usage: python scripts/exp_basis.py [widths, default 768,1024,1536,2048] ; env N (default 20000), DATA, OUT (directory for the JSON)"""
import json, os, sys
sys.path.insert(0, '.')
import numpy as np, torch
import bench
from lantern_b200 import api

widths = [int(w) for w in (sys.argv[1] if len(sys.argv) > 1 else "768,1024,1536,2048").split(",")]
n, data = int(os.environ.get("N", "20000")), os.environ.get("DATA", "structured")
dev = torch.device("cuda", 0)
res = {"gpu": torch.cuda.get_device_name(0), "rows": n, "data": data, "widths": {}}
for d in widths:
    if data == "gauss":
        X = torch.randn((n, d), generator=torch.Generator(device=dev).manual_seed(bench.SEED_CORPUS), device=dev)
    else:
        X = bench.structured_torch(n, d, bench.SEED_CORPUS, dev)
    idx = api.Index(d, "cos", "f32", M=16, efc=64, ef=64)
    idx.add_batch_device(np.arange(1, n + 1, dtype=np.uint64), X.data_ptr(), n, d * 4, "f32")
    idx.build()
    P, sec = idx.screen_basis()
    h = api.Index(d, "cos", "f32", M=16, efc=64, ef=64)
    h.load_buffer(idx.save_buffer())
    P2, sec2 = h.screen_basis()
    same = (P is None and P2 is None) or (P is not None and P2 is not None and np.array_equal(P.view(np.uint32), P2.view(np.uint32)))
    res["widths"][d] = {"k": None if P is None else len(P), "build_choice_s": sec, "load_choice_s": sec2, "same_bits_after_load": same}
    print(d, res["widths"][d], flush=True)
print(json.dumps(res))
if os.environ.get("OUT"):
    os.makedirs(os.environ["OUT"], exist_ok=True)
    with open(os.path.join(os.environ["OUT"], "exp_basis_%s.json" % data), "w") as f:
        json.dump(res, f, indent=1)
