"""Dev experiment: the search screens (LB200_SEARCH_SCREEN 0 = off, 1 = int8, 2 = projected) and search kernels on ONE built
graph (needs a GPU).

Builds a workload's graph once with bench.py's generator and seeds (DATA=gauss: isotropic Gaussian rows and queries instead),
then alternates every (kernel, knob) setting for ROUNDS rounds of STEPS timed search steps each.  Prints, per setting,
queries/s (median and spread over the rounds), kernel time, the share of candidates read in full (full_rows_read /
computed_distances), the screen kind and codes per candidate, the kernel that ran and its cycle split by phase (one warp per
query), that every setting returns identical keys, distances and counters, and the device memory in use after the build (with
the automatically chosen companion) and after each setting's first search (a forced kind encodes its companion then).
usage: python scripts/exp_screen.py [workload] ; env ROUNDS (default 3), STEPS (default 20), KNOBS (default 0,1,2; "auto" =
unset), KERNELS (default "0": the "search_kernel" option, 0 = automatic, 1 = one CTA per query, 2 = one warp per query;
"1w2" = one CTA of 2 warps per query with 12 KB rings, LB200_SEARCH_WARPS=2 LB200_RING_BYTES=12288), DATA (structured |
gauss), OUT (directory for the JSON), INDEX (an index file: loaded instead of building the graph when it exists, else written
after the build, so that two builds of the engine can be timed on one graph in alternating processes).
Per setting it also prints upper_hops_per_query and screened_per_query.  Every candidate of a greedy pass goes through the
screen (unless the walk's distance is NaN), so on one graph screened_per_query minus that of a build whose descent is not
screened is the descent's candidates per query, and that over upper_hops_per_query the mean fill of the lists it visits."""
import hashlib, json, os, sys, time
sys.path.insert(0, '.')
import numpy as np, torch
import bench
from lantern_b200 import api

wl_name = sys.argv[1] if len(sys.argv) > 1 else "cfg3"
wl = bench.WORKLOADS[wl_name]
rounds, steps = int(os.environ.get("ROUNDS", "3")), int(os.environ.get("STEPS", "20"))
knobs = os.environ.get("KNOBS", "0,1,2").split(",")
kernels = os.environ.get("KERNELS", "0").split(",")
settings = [(kn, kb) for kn in kernels for kb in knobs]
data = os.environ.get("DATA", "structured")
n, dim, B, k, ef = wl["n"], wl["dim"], wl["batch"], wl["k"], wl["ef"]
dev = torch.device("cuda", 0)
free0, total = torch.cuda.mem_get_info()
pool = 4
index_file = os.environ.get("INDEX")
load = bool(index_file) and os.path.exists(index_file)
if data == "gauss":
    if not load:
        X = torch.randn((n, dim), generator=torch.Generator(device=dev).manual_seed(bench.SEED_CORPUS), device=dev)
    Q = torch.randn((pool * B, dim), generator=torch.Generator(device=dev).manual_seed(bench.SEED_QUERY), device=dev)
else:
    if not load:
        X = bench.structured_torch(n, dim, bench.SEED_CORPUS, dev)
    Q = bench.structured_torch(pool * B, dim, bench.SEED_QUERY, dev)
idx = api.Index(dim, wl["metric"], "f32", M=wl["M"], efc=wl["efc"], ef=ef)
t = time.time()
if load:
    idx.load(index_file)  # load_buffer chooses the same basis bits from the same rows
else:
    idx.reserve(n)
    idx.add_batch_device(np.arange(1, n + 1, dtype=np.uint64), X.data_ptr(), n, dim * 4, "f32")
    idx.build()
    if index_file:
        idx.save(index_file)
torch.cuda.synchronize()
mem = {"total_gb": total / 1e9, "used_before_gb": (total - free0) / 1e9}
mem["used_after_build_gb"] = (total - torch.cuda.mem_get_info()[0]) / 1e9
basis, basis_s = idx.screen_basis()
mem["basis_seconds"] = basis_s
print("%s (%s): build %.1f s, basis k=%s (%.2f s)" % (wl_name, data, time.time() - t, None if basis is None else len(basis), basis_s),
      flush=True)
ok = torch.empty((B, k), dtype=torch.int64, device=dev)
od = torch.empty((B, k), dtype=torch.float32, device=dev)
oc = torch.empty((B,), dtype=torch.int32, device=dev)
stream = torch.cuda.current_stream()


def step(s):
    idx.search_batch_device(Q[(s % pool) * B].data_ptr(), B, dim * 4, "f32", k, ef, ok.data_ptr(), od.data_ptr(), oc.data_ptr(),
                            stream.cuda_stream)


def apply(kern, knob):
    for var in ("LB200_SEARCH_SCREEN", "LB200_SEARCH_WARPS", "LB200_RING_BYTES"):
        os.environ.pop(var, None)
    if knob != "auto":
        os.environ["LB200_SEARCH_SCREEN"] = knob
    if kern == "1w2":
        os.environ["LB200_SEARCH_WARPS"], os.environ["LB200_RING_BYTES"] = "2", "12288"
    idx.set_option("search_kernel", 1 if kern == "1w2" else int(kern))


def name(kern, knob):
    return "screen=%s" % knob if kernels == ["0"] else "kernel=%s,screen=%s" % (kern, knob)


CYCLES = ("owner_cycles_produce", "owner_cycles_screen", "owner_cycles_evaluate", "owner_cycles_consume")
ref, cyc = {}, {}
for kern, knob in [("0", "auto")] + settings:  # outputs and counters of every pool batch, every way
    apply(kern, knob)
    outs, cy = [], np.zeros(len(CYCLES))
    t = time.time()
    for s in range(pool):
        step(s)
        torch.cuda.synchronize()
        st = idx.last_stats()
        outs.append((ok.cpu().numpy().copy(), od.cpu().numpy().view(np.uint32).copy(), oc.cpu().numpy().copy(),
                     st["computed_distances"], st["base_pops"], st["upper_hops"], st["full_rows_read"], st["screen_kind"],
                     st["screen_dims"], st["search_kernel"], st["algorithmic_bytes"]))
        cy += [st[c] for c in CYCLES]
    ref[name(kern, knob)], cyc[name(kern, knob)] = outs, cy
    print("%s: %d checked batches in %.2f s, kind %d, %d codes per candidate, kernel %d" % (
        name(kern, knob), pool, time.time() - t, outs[0][7], outs[0][8], outs[0][9]), flush=True)
    mem["used_after_search_%s_gb" % name(kern, knob)] = (total - torch.cuda.mem_get_info()[0]) / 1e9
names = [name(kn, kb) for kn, kb in settings]
same = all(all(np.array_equal(a, b) for a, b in zip(o0[:3], o1[:3])) and o0[3:6] == o1[3:6]
           for kb in ref for o0, o1 in zip(ref[names[0]], ref[kb]))
res = {nm: [] for nm in names}
kern_ms = {nm: [] for nm in names}
for r in range(rounds):
    for (kn, knob), nm in zip(settings, names):
        apply(kn, knob)
        for s in range(3):
            step(s)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for s in range(steps):
            step(s)
        torch.cuda.synchronize()
        res[nm].append(steps * B / (time.perf_counter() - t0))
        km = 0.0
        for s in range(4):
            step(s)
            km += idx.last_stats()["kernel_ms"]
        kern_ms[nm].append(km / 4)
        print("round %d %s  %.0f queries/s  kernel %.2f ms/step" % (r, nm, res[nm][-1], kern_ms[nm][-1]), flush=True)
auto = name("0", "auto")
out = {"workload": wl_name, "data": data, "identical_outputs_and_counters": bool(same), "memory": mem,
       "gpu": torch.cuda.get_device_name(0), "auto_screen_kind": ref[auto][0][7], "auto_screen_dims": ref[auto][0][8],
       "auto_search_kernel": ref[auto][0][9],
       # keys, distance bits and counts of the checked batches: equal across processes = the same outputs
       "outputs_sha256": hashlib.sha256(b"".join(a.tobytes() for o in ref[names[0]] for a in o[:3])).hexdigest()}
for nm in names:
    v = np.array(res[nm])
    cd = sum(o[3] for o in ref[nm])
    fr = sum(o[6] for o in ref[nm])
    cy = cyc[nm]
    # candidates that went through the screen, from the byte count: the inverse of Index::last_stats()'s algorithmic_bytes
    # (engine.cu, DESIGN.md 4.1), which assumes f32 rows of 4 * dim bytes, M0 = 2M, one query row per query and a record of
    # 64 bytes for k <= 48, else 128 (projected) or a code row + 16 bytes of metadata (int8): change it with that formula
    kind, sd = ref[nm][0][7], ref[nm][0][8]
    rest = sum(o[10] - o[6] * dim * 4 - o[4] * (4 + 8 * wl["M"]) - o[5] * (4 + 4 * wl["M"]) - B * dim * 4 for o in ref[nm])
    screened = rest / ({1: dim + 16, 2: 64 if sd <= 48 else 128}[kind]) if kind else 0
    out[nm] = {"qps_median": float(np.median(v)), "qps_min": float(v.min()), "qps_max": float(v.max()),
               "kernel_ms_median": float(np.median(kern_ms[nm])), "dist_evals_per_query": cd / (pool * B),
               "full_rows_read_per_query": fr / (pool * B), "full_rows_frac": fr / cd,
               "upper_hops_per_query": sum(o[5] for o in ref[nm]) / (pool * B), "screened_per_query": screened / (pool * B),
               "screen_kind": ref[nm][0][7], "codes_per_candidate": ref[nm][0][8], "search_kernel": ref[nm][0][9],
               "cycle_split": {c[len("owner_cycles_"):]: (float(x / cy.sum()) if cy.sum() else 0.0) for c, x in zip(CYCLES, cy)}}
for nm in names[1:]:
    out["speedup_median_%s_vs_%s" % (nm, names[0])] = out[nm]["qps_median"] / out[names[0]]["qps_median"]
print(json.dumps(out))
if os.environ.get("OUT"):  # directory for the JSON result
    os.makedirs(os.environ["OUT"], exist_ok=True)
    with open(os.path.join(os.environ["OUT"], "exp_screen_%s_%s.json" % (wl_name, data)), "w") as f:
        json.dump(out, f, indent=1)
