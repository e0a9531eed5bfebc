"""Smoke-size walk through the search, build, PQ and exact kernels for compute-sanitizer (memcheck / racecheck / synccheck):
    compute-sanitizer --tool memcheck python scripts/sanitize_small.py
Sizes are tiny on purpose: the sanitizer slows kernels down by one to two orders of magnitude."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lantern_b200 import api  # noqa: E402

rng = np.random.default_rng(0)
n, d, nq, k = 600, 48, 24, 5
X = rng.standard_normal((n, d)).astype(np.float32)
Q = rng.standard_normal((nq, d)).astype(np.float32)
for metric, quant in (("l2sq", "f32"), ("cos", "f16"), ("l2sq", "i8")):
    g = api.Index(d, metric, quant, M=8, efc=32, ef=24)
    g.reserve(n)
    g.add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
    g.build()
    keys, dists, counts = g.search_batch(Q, k)
    assert (counts == k).all()
    g.close()
B = rng.integers(0, 256, (n, 32), dtype=np.uint8)
g = api.Index(256, "hamming", "b1", M=8, efc=32, ef=24)
g.reserve(n)
g.add_batch(np.arange(1, n + 1, dtype=np.uint64), B)
g.build()
g.search_batch(B[:nq], k)
g.close()
cb, rounds = api.train_pq(X, 12, 16, "l2sq", 5, 3)
g = api.Index(d, "l2sq", "f32", M=8, efc=32, ef=24, pq=True, num_centroids=16, num_subvectors=12, codebook=cb)
g.reserve(n)
g.add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
g.build()
g.search_batch(Q, k)
g.close()
api.exact_search(X, Q, k, "l2sq")
api.exact_search(X, Q, k, "cos")
# tensor-core exhaustive search (wgmma filter + re-rank), forced on this small problem
os.environ["LB200_EXACT"] = "tc"
kt, dt = api.exact_search(X, Q, k, "l2sq")
os.environ["LB200_EXACT"] = "simt"
ks, ds = api.exact_search(X, Q, k, "l2sq")
os.environ.pop("LB200_EXACT")
assert np.array_equal(kt, ks) and np.array_equal(dt.view(np.uint32), ds.view(np.uint32))
# the same through the filter's test hook, which copies its intermediate buffers out
pr = api.exact_tc_probe(X, Q, k, "cos")
assert not pr["unsafe"].any()
# the warp-per-query kernel alone and as a two-rank group on one device (owner + helper pool, mailboxes, fused all-gather)
g = api.Index(d, "cos", "f32", M=8, efc=32, ef=24)
g.reserve(n)
g.add_batch(np.arange(1, n + 1, dtype=np.uint64), X)
g.build()
k1, d1, _ = g.search_batch(Q, k)
g.set_option("search_kernel", 2)
k2, d2, _ = g.search_batch(Q, k)
assert np.array_equal(k1, k2) and np.array_equal(d1.view(np.uint32), d2.view(np.uint32))
grp = api.Group.local([0, 0])
grp.distribute(g, root=0, max_batch=64)
k3, d3, _ = grp.search_batch(Q, k)
assert np.array_equal(k1, k3) and np.array_equal(d1.view(np.uint32), d3.view(np.uint32))
grp.close()
g.close()
# the warp-per-query kernel with the projected screen (records, the per-batch pre-pass, q~ in the warp's shared memory)
Xw = (rng.standard_normal((n, 16)) @ rng.standard_normal((16, 320)) + 0.05 * rng.standard_normal((n, 320))).astype(np.float32)
os.environ["LB200_SEARCH_SCREEN"] = "2"
g = api.Index(320, "cos", "f32", M=8, efc=32, ef=24)
g.reserve(n)
g.add_batch(np.arange(1, n + 1, dtype=np.uint64), Xw)
g.build()
g.set_option("search_kernel", 1)
k1, d1, _ = g.search_batch(Xw[:nq], k)
g.set_option("search_kernel", 2)
k2, d2, _ = g.search_batch(Xw[:nq], k)
assert g.last_stats()["screen_kind"] == 2
assert np.array_equal(k1, k2) and np.array_equal(d1.view(np.uint32), d2.view(np.uint32))
os.environ.pop("LB200_SEARCH_SCREEN")
g.close()
print("sanitize_small: done, %d kernel launches" % api.kernel_launches())
