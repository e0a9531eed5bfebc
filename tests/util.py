"""Shared helpers for the parity tests."""
import numpy as np


def structured(n, d, seed, latent=32, noise=0.05):
    """Low-intrinsic-dimension synthetic vectors (SURVEY.md 8d): x = z P + noise * eps."""
    rng = np.random.default_rng(seed)
    P = (np.random.default_rng(1234).standard_normal((latent, d)) / np.sqrt(latent)).astype(np.float32)
    z = rng.standard_normal((n, latent)).astype(np.float32)
    return (z @ P + noise * rng.standard_normal((n, d)).astype(np.float32)).astype(np.float32)


EXACT_FP32 = 1 << 24  # every integer of magnitude <= 2^24 is an fp32 value: sums of such integers are exact in any order


def exact_int_rows(rng, n, d, r, metric):
    """Integer coordinates in [-r, r] whose distances are exact in fp32 whatever the summation order: every product and
    every partial sum is an integer below 2^24 (l2sq: d (2r)^2; cos: d r^2 for a.b, |a|^2 and |b|^2)."""
    bound = d * (2 * r) ** 2 if metric == "l2sq" else d * r * r
    assert bound < EXACT_FP32, (metric, d, r, bound)
    return rng.integers(-r, r + 1, (n, d)).astype(np.float32)


def hamming_rows(n, bits, seed, protos_seed=5, flip=0.1):
    """Clustered packed bits (16 random prototypes, each bit flipped with probability `flip`): exact ties everywhere.
    Bits past `bits` in the last byte are zero."""
    protos = np.random.default_rng(protos_seed).random((16, bits)) < 0.5
    r = np.random.default_rng(seed)
    rows = protos[r.integers(0, 16, n)] ^ (r.random((n, bits)) < flip)
    return np.packbits(rows, axis=1)


def build_port_index(portlib, X, metric="l2sq", quant="f32", M=16, efc=128, ef=64, keys=None, **kw):
    n = len(X)
    dim = X.shape[1] * 8 if X.dtype == np.uint8 else X.shape[1]
    idx = portlib.PortIndex(dim, metric, quant, M=M, efc=efc, ef=ef, **kw)
    idx.reserve(n)
    keys = np.arange(1, n + 1, dtype=np.uint64) if keys is None else keys
    for i in range(n):
        idx.add(keys[i], X[i])
    return idx


def compare_results(keys_a, dists_a, keys_b, dists_b, rtol=1e-5, atol=1e-6):
    """Position-wise id equality, tolerating permutations inside groups of (near-)equal distances.
    Returns (n_exact_rows, n_rows_ok)."""
    nq = len(keys_a)
    exact = ok = 0
    for q in range(nq):
        ka, kb, da, db = keys_a[q], keys_b[q], dists_a[q], dists_b[q]
        if np.array_equal(ka, kb):
            exact += 1
            ok += 1
            continue
        # distances must agree position-wise within tolerance and differing ids must sit in near-tie groups
        if not np.allclose(da, db, rtol=rtol * 10, atol=atol * 10):
            continue
        good = True
        for i in np.nonzero(ka != kb)[0]:
            # id kb[i] must appear in ka at a position whose distance is within tolerance of da[i]
            pos = np.nonzero(ka == kb[i])[0]
            if len(pos) == 0:
                # allowed only at the tail boundary: distance equal to the last one
                if not np.isclose(db[i], da[-1], rtol=rtol * 10, atol=atol * 10):
                    good = False
            elif not np.isclose(da[pos[0]], db[i], rtol=rtol * 10, atol=atol * 10):
                good = False
        ok += good
    return exact, ok


def recall(found, truth):
    hits = 0
    for f, t in zip(found, truth):
        hits += len(set(f.tolist()) & set(t.tolist()))
    return hits / truth.size


def adjacency_lists(buf, M, stored_bytes):
    """Parse a usearch/lantern index file (SURVEY App. B) into {(node, level): tuple(neighbour ids)} plus the level array.
    Vectors and keys are skipped: comparisons through this helper look at the graph only."""
    b = np.asarray(buf, dtype=np.uint8).tobytes()
    n = int(np.frombuffer(b, np.uint64, 1, 80)[0])
    M0 = 2 * M
    lists, levels = {}, np.zeros(n, np.int16)
    p = 136
    for i in range(n):
        lvl = int(np.frombuffer(b, np.int16, 1, p + 8)[0])
        levels[i] = lvl
        p += 10
        for l in range(lvl + 1):
            width = M0 if l == 0 else M
            cnt = int(np.frombuffer(b, np.uint32, 1, p)[0])
            raw = np.frombuffer(b, np.uint8, 6 * width, p + 4).reshape(width, 6)[:cnt]
            ids = raw[:, :4].copy().view(np.uint32)[:, 0]
            lists[(i, l)] = tuple(int(x) for x in ids)
            p += 4 + 6 * width
        p += stored_bytes
    assert p == len(b), (p, len(b))
    return lists, levels


def distance64(a, b, metric, quant):
    """Distance of two storage-domain rows (f32, f16 as uint16 bits, i8, b1 packed bytes) in float64."""
    if quant == "b1":
        return float(np.unpackbits(np.bitwise_xor(a, b)).sum())
    a = (a.view(np.float16) if quant == "f16" else a).astype(np.float64)
    b = (b.view(np.float16) if quant == "f16" else b).astype(np.float64)
    if metric == "l2sq":
        return float(((a - b) ** 2).sum())
    a2, b2 = float(a @ a), float(b @ b)
    if a2 == 0 and b2 == 0:
        return 0.0
    if a2 == 0 or b2 == 0:
        return 1.0
    return 1.0 - float(a @ b) / (np.sqrt(a2) * np.sqrt(b2))


def describe_file_difference(buf_a, buf_b, M, stored_bytes, rows, metric, quant, dims, port, names=("gpu", "model")):
    """Where two index files of the same rows differ, in terms a person can debug from: the first differing (node, level)
    adjacency list of each file, and for every id in either list its distance to the node in float64 and by the oracle's
    fp32 metric.  Equal distances in a different order point at tie order; different distances at the kernel."""
    a, b = np.asarray(buf_a, np.uint8), np.asarray(buf_b, np.uint8)
    if len(a) != len(b):
        return "file lengths differ: %s %d bytes, %s %d bytes" % (names[0], len(a), names[1], len(b))
    la, lva = adjacency_lists(a, M, stored_bytes)
    lb, lvb = adjacency_lists(b, M, stored_bytes)
    if not np.array_equal(lva, lvb):
        return "level draws differ, first at node %d" % int(np.nonzero(lva != lvb)[0][0])
    differ = [k for k in sorted(la) if la[k] != lb[k]]
    if not differ:
        return "adjacency lists identical; first differing byte at offset %d" % int(np.nonzero(a != b)[0][0])
    node, level = differ[0]
    out = ["%d of %d adjacency lists differ; first at node %d, level %d" % (len(differ), len(la), node, level),
           "  %-5s %s" % (names[0], list(la[(node, level)])), "  %-5s %s" % (names[1], list(lb[(node, level)]))]
    ids = sorted(set(la[(node, level)]) | set(lb[(node, level)]), key=lambda i: (distance64(rows[node], rows[i], metric, quant), i))
    for i in ids:
        out.append("  id %6d  float64 %-22.17g oracle fp32 %-14.9g in %s" % (
            i, distance64(rows[node], rows[i], metric, quant), port.distance(rows[node], rows[i], metric, quant, dims),
            "+".join(n for n, l in zip(names, (la, lb)) if i in l[(node, level)]) or "-"))
    return "\n".join(out)
