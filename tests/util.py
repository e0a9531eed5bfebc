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


def make_rows(port, quant, metric, dims, rows, n, seed):
    """(input rows as passed to both builds, the same rows in the storage domain) for exact-distance builds.
    rows: ("int", r) integers in [-r, r]; ("int0", r) the same plus all-zero and duplicate rows; ("i8", s) uniform in
    [-s, s] cast to int8 (plus rows that cast to all zeros); ("bits",) clustered packed bits.  Asserts that every distance between two
    of them is exact in fp32 (see tests/test_gpu_build_model.py)."""
    rng = np.random.default_rng(seed)
    kind = rows[0]
    if kind == "bits":
        assert dims < EXACT_FP32
        X = hamming_rows(n, dims, seed)
        return X, X
    if kind == "i8":
        s = rows[1]
        X = rng.uniform(-s, s, (n, dims)).astype(np.float32)
        zero = rng.choice(n, n // 50, replace=False)  # |x| < 0.01: casts to an all-zero row (cos zero-norm rule)
        X[zero] = rng.uniform(-0.0099, 0.0099, (len(zero), dims)).astype(np.float32)
        r = min(100, int(np.floor(100 * s)))  # int8 cast: trunc(clamp(100 x, -100, 100))
        assert (dims * (2 * r) ** 2 if metric == "l2sq" else dims * r * r) < EXACT_FP32
        S = port.cast_f32(X, "i8")
        assert np.abs(S.astype(np.int32)).max() <= r and (np.abs(S).sum(1) == 0).any()
        return X, S
    X = exact_int_rows(rng, n, dims, rows[1], metric)
    if quant == "f16":
        assert rows[1] <= 2048  # integers up to 2048 are f16 values: the cast is exact on both sides
    if kind == "int0":  # zero-norm rows (both cos zero-norm cases) and exact duplicates (distance-0 ties)
        X[rng.choice(n, n // 100, replace=False)] = 0
        src, dst = rng.choice(n, (2, n // 50), replace=False)
        X[dst] = X[src]
    S = port.cast_f32(X, quant) if quant != "f32" else X
    if quant == "f16":
        assert np.array_equal(S.view(np.float16).astype(np.float32), X)
    return X, S


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


# ---- float64 reference with an a-priori bound on the fp32 kernels' rounding -------------------------------------------
U32 = 2.0 ** -24  # unit roundoff of fp32
ELEM_BITS = {"f32": 32, "f16": 16, "i8": 8, "b1": 1}


def gamma32(m):
    """gamma(m) = m u / (1 - m u): the relative error bound of m successive fp32 roundings (Higham, Accuracy and Stability of
    Numerical Algorithms, 3.1)."""
    return m * U32 / (1 - m * U32)


def row_bytes(quant, dims):
    """Bytes of one stored row, zero-padded to whole 16-byte chunks (common.cuh scalar_row_bytes, rounded up to 16)."""
    raw = (dims * ELEM_BITS[quant] + 7) // 8
    return (raw + 15) // 16 * 16


def chunk_passes(rb):
    """Chunks each lane of a warp folds in sequence: lane l owns chunks l, l + 32, ... of a row of `rb` bytes."""
    return (rb // 16 + 31) // 32


def sum_depths(quant, metric, P):
    """Longest chain of fp32 roundings in the kernels' distance sums (distance.cuh), P chunk passes per lane:
    (row sums ab / b2 / (a-b)^2, the query's a2).  l2sq: the rounded a - b counts twice (it is squared), then P (f32) or 2P
    (f16) fmas per accumulator, 2 adds across accumulators and 5 shuffle levels.  cos: 2P (f32) or 4P (f16) fmas per
    accumulator, 1 add and 5 shuffles; a2 takes 4 (f32) or 8 (f16) roundings per chunk, P chunk adds and 5 shuffles."""
    per = 1 if quant == "f32" else 2
    if metric == "l2sq":
        return per * P + 9, 0
    return 2 * per * P + 6, 4 * per + P + 5


def decode64(S, quant):
    """Storage-domain rows (f32, f16 as uint16 bits, i8) as float64 values; f16 decodes exactly."""
    S = np.asarray(S)
    return (S.view(np.float16) if quant == "f16" else S).astype(np.float64)


def reference64(A, B, metric, quant):
    """Distances [len(A)][len(B)] between storage-domain rows in float64, and a bound on the error of the fp32 kernels.

    b1: popcounts, exact.  i8: integer sums, exact while below 2^24 (beyond that one rounding of the exact int32 sum).
    f32 / f16: gamma(depth) times the sum of the absolute terms (sum_depths); for cos the ab, a2 and b2 bounds are carried
    through 1 - ab / (sqrt(a2) sqrt(b2)) -- two square roots, a product, a quotient and a difference, each one rounding --
    plus 2 ulp.  l2sq sums (a - b)^2 directly in float64, whose own rounding adds (d + 2) 2^-52 D to the bound."""
    if quant == "b1":
        A, B = np.asarray(A, np.uint8), np.asarray(B, np.uint8)
        D = np.stack([np.bitwise_count(np.bitwise_xor(a[None, :], B)).sum(1) for a in A]).astype(np.float64)
        return D, np.zeros_like(D)
    a, b = decode64(A, quant), decode64(B, quant)
    P = chunk_passes(row_bytes(quant, a.shape[1]))
    m_row, m_a2 = sum_depths(quant, metric, P)
    a2, b2 = (a * a).sum(1), (b * b).sum(1)
    if metric == "l2sq":
        D = np.empty((len(a), len(b)))
        step = max(1, (1 << 24) // max(1, b.size))
        for s in range(0, len(a), step):
            diff = a[s:s + step, None, :] - b[None, :, :]
            D[s:s + step] = np.einsum("qnd,qnd->qn", diff, diff)
        if quant == "i8":  # exact in float64 (integers far below 2^53); so is the kernel's integer sum, its cast rounds
            return D, np.where(D < 2 ** 24, 0.0, U32 * D)
        return D, gamma32(m_row) * D + (a.shape[1] + 2) * 2.0 ** -52 * D + m_row * 2.0 ** -149
    ab = a @ b.T
    S = np.abs(a) @ np.abs(b).T
    if quant == "i8":  # int32 sums, exact; each becomes a float once (fadd chain for a2: exact below 2^24)
        g_ab = np.where(S < 2 ** 24, 0.0, U32)
        g_a = np.where(a2 < 2 ** 24, 0.0, gamma32(P + 6))[:, None]
        g_b = np.where(b2 < 2 ** 24, 0.0, U32)[None, :]
    else:
        g_ab, g_a, g_b = gamma32(m_row), gamma32(m_a2), gamma32(m_row)
    na, nb = np.sqrt(a2)[:, None], np.sqrt(b2)[None, :]
    den = np.where((na > 0) & (nb > 0), na * nb, 1.0)
    x = ab / den
    eta = (g_a + g_b) / 2 + 3 * U32  # relative error of the computed sqrt(a2) * sqrt(b2)
    ex = (g_ab * S / den + np.abs(x) * eta) / (1 - eta)
    ex = ex + U32 * (np.abs(x) + ex)  # the quotient
    D = 1.0 - x
    bound = ex + U32 * (np.abs(D) + ex) + 2 * 2 * U32 * np.maximum(np.abs(D), 2.0 ** -24)
    zero_a, zero_b = (a2 == 0)[:, None], (b2 == 0)[None, :]
    D = np.where(zero_a & zero_b, 0.0, np.where(zero_a | zero_b, 1.0, D))
    bound = np.where(zero_a | zero_b, 0.0, bound * (1 + 1e-6))
    return D, bound


def check_distances(got, D, bound, what=""):
    """Every returned fp32 distance lies within its bound of the float64 one."""
    err = np.abs(got.astype(np.float64) - D)
    bad = np.argwhere(~(err <= bound))
    assert len(bad) == 0, "%s: %d distances outside the bound, first at %s: got %r, float64 %r, bound %r" % (
        what, len(bad), tuple(bad[0]), float(got[tuple(bad[0])]), float(D[tuple(bad[0])]), float(bound[tuple(bad[0])]))


def check_topk(keys, dists, D, bound, k, what=""):
    """Tie-aware check of an exhaustive top-k (ids = row offsets) against float64 distances D [nq][n] with bounds: the
    distances are within their bounds and ascending, the ids distinct, and an id differs from the float64 top-k only where
    its float64 distance lies within twice the bound of the k-th one."""
    n = D.shape[1]
    kk = min(k, n)
    for q in range(len(D)):
        ids = keys[q, :kk].astype(np.int64)
        assert (ids >= 0).all() and (ids < n).all() and len(set(ids.tolist())) == kk, (what, q, ids[:8])
        check_distances(dists[q, :kk], D[q, ids], bound[q, ids], "%s q%d" % (what, q))
        assert (np.diff(dists[q, :kk]) >= 0).all(), (what, q)
        order = np.lexsort((np.arange(n), D[q]))
        kth = D[q, order[kk - 1]]
        tol = 2 * bound[q, order[:kk]].max()  # twice the bound at the k-th distance (or any float64 top-k one)
        assert (D[q, ids] <= kth + tol).all(), (what, q, "an id outside the float64 top-k and its ties")
        must = np.nonzero(D[q] < kth - tol)[0]
        assert np.isin(must, ids).all(), (what, q, "a float64 top-k id clear of the k-th distance is missing")
        if k > n:
            assert (keys[q, n:] == np.iinfo(np.uint64).max).all() and np.isinf(dists[q, n:]).all(), (what, q)
