"""Numerics of the PQ asymmetric-distance path against float64 over decoded rows.

The distance from a value v to a stored PQ row j is a sum of look-up table entries, lut[s][code_js], where the table is built
from v: |v_s - c_s|^2 (l2sq) or v_s . c_s (cos, which then combines the dot product with |v|^2 and the summed centroid norms).
api.pq_probe runs the evaluator of the search and build kernels (PqEval) on a built index for every (value, stored row)
pair, with each of the three ways a table is made: precomputed for a search batch, built inside the kernel (batches whose
tables pass 1 GB, and the build), or copied from the centroid-pair table when the value is a stored node (refine, reverse
links).  The reference is numpy float64 over the decoded rows (codebook slices gathered by code).  The oracle is used only
where a whole search or k-means run is compared."""
import math
import re

import numpy as np
import pytest

from util import structured

pytestmark = pytest.mark.gpu

U = 2.0 ** -24  # unit roundoff of fp32
M = 8  # connectivity of the test indexes (level-0 lists of 16)


# ---- index files with chosen codes ------------------------------------------------------------------------------------

def _code_offsets(buf, M, nsub):
    """Byte offset of every node's code row in an index file (the node tapes util.adjacency_lists walks)."""
    b = np.asarray(buf, dtype=np.uint8)
    n = int(b[80:88].view(np.uint64)[0])
    p, out = 136, []
    for _ in range(n):
        lvl = int(b[p + 8:p + 10].view(np.int16)[0])
        p += 10 + (4 + 12 * M) + lvl * (4 + 6 * M)
        out.append(p)
        p += nsub
    assert p == len(b)
    return out


def get_codes(buf, M, nsub):
    b = np.asarray(buf, dtype=np.uint8)
    return np.stack([b[o:o + nsub] for o in _code_offsets(b, M, nsub)])


def set_codes(buf, codes, M):
    b = np.array(buf, dtype=np.uint8)
    for i, o in enumerate(_code_offsets(b, M, codes.shape[1])):
        b[o:o + codes.shape[1]] = codes[i]
    return b


def decode64(cb, codes, nsub):
    """[n][nsub][subdim] float64: the codebook slices the codes select."""
    ncent, d = cb.shape
    return cb.astype(np.float64).reshape(ncent, nsub, d // nsub)[codes, np.arange(nsub)]


def new_index(eng, metric, cb, nsub, **kw):
    return eng.Index(cb.shape[1], metric, "f32", M=M, efc=32, ef=32, pq=True, num_centroids=len(cb), num_subvectors=nsub,
                     codebook=cb, **kw)


def pq_index(eng, metric, cb, nsub, codes):
    """A built index whose stored rows hold exactly `codes`: the engine builds a graph over the decoded rows, and the saved
    file's code bytes are replaced before it is loaded into a fresh index (codes >= 128 widen the look-up tables)."""
    n, d = len(codes), cb.shape[1]
    g = new_index(eng, metric, cb, nsub)
    g.reserve(n)
    g.add_batch(np.arange(1, n + 1, dtype=np.uint64), decode64(cb, codes, nsub).reshape(n, d).astype(np.float32))
    g.build()
    h = new_index(eng, metric, cb, nsub)
    h.load_buffer(set_codes(g.save_buffer(), codes, M))
    return h


# ---- float64 reference and the error bound of the kernel's fp32 arithmetic ------------------------------------------

def tables64(v, cb, nsub, W, metric):
    """(T, A) [nsub][W]: the exact table of value v (float64) and the sum of |terms| of every entry."""
    sd = cb.shape[1] // nsub
    t = v.astype(np.float64).reshape(nsub, 1, sd)
    c = cb[:W].astype(np.float64).reshape(W, nsub, sd).transpose(1, 0, 2)
    terms = (t - c) ** 2 if metric == "l2sq" else t * c
    return terms.sum(-1), np.abs(terms).sum(-1)


def chunk_depth(nsub):
    """Roundings of the sum over a code row's 16-byte chunks: sequential over cpr chunks, or (more than kPqPartPerWarp = 64
    chunks) ceil(cpr / 32) per lane and 5 butterfly levels."""
    cpr = (nsub + 15) // 16
    return cpr if cpr <= 64 else (cpr + 31) // 32 + 5


def distance_bound(metric, sd, nsub, d, Aj, a2, b2, ab, mode):
    """Per-pair bound on |d_kernel - d64| (first order in u, with 1 % for the higher-order terms).
    The dot product or squared distance: a table entry is subdim fmas after a subtraction (sd + 2), a chunk adds 16 entries,
    the chunk partials add up chunk_depth(nsub) more -- each rounding relative to the sum of |terms| Aj.
    cos also carries |v|^2 (load_value / pq_query_tables_kernel: ceil(d / 32) terms per lane and 5 butterfly levels; a node
    value: subdim fmas per centroid norm, ceil(nsub / 32) per lane and 5 levels), b2 (centroid norms summed like the entries)
    and the replay of cos_from_parts: two square roots, a product, a quotient and 1 - r."""
    depth = sd + 2 + 16 + chunk_depth(nsub)
    if metric == "l2sq":
        return 1.01 * depth * U * Aj
    ea = (sd + 1 + math.ceil(nsub / 32) + 6) * U if mode == "node" else (math.ceil(d / 32) + 6) * U
    eb = (sd + 1 + 16 + chunk_depth(nsub)) * U
    den = np.sqrt(a2 * b2)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(den > 0, ab / den, 0.0)
        e = depth * U * Aj / den + np.abs(r) * (ea / 2 + eb / 2 + 4 * U) + U * np.abs(1 - r) + U
    return 1.01 * e


def cos64(ab, a2, b2):
    """cos_from_parts (distance.cuh) in float64: both norms zero -> 0, one zero -> 1."""
    with np.errstate(divide="ignore", invalid="ignore"):
        d = 1.0 - ab / np.sqrt(a2 * b2)
    d = np.where((a2 == 0) | (b2 == 0), 1.0, d)
    return np.where((a2 == 0) & (b2 == 0), 0.0, d)


# ---- the geometry matrix ----------------------------------------------------------------------------------------------
# (dims, nsub, ncent, hi): stored codes in [0, hi).  The table is 128 wide when ncent > 128 and every code is below 128,
# else ncent wide.  subdim 1, 3, 4, 6, 16, 96; ncent 16, 128, 129, 256; code rows of 1, 6 and 96 chunks (the last takes the
# wide-row branch of PqEval::eval: more than 1024 subvectors); 3 x 129 is a table that is not a whole number of 16-byte chunks.
GEOMS = [
    (8, 8, 16, 16),
    (24, 8, 129, 128),
    (9, 3, 129, 129),
    (384, 96, 256, 128),
    (576, 96, 256, 256),
    (16, 1, 128, 128),
    (1536, 96, 256, 128),
    (96, 1, 256, 256),
    (768, 8, 256, 256),
    (1536, 1536, 16, 16),
]
GEOM_IDS = ["d%d-n%d-c%d-w%d" % (d, s, c, 128 if c > 128 and h <= 128 else c) for d, s, c, h in GEOMS]


def geometry(d, nsub, ncent, hi, seed):
    """Codebook (centroid 0 is zero: zero norms), codes (rows 0..hi-1 hold every code in every subvector, row hi decodes to
    the zero vector, the rest are random) and values (random, zero, a stored row exactly, a large one)."""
    rng = np.random.default_rng(seed)
    cb = rng.standard_normal((ncent, d)).astype(np.float32)
    cb[0] = 0.0
    n = hi + 200
    codes = rng.integers(0, hi, (n, nsub))
    codes[:hi] = (np.arange(hi)[:, None] + np.arange(nsub)[None, :]) % hi
    codes[hi] = 0
    codes = codes.astype(np.uint8)
    V = rng.standard_normal((6, d)).astype(np.float32)
    V[1] = 0.0
    V[2] = decode64(cb, codes[5:6], nsub).reshape(d).astype(np.float32)
    V[3] *= 1000.0
    return cb, codes, V


def check_probe(metric, cb, codes, nsub, W, values64, d, lut, v2, mode):
    """Every table entry and every distance of a probe against float64; returns the largest |d - d64| / eps."""
    sd = cb.shape[1] // nsub
    dec = decode64(cb, codes, nsub)
    b2 = (dec ** 2).sum((1, 2))
    cols = np.arange(nsub)
    worst = 0.0
    for i, v in enumerate(values64):
        T, A = tables64(v, cb, nsub, W, metric)
        # entries: (sd + 2) u sum|terms| (a pair-table entry is the same arithmetic with a centroid as the value)
        err = np.abs(lut[i].astype(np.float64) - T)
        assert (err <= 1.0001 * (sd + 2) * U * A).all(), (mode, i, np.unravel_index(np.argmax(err - (sd + 2) * U * A), err.shape))
        d64 = T[cols, codes].sum(1)
        Aj = A[cols, codes].sum(1)
        a2 = float((v.astype(np.float64) ** 2).sum())
        if metric == "cos" or mode == "batch":  # |v|^2 (a l2sq table built in the kernel does not carry it)
            if mode == "node":
                ea = (sd + 1 + math.ceil(nsub / 32) + 6) * U
            else:
                ea = (math.ceil(cb.shape[1] / 32) + 6) * U
            assert abs(float(v2[i]) - a2) <= 1.01 * ea * a2, (mode, i, float(v2[i]), a2)
        if metric == "cos":
            ab = d64
            d64 = cos64(ab, a2, b2)
            zero = (a2 == 0) | (b2 == 0)
            assert np.array_equal(d[i][zero], d64[zero].astype(np.float32)), (mode, i)  # the {0, 1} table of cos_from_parts
        else:
            ab, zero = None, np.zeros(len(codes), bool)
        eps = distance_bound(metric, sd, nsub, cb.shape[1], Aj, a2, b2, ab, mode)
        err = np.abs(d[i].astype(np.float64) - d64)
        ok = ~zero
        assert (err[ok] <= eps[ok] + 1e-30).all(), (mode, i, np.max(err[ok] / (eps[ok] + 1e-30)))
        if ok.any():
            worst = max(worst, float(np.max(err[ok] / (eps[ok] + 1e-30))))
    return worst


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("geom", GEOMS, ids=GEOM_IDS)
def test_probe_tables_and_distances_against_float64(eng, metric, geom):
    d, nsub, ncent, hi = geom
    cb, codes, V = geometry(d, nsub, ncent, hi, seed=d + nsub + ncent + hi)
    h = pq_index(eng, metric, cb, nsub, codes)
    # passes of 128 candidates (search_expand 8 x 16) or of 16: several eval() passes per value, the last one ragged
    expand = 8 if GEOMS.index(geom) % 2 == 0 else 1
    h.set_option("search_expand", expand)
    W = 128 if ncent > 128 and hi <= 128 else ncent
    out = {}
    for mode in ("batch", "kernel"):
        dist, lut, v2 = eng.pq_probe(h, mode, values=V)
        assert lut.shape == (len(V), nsub, W)
        out[mode] = (dist, lut, v2, check_probe(metric, cb, codes, nsub, W, V, dist, lut, v2, mode))
    # the two kinds of value tables are the same arithmetic: the same bits
    (db, lb, vb, rb), (dk, lk, vk, rk) = out["batch"], out["kernel"]
    assert np.array_equal(lb.view(np.uint32), lk.view(np.uint32))
    assert np.array_equal(db.view(np.uint32), dk.view(np.uint32))
    if metric == "cos":
        assert np.array_equal(vb.view(np.uint32), vk.view(np.uint32))
    # node values (rows 0..hi-1 select every centroid of every subvector, so every centroid-pair entry of pq_pair is read)
    nodes = np.arange(hi + 1, dtype=np.uint32)
    dist, lut, v2 = eng.pq_probe(h, "node", nodes=nodes)
    node_values = decode64(cb, codes[nodes], nsub).reshape(len(nodes), d)
    rn = check_probe(metric, cb, codes, nsub, W, node_values, dist, lut, v2, "node")
    print("PQ-NUMERICS %s d=%d nsub=%d ncent=%d W=%d max|d-d64|/eps batch=%.3g kernel=%.3g node=%.3g batch==kernel bits: yes"
          % (metric, d, nsub, ncent, W, rb, rk, rn))


@pytest.mark.parametrize("geom", [GEOMS[2], GEOMS[3], GEOMS[4], GEOMS[9]], ids=[GEOM_IDS[i] for i in (2, 3, 4, 9)])
@pytest.mark.parametrize("metric", ["l2sq", "cos"])
def test_search_same_with_either_table_kind(eng, metric, geom):
    """One batch with the batch's tables precomputed, and again with every CTA building its own table (option
    pq_query_tables = 0, the path of batches whose tables pass 1 GB): identical ids, distance bits, counts and counters."""
    d, nsub, ncent, hi = geom
    cb, codes, _ = geometry(d, nsub, ncent, hi, seed=7)
    h = pq_index(eng, metric, cb, nsub, codes)
    Q = (decode64(cb, codes[np.random.default_rng(8).integers(0, len(codes), 120)], nsub).reshape(120, d)
         + 0.3 * np.random.default_rng(9).standard_normal((120, d))).astype(np.float32)
    res = []
    for on in (1, 0):
        h.set_option("pq_query_tables", on)
        k, dd, c = h.search_batch(Q, 10, ef=48)
        res.append((k, dd.view(np.uint32), c, h.last_stats()))
    (k1, d1, c1, s1), (k0, d0, c0, s0) = res
    assert np.array_equal(k1, k0) and np.array_equal(d1, d0) and np.array_equal(c1, c0)
    for f in ("computed_distances", "base_pops", "upper_hops", "limbo_overflows"):
        assert s1[f] == s0[f], f
    assert (c1 == 10).all()


# ---- searches on the oracle's graph -----------------------------------------------------------------------------------

def port_pq(port, X, cb, nsub, metric, compat128, **kw):
    idx = port.PortIndex(X.shape[1], metric, "f32", pq=True, num_centroids=len(cb), num_subvectors=nsub, codebook=cb,
                         pq_compat128=compat128, **kw)
    idx.reserve(len(X))
    for i, v in enumerate(X):
        idx.add(i + 1, v)
    return idx


def assert_search_matches_float64(metric, cb, codes, nsub, Q, keys, dists, oracle_keys):
    """The engine's distances within the per-pair bound of float64 over the decoded corpus, and the engine's and the oracle's
    ids equal to the float64 brute force at every rank whose float64 gaps to the neighbouring ranks exceed both programs'
    rounding.  The oracle decodes the row and sums all dims in fp32 one after the other: distance_bound with subdim := dims
    and a node-style |v|^2 (dims + 1 roundings) bounds that arithmetic too, and it is never below the engine's bound."""
    dec = decode64(cb, codes, nsub)
    n, d = len(codes), cb.shape[1]
    sd = d // nsub
    k = keys.shape[1]
    cols = np.arange(nsub)
    b2 = (dec ** 2).sum((1, 2))
    for q, v in enumerate(Q):
        T, A = tables64(v, cb, nsub, cb.shape[0], metric)
        d64, Aj = T[cols, codes].sum(1), A[cols, codes].sum(1)
        a2 = float((v.astype(np.float64) ** 2).sum())
        ab = d64
        if metric == "cos":
            d64 = cos64(ab, a2, b2)
        eps = distance_bound(metric, sd, nsub, d, Aj, a2, b2, ab, "batch")
        rows = keys[q].astype(np.int64) - 1
        assert (np.abs(dists[q] - d64[rows]) <= eps[rows]).all(), q
        eps_both = np.maximum(eps, distance_bound(metric, d, nsub, d, Aj, a2, b2, ab, "node"))
        order = np.argsort(d64, kind="stable")
        ds, es = d64[order], eps_both[order]
        oracle_rows = oracle_keys[q].astype(np.int64) - 1
        for i in range(k):
            below = i == 0 or ds[i] - ds[i - 1] > es[i] + es[i - 1]
            above = ds[i + 1] - ds[i] > es[i] + es[i + 1]
            if below and above:
                assert rows[i] == order[i] and oracle_rows[i] == order[i], (q, i, rows[i], oracle_rows[i], order[i])


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
def test_width256_search_on_oracle_graph(eng, port, metric):
    """Codes up to 255 (the oracle's encoder without the compat-128 loop quirk): the engine loads the oracle's file with
    256-wide tables and searches the same graph.  ef >= n makes both walks exhaustive over the graph."""
    rng = np.random.default_rng(41)
    d, nsub, ncent, n, nq, k = 64, 16, 256, 1000, 40, 10
    X, Q = structured(n, d, 41), structured(nq, d, 42)
    cb = X[rng.choice(n, ncent, replace=False)].copy()
    p = port_pq(port, X, cb, nsub, metric, False, M=M, efc=64, ef=32)
    g = new_index(eng, metric, cb, nsub)
    buf = p.save_buffer()
    g.load_buffer(buf)
    codes = get_codes(buf, M, nsub)
    assert codes.max() >= 128
    gk, gd, gc = g.search_batch(Q, k, ef=1024)
    pk, pd, pc, _ = p.search_batch(Q, k, ef=1024)
    assert np.array_equal(gc.astype(np.int64), pc)
    assert np.allclose(gd, pd, rtol=1e-5, atol=1e-5), np.abs(gd - pd).max()
    assert_search_matches_float64(metric, cb, codes, nsub, Q, gk, gd, pk)


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
def test_wide_code_rows_end_to_end(eng, port, metric):
    """dims = nsub = 1536 with 16 centroids: code rows of 96 chunks take PqEval::eval's wide-row branch in every search and
    build distance.  (PQ indexes refuse 2000 dimensions or more, so 1025..1999 subvectors are the whole range of that branch.)"""
    rng = np.random.default_rng(43)
    d = nsub = 1536
    ncent, n, nq, k = 16, 500, 30, 10
    X, Q = structured(n, d, 43), structured(nq, d, 44)
    cb = X[rng.choice(n, ncent, replace=False)].copy()
    p = port_pq(port, X, cb, nsub, metric, True, M=M, efc=48, ef=32)
    g = new_index(eng, metric, cb, nsub)
    buf = p.save_buffer()
    g.load_buffer(buf)
    codes = get_codes(buf, M, nsub)
    gk, gd, gc = g.search_batch(Q, k, ef=512)
    pk, pd, pc, _ = p.search_batch(Q, k, ef=512)
    assert np.array_equal(gc.astype(np.int64), pc)
    assert np.allclose(gd, pd, rtol=1e-5, atol=1e-5), np.abs(gd - pd).max()
    assert_search_matches_float64(metric, cb, codes, nsub, Q, gk, gd, pk)
    # the engine's own batched build at this geometry: recall against the brute force over the decoded corpus
    N = 3000
    Y = structured(N, d, 45)
    b = new_index(eng, metric, cb, nsub)
    b.reserve(N)
    b.add_batch(np.arange(1, N + 1, dtype=np.uint64), Y)
    b.build()
    bk, _, _ = b.search_batch(Q, k, ef=128)
    dec = eng.dequantize_pq(cb, eng.quantize_pq(cb, Y, nsub, compat128=True)).astype(np.float64)
    if metric == "l2sq":
        D = (Q.astype(np.float64) ** 2).sum(1)[:, None] - 2 * Q.astype(np.float64) @ dec.T + (dec ** 2).sum(1)[None]
    else:
        D = 1 - (Q.astype(np.float64) @ dec.T) / np.outer(np.linalg.norm(Q.astype(np.float64), axis=1), np.linalg.norm(dec, axis=1))
    truth = np.argsort(D, axis=1)[:, :k] + 1
    rec = np.mean([len(set(a.tolist()) & set(t.tolist())) / k for a, t in zip(bk, truth)])
    assert rec > 0.85, rec  # hnsw_pq_index.sql:129-131: index recall within 0.1 of PQ-exact


# ---- a table too large for shared memory ------------------------------------------------------------------------------

def test_table_too_large_for_shared_memory_is_refused_at_load(eng):
    """dims = nsub = 232, 256 centroids: the index is accepted (its codes stay below 128, a 232 x 128 table), but a file
    holding a code >= 128 needs the 232 x 256 table, more than the 227 KB a CTA may have.  Loading it is refused with the
    size the kernels' layout needs, and nothing changes: the index answers as before, other indexes search as before."""
    rng = np.random.default_rng(51)
    d = nsub = 232
    cb = rng.standard_normal((256, d)).astype(np.float32)
    codes = rng.integers(0, 128, (300, nsub)).astype(np.uint8)
    h = pq_index(eng, "l2sq", cb, nsub, codes)
    Q = rng.standard_normal((20, d)).astype(np.float32)
    k0, d0, c0 = h.search_batch(Q, 5)
    wide = codes.copy()
    wide[7, 3] = 200
    buf = set_codes(h.save_buffer(), wide, M)
    for idx in (h, new_index(eng, "l2sq", cb, nsub)):
        with pytest.raises(eng.EngineError) as e:
            idx.load_buffer(buf)
        m = re.search(r"232 x 256 look-up table needs (\d+) bytes of shared memory per CTA; the device allows (\d+)", str(e.value))
        assert m and int(m.group(1)) > int(m.group(2)), str(e.value)
    k1, d1, c1 = h.search_batch(Q, 5)
    assert np.array_equal(k0, k1) and np.array_equal(d0.view(np.uint32), d1.view(np.uint32)) and np.array_equal(c0, c1)
    X = structured(500, 32, 52)
    other = eng.Index(32, "l2sq", "f32", M=8, efc=32, ef=32)
    other.add_batch(np.arange(1, 501, dtype=np.uint64), X)
    ok, od, _ = other.search_batch(X[:10], 3)
    assert (ok[:, 0] == np.arange(1, 11)).all() and (od[:, 0] == 0).all()


# ---- the encoder --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("compat128", [True, False])
@pytest.mark.parametrize("sd,nsub,ncent", [(1, 8, 16), (3, 8, 129), (12, 8, 256), (96, 2, 256)])
def test_quantize_is_float64_argmin_lowest_id(eng, sd, nsub, ncent, compat128):
    """quantize_pq picks, per subvector, the centroid at the smallest squared distance, the lowest id among exact ties
    (duplicated centroids in the same lane of the encoder's warp, the next lane, and past the compat-128 limit).  Where two
    centroids are closer than the fp32 rounding of their distances (one ulp apart) either may win.  compat128 considers
    centroids 0..127 only.  dequantize_pq returns the selected slices bit for bit."""
    rng = np.random.default_rng(sd * 1000 + ncent)
    d = sd * nsub
    cb = rng.standard_normal((ncent, d)).astype(np.float32)
    cb3 = cb.reshape(ncent, nsub, sd)
    base = np.arange(nsub) % 16
    for s in range(nsub):
        c = int(base[s])
        for dup in (c + 1, c + 32, c + 128):
            if dup < ncent:
                cb3[dup, s] = cb3[c, s]
        if c + 64 < ncent:
            cb3[c + 64, s] = cb3[c, s]
            cb3[c + 64, s, 0] = np.nextafter(cb3[c, s, 0], np.float32(np.inf))
    n = 600
    X = rng.standard_normal((n, d)).astype(np.float32).reshape(n, nsub, sd)
    X[:200] = cb3[base, np.arange(nsub)] + np.float32(1e-3) * rng.standard_normal((200, nsub, sd)).astype(np.float32)
    X[200:300] = cb3[base, np.arange(nsub)]  # exactly on the tied centroids
    X = X.reshape(n, d)
    codes = eng.quantize_pq(cb, X, nsub, compat128=compat128)
    limit = 128 if compat128 and ncent > 128 else ncent
    assert codes.max() < limit
    x64 = X.astype(np.float64).reshape(n, nsub, sd)
    c64 = cb3[:limit].astype(np.float64)
    for s in range(nsub):
        D = ((x64[:, s, None, :] - c64[None, :, s, :]) ** 2).sum(-1)  # [n][limit]
        e = (sd + 3) * U * D  # bound on the fp32 rounding of each distance
        for i in range(n):
            dist, c = D[i], int(codes[i, s])
            m = dist.min()
            group = np.nonzero(dist == m)[0]  # exact ties: duplicated centroids, whose fp32 distances are equal too
            # the choice is a float64 minimum up to rounding (a centroid one ulp away may win) ...
            assert dist[c] - m <= 1.01 * (e[i, c] + e[i, group[0]]), (i, s, c, group)
            # ... and among exact ties the lowest id
            if dist[c] == m:
                assert c == group[0], (i, s, c, group)
    dec = eng.dequantize_pq(cb, codes)
    assert np.array_equal(dec.view(np.uint32), cb3[codes, np.arange(nsub)].reshape(n, d).view(np.uint32))
    again = eng.quantize_pq(cb, dec, nsub, compat128=compat128)
    assert np.array_equal(eng.dequantize_pq(cb, again).view(np.uint32), dec.view(np.uint32))


# ---- k-means ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("metric", ["l2sq", "cos"])
@pytest.mark.parametrize("sd", [64, 96])
def test_kmeans_wide_subvectors_against_oracle(eng, port, metric, sd):
    """train_pq at subdim 64 and 96 (the two branches of kmeans_update_kernel) against port.kmeans from the same initial
    rows.  Data are multiples of 2^-8 with small sums, so every centroid sum is exact in both.  Initial centres 3 and 9 of
    every subvector are one outlier row and its copy: they tie for the two outlier rows and the lower id wins, so centre 9
    stays empty in every round and keeps its initial value (the count == 0 branch of the update, from the first assignment
    on; a cluster that loses the members it had is not constructed here).  Training twice gives the same bits."""
    rng = np.random.default_rng(sd)
    nsub, ncent, n = 2, 16, 3000
    d = sd * nsub
    centers = rng.standard_normal((14, d)) * 3
    lab = rng.integers(0, 14, n - 2)
    X = np.empty((n, d))
    X[:n - 2] = centers[lab] + rng.standard_normal((n - 2, d))
    X[n - 2] = X[n - 1] = 12.0 * np.sign(rng.standard_normal(d))
    X = (np.round(X * 256) / 256).astype(np.float32)
    init = np.empty((nsub, ncent), np.uint32)
    firsts = [int(np.nonzero(lab == c)[0][0]) for c in range(14)]
    for s in range(nsub):
        init[s] = firsts[:3] + [n - 2] + firsts[3:8] + [n - 1] + firsts[8:]
    gcb, grounds = eng.train_pq(X, nsub, ncent, metric, max_iter=25, init_rows=init)
    pcb, prounds = port.kmeans(X, nsub, ncent, init, metric, max_iter=25)
    assert grounds == prounds
    assert np.allclose(gcb, pcb, rtol=2e-7, atol=0), np.abs(gcb - pcb).max()
    assert np.array_equal(gcb[9], X[n - 1]) and np.array_equal(gcb[3], X[n - 2])
    gcb2, grounds2 = eng.train_pq(X, nsub, ncent, metric, max_iter=25, init_rows=init)
    assert grounds2 == grounds and np.array_equal(gcb2.view(np.uint32), gcb.view(np.uint32))
