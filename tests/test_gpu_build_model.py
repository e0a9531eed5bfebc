"""The GPU build (build_insert_kernel / build_reverse_kernel) against its CPU model, byte for byte, for every scalar kind.

Each case builds the same keys and rows twice: on the GPU (add_batch + build, build_batch / build_ratio set), and with the
oracle's model of the batched build (ora_add_batch_engine) in the engine's tie order (set_engine_order before adding), and
demands identical index files.  That is only a fair demand when both sides compute the same fp32 bits for every distance,
so every row here is chosen for exact distances: integer coordinates whose products and partial sums stay below 2^24 (any
summation order, fmaf or not, gives the same value), int8 rows whose int32 (GPU) and fp32 (oracle) sums agree below 2^24,
and packed bits (popcounts).  Such data is full of exact distance ties, which is what makes the tie order matter.

The cases cover f32 l2sq / cos (with all-zero and duplicate rows), f16, i8 and b1 rows of several widths, batches of 1,
64 and 1024, M = 4, 16, 32 and 48, efc = 16 and 128, a second build into a built index across a capacity growth, the
device add path with a strided tensor, and the full-bitmap clear of the walks' visited set (touched_cap = 32).
"""
import numpy as np
import pytest

from util import describe_file_difference, make_rows

# name: (quant, metric, dims, rows, n, M, efc, build_batch, build_ratio, extra)
#   rows: ("int", r) integers in [-r, r]; ("int0", r) the same plus all-zero and duplicate rows; ("i8", s) uniform in
#   [-s, s] cast to int8 (plus rows that cast to all zeros); ("bits",) clustered packed bits
#   extra: "grow" = two builds, the second into the built index after a capacity growth; "device" = rows added from a
#   CUDA tensor with a row stride wider than the row; "touched32" = touched_cap 32
CASES = {
    "f32-l2sq-d16-M16-b64": ("f32", "l2sq", 16, ("int", 300), 3000, 16, 128, 64, 64, ""),
    "f32-l2sq-d48-M4-efc16-b1": ("f32", "l2sq", 48, ("int", 8), 3000, 4, 16, 1, 64, ""),
    "f32-l2sq-d100-M16-b1024": ("f32", "l2sq", 100, ("int", 100), 8000, 16, 128, 1024, 4, ""),
    "f32-cos-d32-M32-b64": ("f32", "cos", 32, ("int0", 8), 3000, 32, 128, 64, 64, ""),
    "f32-cos-d48-M48-b1": ("f32", "cos", 48, ("int0", 40), 2000, 48, 128, 1, 64, ""),
    "f32-cos-d24-M4-efc16-grow": ("f32", "cos", 24, ("int0", 6), 3000, 4, 16, 64, 16, "grow"),
    "f16-l2sq-d72-M16-efc16-grow": ("f16", "l2sq", 72, ("int", 200), 3000, 16, 16, 64, 16, "grow"),
    "f16-cos-d100-M32-b64": ("f16", "cos", 100, ("int0", 300), 2000, 32, 64, 64, 16, ""),
    "i8-l2sq-d1000-M16-b64": ("i8", "l2sq", 1000, ("i8", 0.5), 700, 16, 64, 64, 8, ""),
    "i8-cos-d80-M48-device": ("i8", "cos", 80, ("i8", 2.0), 2000, 48, 64, 64, 64, "device"),
    "b1-768-M16-b1": ("b1", "hamming", 768, ("bits",), 3000, 16, 128, 1, 64, ""),
    "b1-768-M16-b64-grow": ("b1", "hamming", 768, ("bits",), 3000, 16, 128, 64, 64, "grow"),
    "b1-100-M4-efc16-touched32": ("b1", "hamming", 100, ("bits",), 3000, 4, 16, 64, 64, "touched32"),
    "b1-768-M32-b1024": ("b1", "hamming", 768, ("bits",), 8000, 32, 128, 1024, 4, ""),
    "b1-6144-M32-b64": ("b1", "hamming", 6144, ("bits",), 1500, 32, 64, 64, 16, ""),
}


def batch_sizes(levels, batch_cap, build_ratio):
    """The batch schedule of a first build (ora_add_batch_engine, build.cu plan_batches) for nodes of these levels."""
    sizes, top, visible, pos, P = [1], int(levels[0]), 1, 1, len(levels)
    while pos < P:
        bsz = 1
        if levels[pos] <= top:
            bsz = min(P - pos, batch_cap, max(1, visible // build_ratio))
            above = np.nonzero(levels[pos + 1:pos + bsz] > top)[0]
            if len(above):
                bsz = int(above[0]) + 1
        if levels[pos] > top:
            top = int(levels[pos])
        sizes.append(bsz)
        visible += bsz
        pos += bsz
    return sizes


def parts_of(n, extra):
    return [(0, n // 2), (n // 2, n)] if extra == "grow" else [(0, n)]


@pytest.mark.parametrize("name", list(CASES))
def test_rows_have_exact_distances(port, name):
    """CPU: the generators hold their exactness bounds, and the cases of batch 1 and 1024 really insert batches of that
    size (build_ratio 4 on 8000 rows; at build_ratio 64 on 3000 rows no batch exceeds 46)."""
    quant, metric, dims, rows, n, M, efc, batch, ratio, extra = CASES[name]
    X, S = make_rows(port, quant, metric, dims, rows, n, seed=len(name))
    assert len(X) == n and len(S) == n
    if extra != "grow":
        sizes = batch_sizes(port.level_sequence(M, n), batch, ratio)
        assert sum(sizes) == n and max(sizes) <= batch
        if batch in (1, 1024):
            assert max(sizes) == batch, (name, max(sizes))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_gpu_build_equals_cpu_model(eng, port, name):
    quant, metric, dims, rows, n, M, efc, batch, ratio, extra = CASES[name]
    X, S = make_rows(port, quant, metric, dims, rows, n, seed=len(name))
    keys = np.arange(1, n + 1, dtype=np.uint64) * 7
    parts = parts_of(n, extra)

    p = port.PortIndex(dims, metric, quant, M=M, efc=efc, ef=32)
    p.set_engine_order(True)
    p.reserve(n)
    for a, b in parts:
        p.add_batch_engine(keys[a:b], X[a:b], batch, ratio)

    g = eng.Index(dims, metric, quant, M=M, efc=efc, ef=32)
    g.set_option("build_batch", batch)
    g.set_option("build_ratio", ratio)
    if extra == "touched32":
        g.set_option("touched_cap", 32)
    if extra == "grow":
        g.reserve(n // 4)  # the first add grows the capacity, the reserve before the second grows it again
        g.add_batch(keys[:n // 2], X[:n // 2])
        g.build()
        assert g.size() == n // 2
        g.reserve(n)
        g.add_batch(keys[n // 2:], X[n // 2:])
        g.build()
    elif extra == "device":
        import torch
        T = torch.full((n, dims + 5), float("nan"), dtype=torch.float32, device="cuda")
        T[:, :dims] = torch.from_numpy(X).cuda()
        torch.cuda.synchronize()
        g.reserve(n)
        g.add_batch_device(keys, T.data_ptr(), n, T.stride(0) * 4, "f32")
        g.build()
        del T
    else:
        g.reserve(n)
        g.add_batch(keys, X)
        g.build()
    assert g.size() == n

    gb, pb = g.save_buffer(), p.save_buffer()
    stored = S.shape[1] * S.itemsize
    assert np.array_equal(gb, pb), describe_file_difference(gb, pb, M, stored, S, metric, quant, dims, port)
