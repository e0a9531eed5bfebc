"""ctypes binding of liblantern_b200.so -- the harness-side view of the C ABI (include/lantern_b200.h).

The product is the shared library; this module only marshals numpy arrays / raw device pointers into
it for tests and bench.py, mirroring usearch's `Index` surface (U/rust/lib.rs:1-92: new, reserve,
add, search, save, load, size, ...).  It never computes anything itself and there is no fallback:
if the library or a GPU is missing, calls raise.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "liblantern_b200.so")

METRIC = {"cos": 1, "ip": 2, "l2sq": 3, "hamming": 8}
SCALAR = {"f32": 1, "f64": 2, "f16": 3, "i8": 4, "b1": 5}
NP_OF = {"f32": np.float32, "f16": np.uint16, "i8": np.int8, "b1": np.uint8}


class InitOptions(C.Structure):  # == usearch_init_options_t (U/c/usearch.h:74-117)
    _fields_ = [
        ("metric_kind", C.c_int),
        ("metric", C.c_void_p),
        ("quantization", C.c_int),
        ("dimensions", C.c_size_t),
        ("connectivity", C.c_size_t),
        ("expansion_add", C.c_size_t),
        ("expansion_search", C.c_size_t),
        ("multi", C.c_bool),
        ("retriever_ctx", C.c_void_p),
        ("retriever", C.c_void_p),
        ("retriever_mut", C.c_void_p),
        ("num_threads", C.c_size_t),
        ("pq", C.c_bool),
        ("num_centroids", C.c_size_t),
        ("num_subvectors", C.c_size_t),
    ]


class IndexMetadata(C.Structure):  # == usearch_index_metadata_t (usearch.h:119-131)
    _fields_ = [
        ("init_options", InitOptions),
        ("inverse_log_connectivity", C.c_double),
        ("neighbors_bytes", C.c_size_t),
        ("neighbors_base_bytes", C.c_size_t),
        ("dimensions", C.c_size_t),
        ("expansion_search", C.c_size_t),
        ("expansion_add", C.c_size_t),
        ("connectivity", C.c_size_t),
        ("metric_kind", C.c_int),
    ]


class SearchStats(C.Structure):
    _fields_ = [("queries", C.c_uint64), ("computed_distances", C.c_uint64), ("base_pops", C.c_uint64),
                ("upper_hops", C.c_uint64), ("algorithmic_bytes", C.c_uint64), ("kernel_ms", C.c_double),
                ("limbo_overflows", C.c_uint64), ("full_rows_read", C.c_uint64), ("screen_kind", C.c_uint32),
                ("screen_dims", C.c_uint32), ("search_kernel", C.c_uint32), ("reserved", C.c_uint32),
                ("owner_cycles_produce", C.c_uint64), ("owner_cycles_screen", C.c_uint64), ("owner_cycles_evaluate", C.c_uint64),
                ("owner_cycles_consume", C.c_uint64)]


class BuildStats(C.Structure):
    _fields_ = [("vectors", C.c_uint64), ("computed_distances", C.c_uint64), ("algorithmic_bytes", C.c_uint64),
                ("device_ms", C.c_double)]


class GroupStats(C.Structure):
    _fields_ = [("rank", C.c_int), ("world", C.c_int), ("queries", C.c_uint64), ("owner_computed_distances", C.c_uint64),
                ("owner_base_pops", C.c_uint64), ("owner_upper_hops", C.c_uint64), ("owner_rounds", C.c_uint64),
                ("local_rows_evaluated", C.c_uint64), ("local_row_bytes", C.c_uint64), ("rows_held", C.c_uint64),
                ("kernel_ms", C.c_double), ("owner_cycles_produce", C.c_uint64), ("owner_cycles_local", C.c_uint64),
                ("owner_cycles_wait", C.c_uint64), ("owner_cycles_consume", C.c_uint64)]


class GroupRankInfo(C.Structure):
    _fields_ = [("rank", C.c_int), ("world", C.c_int), ("rows_begin", C.c_uint64), ("rows_end", C.c_uint64),
                ("bytes_rows", C.c_uint64), ("bytes_graph", C.c_uint64), ("bytes_scratch", C.c_uint64),
                ("bytes_mailbox", C.c_uint64)]


ALLGATHER_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t)
ERRP = C.POINTER(C.c_char_p)

# name -> (restype, argtypes); the same table drives the symbol-export test
SIGNATURES = {
    "lb200_init": (C.c_void_p, [C.POINTER(InitOptions), C.c_void_p, ERRP]),
    "lb200_free": (None, [C.c_void_p, ERRP]),
    "lb200_size": (C.c_size_t, [C.c_void_p, ERRP]),
    "lb200_capacity": (C.c_size_t, [C.c_void_p, ERRP]),
    "lb200_dimensions": (C.c_size_t, [C.c_void_p, ERRP]),
    "lb200_connectivity": (C.c_size_t, [C.c_void_p, ERRP]),
    "lb200_expansion_add": (C.c_size_t, [C.c_void_p, ERRP]),
    "lb200_expansion_search": (C.c_size_t, [C.c_void_p, ERRP]),
    "lb200_index_metadata": (IndexMetadata, [C.c_void_p, ERRP]),
    "lb200_reserve": (None, [C.c_void_p, C.c_size_t, ERRP]),
    "lb200_add": (None, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, ERRP]),
    "lb200_add_batch": (None, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, ERRP]),
    "lb200_add_batch_device": (None, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, ERRP]),
    "lb200_build": (None, [C.c_void_p, ERRP]),
    "lb200_last_build_stats": (None, [C.c_void_p, C.POINTER(BuildStats), ERRP]),
    "lb200_set_option": (None, [C.c_void_p, C.c_char_p, C.c_size_t, ERRP]),
    "lb200_search_ef": (C.c_size_t, [C.c_void_p, C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, C.c_bool, C.c_void_p,
                                      C.c_void_p, ERRP]),
    "lb200_search": (C.c_size_t, [C.c_void_p, C.c_void_p, C.c_int, C.c_size_t, C.c_void_p, C.c_void_p, ERRP]),
    "lb200_search_batch": (None, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t, C.c_size_t,
                                  C.c_void_p, C.c_void_p, C.c_void_p, ERRP]),
    "lb200_search_batch_device": (None, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t,
                                         C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, ERRP]),
    "lb200_last_search_stats": (None, [C.c_void_p, C.POINTER(SearchStats), ERRP]),
    "lb200_serialized_length": (C.c_size_t, [C.c_void_p, ERRP]),
    "lb200_save_buffer": (None, [C.c_void_p, C.c_void_p, C.c_size_t, ERRP]),
    "lb200_load_buffer": (None, [C.c_void_p, C.c_void_p, C.c_size_t, ERRP]),
    "lb200_view_buffer": (None, [C.c_void_p, C.c_void_p, C.c_size_t, ERRP]),
    "lb200_save": (None, [C.c_void_p, C.c_char_p, ERRP]),
    "lb200_load": (None, [C.c_void_p, C.c_char_p, ERRP]),
    "lb200_view": (None, [C.c_void_p, C.c_char_p, ERRP]),
    "lb200_metadata_buffer": (None, [C.c_void_p, C.c_size_t, C.POINTER(InitOptions), ERRP]),
    "lb200_metadata": (None, [C.c_char_p, C.POINTER(InitOptions), ERRP]),
    "lb200_update_header": (None, [C.c_void_p, C.c_void_p, ERRP]),
    "lb200_count": (C.c_size_t, [C.c_void_p, C.c_uint64, ERRP]),
    "lb200_contains": (C.c_bool, [C.c_void_p, C.c_uint64, ERRP]),
    "lb200_header_get_entry_slot": (C.c_uint64, [C.c_void_p]),
    "lb200_header_set_entry_slot": (None, [C.c_void_p, C.c_uint64]),
    "lb200_distance": (C.c_float, [C.c_void_p, C.c_void_p, C.c_int, C.c_size_t, C.c_int, ERRP]),
    "lb200_distance_batch": (None, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t,
                                    C.c_int, C.c_void_p, ERRP]),
    "lb200_exact_search": (None, [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int,
                                  C.c_size_t, C.c_int, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                  C.c_size_t, ERRP]),
    "lb200_exact_search_device": (None, [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int,
                                         C.c_size_t, C.c_int, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, ERRP]),
    "lb200_exact_tc_probe": (None, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p, ERRP]),
    "lb200_search_screen_probe": (None, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_void_p,
                                         C.c_void_p, ERRP]),
    "lb200_search_pscreen_probe": (None, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_void_p,
                                          C.c_size_t, C.c_void_p, C.c_void_p, ERRP]),
    "lb200_screen_basis": (C.c_size_t, [C.c_void_p, C.c_void_p, C.POINTER(C.c_double), ERRP]),
    "lb200_pq_probe": (None, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t),
                              C.POINTER(C.c_size_t), C.c_void_p, C.c_void_p, ERRP]),
    "lb200_cast": (None, [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_int, ERRP]),
    "lb200_cast_batch": (None, [C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_void_p, ERRP]),
    "lb200_quantize_pq": (None, [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                 C.c_int, ERRP]),
    "lb200_dequantize_pq": (None, [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                   ERRP]),
    "lb200_train_pq": (C.c_int, [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t, C.c_uint64,
                                 C.c_void_p, C.c_void_p, ERRP]),
    "lb200_train_pq_device": (C.c_int, [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int,
                                        C.c_size_t, C.c_uint64, C.c_void_p, C.c_void_p, ERRP]),
    "lb200_merge_shards_device": (None, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p,
                                         C.c_void_p, C.c_void_p, ERRP]),
    "lb200_group_create": (C.c_void_p, [C.c_int, C.c_int, ALLGATHER_FN, C.c_void_p, ERRP]),
    "lb200_group_create_local": (C.c_void_p, [C.c_void_p, C.c_int, ERRP]),
    "lb200_group_free": (None, [C.c_void_p, ERRP]),
    "lb200_group_distribute": (None, [C.c_void_p, C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, ERRP]),
    "lb200_group_load_buffer": (None, [C.c_void_p, C.POINTER(InitOptions), C.c_void_p, C.c_size_t, C.c_int, C.c_size_t,
                                       C.c_size_t, ERRP]),
    "lb200_group_load": (None, [C.c_void_p, C.POINTER(InitOptions), C.c_char_p, C.c_int, C.c_size_t, C.c_size_t, ERRP]),
    "lb200_group_rank_info": (None, [C.c_void_p, C.c_int, C.POINTER(GroupRankInfo), ERRP]),
    "lb200_group_build": (None, [C.c_void_p, C.c_void_p, C.c_int, ERRP]),
    "lb200_group_index_init": (None, [C.c_void_p, C.POINTER(InitOptions), C.c_size_t, C.c_size_t, C.c_size_t, ERRP]),
    "lb200_group_index_load_buffer": (None, [C.c_void_p, C.POINTER(InitOptions), C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t,
                                             C.c_size_t, ERRP]),
    "lb200_group_index_load": (None, [C.c_void_p, C.POINTER(InitOptions), C.c_char_p, C.c_size_t, C.c_size_t, C.c_size_t, ERRP]),
    "lb200_group_index_reserve": (None, [C.c_void_p, C.c_size_t, ERRP]),
    "lb200_group_index_add_batch": (None, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, ERRP]),
    "lb200_group_index_set_option": (None, [C.c_void_p, C.c_char_p, C.c_size_t, ERRP]),
    "lb200_group_index_build": (None, [C.c_void_p, ERRP]),
    "lb200_group_index_size": (C.c_size_t, [C.c_void_p, ERRP]),
    "lb200_group_index_last_build_stats": (None, [C.c_void_p, C.POINTER(BuildStats), ERRP]),
    "lb200_group_index_serialized_length": (C.c_size_t, [C.c_void_p, ERRP]),
    "lb200_group_index_save_buffer": (None, [C.c_void_p, C.c_void_p, C.c_size_t, ERRP]),
    "lb200_group_index_save": (None, [C.c_void_p, C.c_char_p, ERRP]),
    "lb200_group_search_batch": (None, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t, C.c_size_t,
                                        C.c_void_p, C.c_void_p, C.c_void_p, ERRP]),
    "lb200_group_search_batch_device": (None, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t, C.c_size_t,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, ERRP]),
    "lb200_group_plan": (C.c_int, [C.c_int, C.c_size_t, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    "lb200_group_selftest_exchange": (C.c_int, [C.c_int, C.c_int, ALLGATHER_FN, C.c_void_p]),
    "lb200_group_last_stats": (None, [C.c_void_p, C.c_int, C.POINTER(GroupStats), ERRP]),
    "lb200_device_count": (C.c_int, []),
    "lb200_version": (C.c_char_p, []),
    "lb200_kernel_launches": (C.c_uint64, []),
}

_lib = None


def lib():
    """Loads the engine.  Raises if the library has not been built (no silent fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO):
            raise RuntimeError("liblantern_b200.so is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
        L = C.CDLL(SO)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


class EngineError(RuntimeError):
    pass


def _check(err):
    if err.value:
        raise EngineError(err.value.decode())


def _ptr(x):
    """numpy array -> host pointer; int -> raw (device) pointer; None -> NULL."""
    if x is None:
        return None
    if isinstance(x, int):
        return C.c_void_p(x)
    return C.c_void_p(x.ctypes.data)


def init_options(dim, metric="l2sq", quant="f32", M=16, efc=128, ef=64, pq=False, num_centroids=0, num_subvectors=0):
    o = InitOptions()
    o.metric_kind, o.quantization, o.dimensions = METRIC[metric], SCALAR[quant], dim
    o.connectivity, o.expansion_add, o.expansion_search = M, efc, ef
    o.pq, o.num_centroids, o.num_subvectors = pq, num_centroids, num_subvectors
    return o


class Index:
    """One HNSW index resident in the HBM of the current CUDA device."""

    def __init__(self, dim, metric="l2sq", quant="f32", M=16, efc=128, ef=64, pq=False, num_centroids=0,
                 num_subvectors=0, codebook=None):
        L = lib()
        self.dim, self.metric, self.quant, self.M = dim, metric, quant, M
        self.num_subvectors = num_subvectors
        o = init_options(dim, metric, quant, M, efc, ef, pq, num_centroids, num_subvectors)
        cb = None
        if codebook is not None:
            cb = np.ascontiguousarray(codebook, dtype=np.float32)
        err = C.c_char_p()
        self.h = L.lb200_init(C.byref(o), _ptr(cb), C.byref(err))
        _check(err)
        if not self.h:
            raise EngineError("lb200_init returned NULL")

    def close(self):
        if getattr(self, "h", None) and C is not None and _lib is not None:  # (both vanish during interpreter shutdown)
            err = C.c_char_p()
            _lib.lb200_free(self.h, C.byref(err))
            self.h = None

    __del__ = close

    @staticmethod
    def _kind(arr):
        return SCALAR["b1"] if arr.dtype == np.uint8 else SCALAR["f32"]

    def _call(self, name, *args):
        err = C.c_char_p()
        r = getattr(lib(), name)(self.h, *args, C.byref(err))
        _check(err)
        return r

    def size(self):
        return self._call("lb200_size")

    def capacity(self):
        return self._call("lb200_capacity")

    def reserve(self, n):
        self._call("lb200_reserve", n)

    def metadata(self):
        return self._call("lb200_index_metadata")

    def add(self, key, vec):
        vec = np.ascontiguousarray(vec)
        self._call("lb200_add", int(key), _ptr(vec), self._kind(vec))

    def add_batch(self, keys, vecs):
        vecs = np.ascontiguousarray(vecs)
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        self._call("lb200_add_batch", _ptr(keys), _ptr(vecs), len(keys), vecs.strides[0], self._kind(vecs))

    def add_batch_device(self, keys, dptr, n, stride, kind="f32"):
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        self._call("lb200_add_batch_device", _ptr(keys), C.c_void_p(dptr), n, stride, SCALAR[kind])

    def build(self):
        self._call("lb200_build")

    def last_build_stats(self):
        s = BuildStats()
        self._call("lb200_last_build_stats", C.byref(s))
        return {f: getattr(s, f) for f, _ in BuildStats._fields_}

    def set_option(self, name, value):
        self._call("lb200_set_option", name.encode(), int(value))

    def search(self, q, k, ef=0):
        q = np.ascontiguousarray(q)
        keys = np.zeros(k, np.uint64)
        dists = np.zeros(k, np.float32)
        n = self._call("lb200_search_ef", _ptr(q), self._kind(q), k, ef, False, _ptr(keys), _ptr(dists))
        return keys[:n], dists[:n]

    def search_batch(self, queries, k, ef=0):
        queries = np.ascontiguousarray(queries)
        nq = len(queries)
        keys = np.zeros((nq, k), np.uint64)
        dists = np.zeros((nq, k), np.float32)
        counts = np.zeros(nq, np.uint64)
        self._call("lb200_search_batch", _ptr(queries), nq, queries.strides[0], self._kind(queries), k, ef, _ptr(keys),
                   _ptr(dists), _ptr(counts))
        return keys, dists, counts

    def search_batch_raw(self, q_ptr, nq, stride, kind, k, ef, keys_ptr, dists_ptr, counts_ptr):
        """Host pointers in, host pointers out (pinned or pageable): the reference-facing e2e call."""
        self._call("lb200_search_batch", C.c_void_p(q_ptr), nq, stride, SCALAR[kind], k, ef, C.c_void_p(keys_ptr),
                   C.c_void_p(dists_ptr), C.c_void_p(counts_ptr) if counts_ptr else None)

    def search_batch_device(self, q_dptr, nq, stride, kind, k, ef, keys_dptr, dists_dptr, counts_dptr=0, stream=0):
        self._call("lb200_search_batch_device", C.c_void_p(q_dptr), nq, stride, SCALAR[kind], k, ef, C.c_void_p(keys_dptr),
                   C.c_void_p(dists_dptr), C.c_void_p(counts_dptr) if counts_dptr else None,
                   C.c_void_p(stream) if stream else None)

    def last_stats(self):
        s = SearchStats()
        self._call("lb200_last_search_stats", C.byref(s))
        return {f: getattr(s, f) for f, _ in SearchStats._fields_}

    def screen_basis(self):
        """(k x dims float32 basis of the projected screen, or None when the index keeps none; seconds its choice took)"""
        sec = C.c_double()
        k = self._call("lb200_screen_basis", None, C.byref(sec))
        if not k:
            return None, sec.value
        P = np.zeros((k, self.dim), np.float32)
        self._call("lb200_screen_basis", _ptr(P), None)
        return P, sec.value

    def save_buffer(self):
        n = self._call("lb200_serialized_length")
        buf = np.zeros(n, np.uint8)
        self._call("lb200_save_buffer", _ptr(buf), n)
        return buf

    def load_buffer(self, buf):
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        self._call("lb200_load_buffer", _ptr(buf), len(buf))

    def save(self, path):
        self._call("lb200_save", path.encode())

    def load(self, path):
        self._call("lb200_load", path.encode())


class Group:
    """One graph searched by several GPUs (include/lantern_b200.h, "row-sharded group").

    Group.local(devices)            one process driving len(devices) devices
    Group.ranked(rank, world, ag)   one process per GPU; `ag(send: bytes) -> bytes` is the caller's all-gather
                                    (concatenation of every rank's `send`, rank order), used for bootstrap only
    then once: distribute(index) (an index on the root's GPU) or load(path) / load_buffer(bytes) (each rank reads its rows)
               or index_init(capacity, ...) (an index of the group's own: index_add_batch, index_build, index_save)
               or index_load(path, capacity, ...) / index_load_buffer (the same, opened from a file); index_reserve grows it
    """

    def __init__(self, handle, world, keep=None):
        self.h, self.world, self._keep = handle, world, keep

    @classmethod
    def local(cls, devices):
        arr = (C.c_int * len(devices))(*devices)
        err = C.c_char_p()
        h = lib().lb200_group_create_local(arr, len(devices), C.byref(err))
        _check(err)
        return cls(h, len(devices))

    @staticmethod
    def _callback(world, allgather):
        def _ag(ctx, send, recv, nbytes):
            out = allgather(C.string_at(send, nbytes))
            assert len(out) == nbytes * world, (len(out), nbytes, world)
            C.memmove(recv, out, len(out))
        return ALLGATHER_FN(_ag)

    @staticmethod
    def plan(world, nq, resident_warps, owner_slots_max):
        """(ok, owners, helpers) of a launch (host-only)."""
        o, h = C.c_uint32(), C.c_uint32()
        rc = lib().lb200_group_plan(world, nq, resident_warps, owner_slots_max, C.byref(o), C.byref(h))
        return rc == 0, o.value, h.value

    @staticmethod
    def selftest_exchange(rank, world, allgather):
        """Host-only: drives `allgather` through the C ABI exactly as group creation does; 0 = fine."""
        return lib().lb200_group_selftest_exchange(rank, world, Group._callback(world, allgather), None)

    @classmethod
    def ranked(cls, rank, world, allgather):
        cb = cls._callback(world, allgather)
        err = C.c_char_p()
        h = lib().lb200_group_create(rank, world, cb, None, C.byref(err))
        _check(err)
        return cls(h, world, keep=cb)

    def close(self):
        if getattr(self, "h", None) and C is not None and _lib is not None:
            err = C.c_char_p()
            _lib.lb200_group_free(self.h, C.byref(err))
            self.h = None

    __del__ = close

    def _call(self, name, *args):
        err = C.c_char_p()
        r = getattr(lib(), name)(self.h, *args, C.byref(err))
        _check(err)
        return r

    def distribute(self, index, root=0, max_batch=8192, max_results=0):
        self._call("lb200_group_distribute", index.h if index is not None else None, root, max_batch, max_results)

    def load_buffer(self, buf, dim, metric="l2sq", quant="f32", M=16, efc=128, ef=64, pq=False, root=0, max_batch=8192,
                    max_results=0):
        """The group's graph straight from index file bytes (every rank passes the same bytes); the index options are those
        of Index(...) and are checked against the file as Index.load_buffer checks them."""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        o = init_options(dim, metric, quant, M, efc, ef, pq)
        self._call("lb200_group_load_buffer", C.byref(o), _ptr(buf), len(buf), root, max_batch, max_results)

    def load(self, path, dim, metric="l2sq", quant="f32", M=16, efc=128, ef=64, pq=False, root=0, max_batch=8192,
             max_results=0):
        """load_buffer from a file, mapped read-only by the engine."""
        o = init_options(dim, metric, quant, M, efc, ef, pq)
        self._call("lb200_group_load", C.byref(o), path.encode(), root, max_batch, max_results)

    def rank_info(self, local_rank=0):
        """Row range and device bytes (rows, graph, scratch, mailbox) of a local rank."""
        s = GroupRankInfo()
        self._call("lb200_group_rank_info", local_rank, C.byref(s))
        return {f: getattr(s, f) for f, _ in GroupRankInfo._fields_}

    def build(self, index, root=0):
        """Insert every pending vector of `index` (on rank `root`'s device) with all ranks: lb200_build's graph, byte for byte."""
        self._call("lb200_group_build", index.h if index is not None else None, root)

    # ---- the group's own index (lb200_group_index_*): built straight into the row-sharded layout ----
    def index_init(self, capacity, dim, metric="l2sq", quant="f32", M=16, efc=128, ef=64, pq=False, max_batch=8192,
                   max_results=0):
        """An empty index of the group's own with room for `capacity` rows; rank r holds rows [capacity r / G, capacity (r+1) / G)."""
        o = init_options(dim, metric, quant, M, efc, ef, pq)
        self._call("lb200_group_index_init", C.byref(o), capacity, max_batch, max_results)

    def index_load_buffer(self, buf, capacity, dim, metric="l2sq", quant="f32", M=16, efc=128, ef=64, pq=False, max_batch=8192,
                          max_results=0):
        """An index of the group's own whose contents come from index file bytes, with room for `capacity` rows (0 = the
        file's rows); rank r receives only the rows of [capacity r / G, capacity (r+1) / G).  The options are checked against
        the file as Index.load_buffer checks them."""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        o = init_options(dim, metric, quant, M, efc, ef, pq)
        self._call("lb200_group_index_load_buffer", C.byref(o), _ptr(buf), len(buf), capacity, max_batch, max_results)

    def index_load(self, path, capacity, dim, metric="l2sq", quant="f32", M=16, efc=128, ef=64, pq=False, max_batch=8192,
                   max_results=0):
        """index_load_buffer from a file, mapped read-only by the engine."""
        o = init_options(dim, metric, quant, M, efc, ef, pq)
        self._call("lb200_group_index_load", C.byref(o), path.encode(), capacity, max_batch, max_results)

    def index_reserve(self, capacity):
        """Room for `capacity` rows (nothing happens at or below the current capacity): the ranges become
        [capacity r / G, capacity (r+1) / G) and the rows move to the ranks that now hold them."""
        self._call("lb200_group_index_reserve", capacity)

    def index_add_batch(self, keys, vecs):
        vecs = np.ascontiguousarray(vecs)
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        self._call("lb200_group_index_add_batch", _ptr(keys), _ptr(vecs), len(keys), vecs.strides[0], Index._kind(vecs))

    def index_set_option(self, name, value):
        self._call("lb200_group_index_set_option", name.encode(), int(value))

    def index_build(self):
        self._call("lb200_group_index_build")

    def index_size(self):
        return self._call("lb200_group_index_size")

    def index_last_build_stats(self):
        s = BuildStats()
        self._call("lb200_group_index_last_build_stats", C.byref(s))
        return {f: getattr(s, f) for f, _ in BuildStats._fields_}

    def index_save_buffer(self):
        n = self._call("lb200_group_index_serialized_length")
        buf = np.zeros(n, np.uint8)
        self._call("lb200_group_index_save_buffer", _ptr(buf), n)
        return buf

    def index_save(self, path):
        self._call("lb200_group_index_save", path.encode())

    def search_batch(self, queries, k, ef=0, nq=None, dim_bytes=None, kind=None):
        """Host buffers.  Non-root ranks of a multi-process group pass queries=None with nq / dim_bytes / kind."""
        if queries is not None:
            queries = np.ascontiguousarray(queries)
            nq, stride, kind_id = len(queries), queries.strides[0], Index._kind(queries)
        else:
            stride, kind_id = dim_bytes, SCALAR[kind]
        keys = np.zeros((nq, k), np.uint64)
        dists = np.zeros((nq, k), np.float32)
        counts = np.zeros(nq, np.uint64)
        self._call("lb200_group_search_batch", _ptr(queries), nq, stride, kind_id, k, ef, _ptr(keys), _ptr(dists), _ptr(counts))
        return keys, dists, counts

    def search_batch_raw(self, q_ptr, nq, stride, kind, k, ef, keys_ptr, dists_ptr, counts_ptr):
        self._call("lb200_group_search_batch", C.c_void_p(q_ptr) if q_ptr else None, nq, stride, SCALAR[kind], k, ef,
                   C.c_void_p(keys_ptr), C.c_void_p(dists_ptr), C.c_void_p(counts_ptr) if counts_ptr else None)

    def search_batch_device(self, q_dptr, nq, stride, kind, k, ef, keys_dptr, dists_dptr, counts_dptr=0, stream=0):
        self._call("lb200_group_search_batch_device", C.c_void_p(q_dptr) if q_dptr else None, nq, stride, SCALAR[kind], k, ef,
                   C.c_void_p(keys_dptr) if keys_dptr else None, C.c_void_p(dists_dptr) if dists_dptr else None,
                   C.c_void_p(counts_dptr) if counts_dptr else None, C.c_void_p(stream) if stream else None)

    def last_stats(self, local_rank=0):
        s = GroupStats()
        self._call("lb200_group_last_stats", local_rank, C.byref(s))
        return {f: getattr(s, f) for f, _ in GroupStats._fields_}


def _static(name, *args):
    err = C.c_char_p()
    r = getattr(lib(), name)(*args, C.byref(err))
    _check(err)
    return r


def distance(a, b, metric, quant="f32", dims=None):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if dims is None:
        dims = a.size * 8 if quant == "b1" else a.size
    return _static("lb200_distance", _ptr(a), _ptr(b), SCALAR[quant], dims, METRIC[metric])


def distance_batch(a, b, metric, quant="f32", dims=None):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if dims is None:
        dims = a.shape[1] * 8 if quant == "b1" else a.shape[1]
    out = np.zeros(len(a), np.float32)
    _static("lb200_distance_batch", _ptr(a), a.strides[0], _ptr(b), b.strides[0], len(a), SCALAR[quant], dims,
            METRIC[metric], _ptr(out))
    return out


def exact_search(dataset, queries, k, metric="l2sq", quant="f32", dims=None):
    dataset, queries = np.ascontiguousarray(dataset), np.ascontiguousarray(queries)
    if dims is None:
        dims = dataset.shape[1] * 8 if quant == "b1" else dataset.shape[1]
    nq = len(queries)
    keys = np.zeros((nq, k), np.uint64)
    dists = np.zeros((nq, k), np.float32)
    _static("lb200_exact_search", _ptr(dataset), len(dataset), dataset.strides[0], _ptr(queries), nq, queries.strides[0],
            SCALAR[quant], dims, METRIC[metric], k, 0, _ptr(keys), keys.strides[0], _ptr(dists), dists.strides[0])
    return keys, dists


def exact_search_device(d_dataset, n, d_stride, d_queries, nq, q_stride, k, d_keys, d_dists, metric="l2sq", quant="f32",
                        dims=None, stream=0):
    _static("lb200_exact_search_device", C.c_void_p(d_dataset), n, d_stride, C.c_void_p(d_queries), nq, q_stride,
            SCALAR[quant], dims, METRIC[metric], k, C.c_void_p(d_keys), C.c_void_p(d_dists),
            C.c_void_p(stream) if stream else None)


def exact_tc_probe(dataset, queries, k, metric="l2sq"):
    """Test hook: exact_search with the tensor-core filter forced on, plus the filter's intermediate buffers (dict)."""
    X = np.ascontiguousarray(dataset, dtype=np.float32)
    Q = np.ascontiguousarray(queries, dtype=np.float32)
    n, nq, d = len(X), len(Q), X.shape[1]
    plan, eps = np.zeros(2, np.uint32), np.zeros(4, np.float32)
    args = (_ptr(X), n, _ptr(Q), nq, d, METRIC[metric], k, _ptr(plan), _ptr(eps))
    _static("lb200_exact_tc_probe", *args, *([None] * 8))
    G, KP = int(plan[0]), int(plan[1])
    out = dict(groups=G, KP=KP, eps_rel=float(eps[0]), eps_sum=float(eps[1]), eps_lin=float(eps[2]), eps_abs=float(eps[3]),
               qn=np.zeros(nq, np.float32), xn=np.zeros(n, np.float32), cand_d=np.zeros((nq, G, KP), np.float32),
               cand_i=np.zeros((nq, G, KP), np.uint32), dropped_lb=np.zeros((nq, G), np.float32),
               unsafe=np.zeros(nq, np.uint8), keys=np.zeros((nq, k), np.uint64), dists=np.zeros((nq, k), np.float32))
    _static("lb200_exact_tc_probe", *args, *(_ptr(out[f]) for f in ("qn", "xn", "cand_d", "cand_i", "dropped_lb", "unsafe",
                                                                     "keys", "dists")))
    return out


def search_screen_probe(dataset, queries, metric="l2sq"):
    """Test hook: (lb, d), both [nq][n] float32 -- the search screen's lower bound and the search kernel's fp32 distance."""
    X = np.ascontiguousarray(dataset, dtype=np.float32)
    Q = np.ascontiguousarray(queries, dtype=np.float32)
    lb = np.zeros((len(Q), len(X)), np.float32)
    d = np.zeros((len(Q), len(X)), np.float32)
    _static("lb200_search_screen_probe", _ptr(X), len(X), _ptr(Q), len(Q), X.shape[1], METRIC[metric], _ptr(lb), _ptr(d))
    return lb, d


def search_pscreen_probe(dataset, queries, metric="l2sq", basis=None, k=0):
    """Test hook: (lb, d), both [nq][n] float32 -- the projected screen's lower bound with `basis` (k x dims, any values) or,
    when None, the rows' own basis of k directions (k = 0: the index's choice) -- and the search kernel's fp32 distance."""
    X = np.ascontiguousarray(dataset, dtype=np.float32)
    Q = np.ascontiguousarray(queries, dtype=np.float32)
    lb = np.zeros((len(Q), len(X)), np.float32)
    d = np.zeros((len(Q), len(X)), np.float32)
    P = None if basis is None else np.ascontiguousarray(basis, dtype=np.float32)
    _static("lb200_search_pscreen_probe", _ptr(X), len(X), _ptr(Q), len(Q), X.shape[1], METRIC[metric],
            None if P is None else _ptr(P), len(P) if P is not None else k, _ptr(lb), _ptr(d))
    return lb, d


PQ_PROBE_MODES = {"batch": 0, "kernel": 1, "node": 2}


def pq_probe(index, mode, values=None, nodes=None):
    """Test hook on a built PQ index: (d [count][n], lut [count][nsub][W], v2 [count]) -- the search / build evaluator's
    distance from each value to every stored row, the look-up table it used and |value|^2.  mode "batch" / "kernel": f32
    values with the batch's precomputed tables / tables built in the kernel; "node": stored node ids as values."""
    m = PQ_PROBE_MODES[mode]
    if m == 2:
        vals, nd = None, np.ascontiguousarray(nodes, dtype=np.uint32)
        count = len(nd)
    else:
        vals, nd = np.ascontiguousarray(values, dtype=np.float32), None
        count = len(vals)
    rows, width = C.c_size_t(), C.c_size_t()
    index._call("lb200_pq_probe", m, _ptr(vals), _ptr(nd), count, C.byref(rows), C.byref(width), None, None)
    n, W = rows.value, width.value
    d = np.zeros((count, n), np.float32)
    tab = np.zeros((count, index.num_subvectors * W + 1), np.float32)
    index._call("lb200_pq_probe", m, _ptr(vals), _ptr(nd), count, None, None, _ptr(d), _ptr(tab))
    return d, tab[:, :-1].reshape(count, index.num_subvectors, W), tab[:, -1].copy()


def cast(vectors_f32, quant):
    v = np.ascontiguousarray(vectors_f32, dtype=np.float32)
    d = v.shape[-1]
    flat = v.reshape(-1, d)
    width = {"f32": d, "f16": d, "i8": d, "b1": (d + 7) // 8}[quant]
    out = np.zeros((len(flat), width), NP_OF[quant])
    _static("lb200_cast_batch", _ptr(flat), len(flat), d, SCALAR[quant], _ptr(out))
    return out.reshape(v.shape[:-1] + (width,))


def quantize_pq(codebook, vectors, num_subvectors, compat128=True):
    cb = np.ascontiguousarray(codebook, dtype=np.float32)
    v = np.ascontiguousarray(vectors, dtype=np.float32).reshape(-1, cb.shape[1])
    out = np.zeros((len(v), num_subvectors), np.uint8)
    _static("lb200_quantize_pq", _ptr(cb), cb.shape[1], cb.shape[0], num_subvectors, _ptr(v), len(v), _ptr(out),
            int(compat128))
    return out


def dequantize_pq(codebook, codes):
    cb = np.ascontiguousarray(codebook, dtype=np.float32)
    c = np.ascontiguousarray(codes, dtype=np.uint8)
    c2 = c.reshape(-1, c.shape[-1])
    out = np.zeros((len(c2), cb.shape[1]), np.float32)
    _static("lb200_dequantize_pq", _ptr(cb), cb.shape[1], cb.shape[0], c2.shape[1], _ptr(c2), len(c2), _ptr(out))
    return out


def train_pq(vectors, num_subvectors, num_centroids, metric="l2sq", max_iter=20, seed=1, init_rows=None):
    """k-means codebook float[num_centroids][dims] (product_quantization.c semantics); returns (codebook, rounds)."""
    v = np.ascontiguousarray(vectors, dtype=np.float32)
    cb = np.zeros((num_centroids, v.shape[1]), np.float32)
    ir = None if init_rows is None else np.ascontiguousarray(init_rows, dtype=np.uint32)
    rounds = _static("lb200_train_pq", _ptr(v), len(v), v.shape[1], num_subvectors, num_centroids, METRIC[metric], max_iter, seed,
                     _ptr(ir), _ptr(cb))
    return cb, rounds


def train_pq_device(d_ptr, stride, count, dims, num_subvectors, num_centroids, metric="l2sq", max_iter=20, seed=1):
    cb = np.zeros((num_centroids, dims), np.float32)
    rounds = _static("lb200_train_pq_device", C.c_void_p(d_ptr), stride, count, dims, num_subvectors, num_centroids, METRIC[metric],
                     max_iter, seed, None, _ptr(cb))
    return cb, rounds


def merge_shards_device(d_keys, d_dists, shards, nq, k, d_out_keys, d_out_dists, stream=0):
    _static("lb200_merge_shards_device", C.c_void_p(d_keys), C.c_void_p(d_dists), shards, nq, k, C.c_void_p(d_out_keys),
            C.c_void_p(d_out_dists), C.c_void_p(stream) if stream else None)


def kernel_launches():
    return lib().lb200_kernel_launches()


def device_count():
    return lib().lb200_device_count()
