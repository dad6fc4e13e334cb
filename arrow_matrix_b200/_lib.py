"""ctypes binding of libarrow_b200.so (the C ABI declared in include/arrow_b200.h).

There is no CPU fallback: if the shared library is missing or no CUDA device is present the
calls raise.  Thin object wrappers (`Context`, `Csr`, `Dense`, `RowMap`) keep handles alive and
turn error codes into `ArrowError` with the library's message.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import (POINTER, byref, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_size_t, c_void_p)
from typing import Optional, Sequence, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libarrow_b200.so")

ACCUMULATE = 1
F32, F64 = 0, 1                       # ARROW_F32 / ARROW_F64: element type of dense tiles and CSR values
I32 = 2                               # ARROW_I32: dense tiles of labels / parents (arrow_spmm_sr_witness)
B1 = 3                                # ARROW_B1: bit tiles of the (or, and) semiring; host rows are b1_words(k) uint32 words
BITS = "bits"                         # ``dense_alloc(..., dtype=BITS)``: a bit tile; its host rows are uint32 words
_DTYPE_CODE = {np.dtype(np.float32): F32, np.dtype(np.float64): F64}
_TILE_CODE = {**_DTYPE_CODE, np.dtype(np.int32): I32}
_CODE_TILE = {**{c: dt for dt, c in _TILE_CODE.items()}, B1: BITS}
VARIANT_AUTO, VARIANT_DIRECT, VARIANT_SHFL, VARIANT_TMA, VARIANT_TILES = -1, 0, 1, 2, 3
SR_PLUS_TIMES, SR_MIN_PLUS, SR_MAX_PLUS, SR_OR_AND = 0, 1, 2, 3   # ARROW_SR_*: the semiring of arrow_spmm_sr / arrow_gather_rows_sr
SR_MAX_MIN, SR_MIN_MAX = 4, 5                                       # the bottleneck semirings: widest / minimax paths
SEMIRINGS = {"plus_times": SR_PLUS_TIMES, "min_plus": SR_MIN_PLUS, "max_plus": SR_MAX_PLUS, "or_and": SR_OR_AND,
             "max_min": SR_MAX_MIN, "min_max": SR_MIN_MAX}
IPC_HANDLE_BYTES = 80

EXPORTS = [
    "arrow_b200_abi_version", "arrow_ctx_create", "arrow_ctx_destroy", "arrow_last_error", "arrow_sync",
    "arrow_device_info", "arrow_set_tuning", "arrow_set_option",
    "arrow_csr_upload", "arrow_csr_free", "arrow_csr_info", "arrow_csr_remap_columns",
    "arrow_map_upload", "arrow_map_free", "arrow_map_compose", "arrow_map_invert", "arrow_map_d2h",
    "arrow_dense_alloc", "arrow_dense_free", "arrow_dense_fill", "arrow_dense_h2d", "arrow_dense_d2h",
    "arrow_dense_copy", "arrow_dense_ptr", "arrow_dense_wrap", "arrow_host_alloc", "arrow_host_free",
    "arrow_dense_h2d_lane", "arrow_dense_d2h_lane", "arrow_lane_wait", "arrow_lane_sync", "arrow_set_lane",
    "arrow_event_record", "arrow_event_wait",
    "arrow_spmm", "arrow_spmm_add", "arrow_gather_rows", "arrow_gather_rows_multi",
    "arrow_ipc_export", "arrow_ipc_import", "arrow_peer_barrier",
    "arrow_timer_start", "arrow_timer_stop", "arrow_timer_elapsed_ms", "arrow_launch_count", "arrow_l2_flush",
    "arrow_ptrtable_upload", "arrow_ptrtable_free", "arrow_spmm_ex", "arrow_push_rows", "arrow_reduce_rows",
    "arrow_graph_begin", "arrow_graph_end", "arrow_graph_launch", "arrow_graph_free",
    "arrow_host_alloc_numa", "arrow_bind_thread_to_device_numa", "arrow_preload_kernels",
    "arrow_csr_upload_f64", "arrow_dense_alloc_dtype", "arrow_dense_dtype",
    "arrow_spmm_sr", "arrow_gather_rows_sr", "arrow_dense_count_diff",
    "arrow_spmm_sr_witness", "arrow_tile_rows", "arrow_tile_rows_rule", "arrow_bits_mark_new",
    "arrow_adj_build", "arrow_adj_free", "arrow_adj_info", "arrow_adj_d2h", "arrow_bits_mark_frontier",
    "arrow_bits_push_frontier", "arrow_adj_build_weighted", "arrow_adj_values_d2h", "arrow_sr_mark_frontier",
    "arrow_sr_push_frontier", "arrow_adj_build_in", "arrow_bits_parents", "arrow_bits_path_counts",
    "arrow_adj_keep_record", "arrow_bits_dependencies", "arrow_bits_fill_f64", "arrow_dense_row_sum",
    "arrow_adj_build_loopfree", "arrow_wpaths_counts", "arrow_wpaths_dependencies",
    "arrow_sr_mark_frontier_steps", "arrow_sr_tree_parents", "arrow_dense_count_diff_bits",
    "arrow_out_weights", "arrow_csr_scale_columns", "arrow_pagerank_restart", "arrow_pagerank_update",
    "arrow_connected_components",
]
ABI_VERSION = 15       # ARROW_ABI_VERSION of include/arrow_b200.h this binding was written against


class ArrowError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"libarrow_b200 error {code}: {message}")
        self.code = code


_lib = None


def load_library(build_if_missing: bool = True) -> ctypes.CDLL:
    """dlopen the in-tree library.  A missing or stale library (older than its sources) is rebuilt first when nvcc
    is available -- under a file lock and through a temporary file, so that the ranks of one ``torchrun`` never
    dlopen a half-written file (``build.build``).  A library whose ABI version differs from this binding is refused."""
    global _lib
    if _lib is not None:
        return _lib
    from . import build as _build
    if build_if_missing and _build.needs_build() and _build.can_build():
        _build.build()
    if not os.path.exists(LIB_PATH):
        raise FileNotFoundError(f"{LIB_PATH} not built; run `python -m arrow_matrix_b200.build` (needs nvcc)")
    lib = ctypes.CDLL(LIB_PATH)
    lib.arrow_b200_abi_version.restype = c_int
    found = lib.arrow_b200_abi_version()
    if found != ABI_VERSION:
        raise ImportError(f"{LIB_PATH} exports ABI version {found}, this binding needs {ABI_VERSION}: rebuild it "
                          f"(`python -m arrow_matrix_b200.build --force`)")
    P = c_void_p
    I, I64 = c_int, c_int64
    pI, pI64 = POINTER(c_int), POINTER(c_int64)
    sig = {
        "arrow_b200_abi_version": (c_int, []),
        "arrow_ctx_create": (c_int, [I, P, POINTER(P)]),
        "arrow_ctx_destroy": (None, [P]),
        "arrow_last_error": (c_char_p, [P]),
        "arrow_sync": (c_int, [P]),
        "arrow_device_info": (c_int, [P, pI, pI64, pI64]),
        "arrow_set_tuning": (c_int, [P, I, I]),
        "arrow_set_option": (c_int, [P, I, I]),
        "arrow_csr_upload": (c_int, [P, I64, I64, I64, P, I, P, I, P, pI]),
        "arrow_csr_free": (c_int, [P, I]),
        "arrow_csr_info": (c_int, [P, I, pI64, pI64, pI64, pI64, pI64]),
        "arrow_csr_remap_columns": (c_int, [P, I, I, I64, pI]),
        "arrow_map_upload": (c_int, [P, P, I64, I64, pI]),
        "arrow_map_free": (c_int, [P, I]),
        "arrow_map_compose": (c_int, [P, I, I, pI]),
        "arrow_map_invert": (c_int, [P, I, I64, pI]),
        "arrow_map_d2h": (c_int, [P, I, P, I64]),
        "arrow_dense_alloc": (c_int, [P, I64, I, pI]),
        "arrow_dense_free": (c_int, [P, I]),
        "arrow_dense_fill": (c_int, [P, I, c_float]),
        "arrow_dense_h2d": (c_int, [P, I, I64, I64, P]),
        "arrow_dense_d2h": (c_int, [P, I, I64, I64, P]),
        "arrow_dense_copy": (c_int, [P, I, I64, I, I64, I64]),
        "arrow_dense_ptr": (c_int, [P, I, POINTER(P), pI64, pI]),
        "arrow_dense_wrap": (c_int, [P, P, I64, I, pI]),
        "arrow_dense_h2d_lane": (c_int, [P, I, I, I64, I64, P]),
        "arrow_dense_d2h_lane": (c_int, [P, I, I, I64, I64, P]),
        "arrow_lane_wait": (c_int, [P, I, I]),
        "arrow_lane_sync": (c_int, [P, I]),
        "arrow_set_lane": (c_int, [P, I]),
        "arrow_event_record": (c_int, [P, I, I]),
        "arrow_event_wait": (c_int, [P, I, I]),
        "arrow_host_alloc": (c_int, [c_size_t, POINTER(P)]),
        "arrow_host_free": (c_int, [P]),
        "arrow_spmm": (c_int, [P, I, I, I, I, I, I]),
        "arrow_spmm_add": (c_int, [P, I, I, I, I, I, I]),
        "arrow_gather_rows": (c_int, [P, I, I, I, I]),
        "arrow_gather_rows_multi": (c_int, [P, I, pI, pI64, I, I, I]),
        "arrow_ipc_export": (c_int, [P, I, P]),
        "arrow_ipc_import": (c_int, [P, P, I64, I, pI]),
        "arrow_peer_barrier": (c_int, [P, pI, I, I]),
        "arrow_timer_start": (c_int, [P, I]),
        "arrow_timer_stop": (c_int, [P, I]),
        "arrow_timer_elapsed_ms": (c_int, [P, I, POINTER(c_float)]),
        "arrow_launch_count": (c_int, [P, pI64]),
        "arrow_l2_flush": (c_int, [P]),
        "arrow_ptrtable_upload": (c_int, [P, pI, I, P, P, I64, pI]),
        "arrow_ptrtable_free": (c_int, [P, I]),
        "arrow_spmm_ex": (c_int, [P, I, I, I, I64, I, I, I, I, I]),
        "arrow_push_rows": (c_int, [P, pI, pI64, I, I, I]),
        "arrow_reduce_rows": (c_int, [P, I, I, pI, I, I64]),
        "arrow_graph_begin": (c_int, [P]),
        "arrow_graph_end": (c_int, [P, pI]),
        "arrow_graph_launch": (c_int, [P, I]),
        "arrow_graph_free": (c_int, [P, I]),
        "arrow_host_alloc_numa": (c_int, [c_size_t, I, POINTER(P)]),
        "arrow_bind_thread_to_device_numa": (c_int, [I, pI, pI]),
        "arrow_preload_kernels": (c_int, [P, I]),
        "arrow_csr_upload_f64": (c_int, [P, I64, I64, I64, P, I, P, I, P, pI]),
        "arrow_dense_alloc_dtype": (c_int, [P, I64, I, I, pI]),
        "arrow_dense_dtype": (c_int, [P, I, pI]),
        "arrow_spmm_sr": (c_int, [P, I, I, I, I, I, I]),
        "arrow_gather_rows_sr": (c_int, [P, I, I, I, I]),
        "arrow_dense_count_diff": (c_int, [P, I, I, pI64]),
        "arrow_spmm_sr_witness": (c_int, [P, I, I, I, I, I, I, I, I, I, I]),
        "arrow_tile_rows": (c_int, [P, I, I, pI]),
        "arrow_tile_rows_rule": (c_int, [I, I, I64, I, I]),
        "arrow_bits_mark_new": (c_int, [P, I, I, I, I, pI64]),
        "arrow_adj_build": (c_int, [P, I, pI, pI, I64, pI]),
        "arrow_adj_free": (c_int, [P, I]),
        "arrow_adj_info": (c_int, [P, I, pI64, pI64]),
        "arrow_adj_d2h": (c_int, [P, I, P, P]),
        "arrow_bits_mark_frontier": (c_int, [P, I, I, I, I, I, pI64, pI64, pI64]),
        "arrow_bits_push_frontier": (c_int, [P, I, I, I]),
        "arrow_adj_build_weighted": (c_int, [P, I, pI, pI, I64, pI]),
        "arrow_adj_values_d2h": (c_int, [P, I, P]),
        "arrow_sr_mark_frontier": (c_int, [P, I, I, I, pI64, pI64, pI64]),
        "arrow_sr_push_frontier": (c_int, [P, I, I, I, I]),
        "arrow_adj_build_in": (c_int, [P, I, pI, pI, I64, pI]),
        "arrow_bits_parents": (c_int, [P, I, I, I, I, I, pI64]),
        "arrow_bits_path_counts": (c_int, [P, I, I, I, I, I, pI64]),
        "arrow_adj_keep_record": (c_int, [P, I, I]),
        "arrow_bits_dependencies": (c_int, [P, I, I, I, I, I, pI64]),
        "arrow_bits_fill_f64": (c_int, [P, I, I, I, c_double]),
        "arrow_dense_row_sum": (c_int, [P, I, I]),
        "arrow_adj_build_loopfree": (c_int, [P, I, pI, pI, I64, I, pI]),
        "arrow_wpaths_counts": (c_int, [P, I, I, I, I, I, I, pI64, pI64]),
        "arrow_wpaths_dependencies": (c_int, [P, I, I, I, I, I, I, pI64]),
        "arrow_sr_mark_frontier_steps": (c_int, [P, I, I, I, I, I, pI64, pI64, pI64]),
        "arrow_sr_tree_parents": (c_int, [P, I, I, I, I, I, pI64]),
        "arrow_dense_count_diff_bits": (c_int, [P, I, I, pI64]),
        "arrow_out_weights": (c_int, [P, I, pI, pI, I64, I, I, pI64, pI64, pI64]),
        "arrow_csr_scale_columns": (c_int, [P, I, I, I, pI]),
        "arrow_pagerank_restart": (c_int, [P, I, I, I, I, I, POINTER(c_double), pI64, pI64]),
        "arrow_pagerank_update": (c_int, [P, I, I, I, I, I, I, c_double, POINTER(c_double)]),
        "arrow_connected_components": (c_int, [P, I, pI, pI, I64, I, I, pI64]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)          # AttributeError here = the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def _ptr(a: Optional[np.ndarray]) -> c_void_p:
    return c_void_p(None) if a is None else c_void_p(a.ctypes.data)


def b1_words(k: int) -> int:
    """uint32 words per row of a bit tile of ``k`` columns: one bit per column; one word for k <= 32, else padded to a
    multiple of 4 words"""
    return 1 if int(k) <= 32 else ((int(k) + 31) // 32 + 3) & ~3


def pack_bits(X: np.ndarray) -> np.ndarray:
    """bool (or any: non-zero is true) [n x k] -> uint32 [n x b1_words(k)]: column c is bit c % 32 of word c // 32,
    padding bits are zero"""
    X = np.asarray(X)
    if X.ndim != 2:
        raise ValueError(f"expected a 2-d array, got shape {X.shape}")
    n, k = X.shape
    by = np.packbits(X != 0, axis=1, bitorder="little")
    out = np.zeros((n, b1_words(k) * 4), dtype=np.uint8)
    out[:, :by.shape[1]] = by
    return out.view("<u4").astype(np.uint32, copy=False)


def unpack_bits(words: np.ndarray, k: int) -> np.ndarray:
    """uint32 [n x w] words -> bool [n x k] (the inverse of ``pack_bits``; padding bits are ignored)"""
    words = np.ascontiguousarray(words, dtype="<u4")
    if words.ndim != 2 or words.shape[1] * 32 < k:
        raise ValueError(f"{words.shape} words cannot hold {k} columns")
    return np.unpackbits(words.view(np.uint8), axis=1, count=int(k), bitorder="little").astype(bool)


def element_type(dtype) -> np.dtype:
    """``np.float32`` or ``np.float64`` (the element types the library computes in); anything else raises."""
    dt = np.dtype(dtype)
    if dt not in _DTYPE_CODE:
        raise ValueError(f"unsupported element type {dt}: the library computes in float32 or float64")
    return dt


class PinnedArray:
    """Page-locked host staging buffer exposed as a numpy array (freed on `close()`/GC)."""

    def __init__(self, shape, dtype=np.float32, numa_device: Optional[int] = None):
        """``numa_device`` given: the buffer is placed on the NUMA node that GPU hangs off (arrow_host_alloc_numa)."""
        lib = load_library()
        self.shape = tuple(int(s) for s in np.atleast_1d(shape))
        self.dtype = np.dtype(dtype)
        nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        p = c_void_p()
        if numa_device is None:
            rc = lib.arrow_host_alloc(c_size_t(max(nbytes, 16)), byref(p))
        else:
            rc = lib.arrow_host_alloc_numa(c_size_t(max(nbytes, 16)), int(numa_device), byref(p))
        if rc != 0:
            raise ArrowError(rc, (lib.arrow_last_error(None) or b"").decode())
        self._p = p
        buf = (ctypes.c_char * max(nbytes, 16)).from_address(p.value)
        self.array = np.frombuffer(buf, dtype=self.dtype, count=int(np.prod(self.shape))).reshape(self.shape)

    def close(self):
        if getattr(self, "_p", None) is not None and self._p.value:
            self.array = None
            load_library().arrow_host_free(self._p)
            self._p = c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def bind_thread_to_device_numa(device: int):
    """Pin the calling thread to the CPUs of the NUMA node ``device`` hangs off; returns ``(node, n_cpus)``
    (``(-1, 0)`` when the topology is unknown and nothing was changed)."""
    lib = load_library()
    node, n = c_int(-1), c_int(0)
    lib.arrow_bind_thread_to_device_numa(int(device), byref(node), byref(n))
    return node.value, n.value


class Context:
    """One device context = one stream = one host thread (arrow_b200.h)."""

    def __init__(self, device: int = 0, stream: Optional[int] = None):
        self.lib = load_library()
        self._h = c_void_p()
        rc = self.lib.arrow_ctx_create(int(device), c_void_p(stream) if stream else c_void_p(None), byref(self._h))
        if rc != 0:
            raise ArrowError(rc, (self.lib.arrow_last_error(None) or b"").decode())
        self.device = int(device)

    # -- plumbing ---------------------------------------------------------------------------
    def _check(self, rc: int):
        if rc != 0:
            raise ArrowError(rc, (self.lib.arrow_last_error(self._h) or b"").decode())

    def close(self):
        if self._h:
            self.lib.arrow_ctx_destroy(self._h)
            self._h = c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sync(self):
        self._check(self.lib.arrow_sync(self._h))

    def preload_kernels(self, k: int):
        """load every kernel a step with ``k`` feature columns can launch, before any peer barrier is in flight"""
        self._check(self.lib.arrow_preload_kernels(self._h, int(k)))

    def device_info(self):
        sm, fr, tot = c_int(), c_int64(), c_int64()
        self._check(self.lib.arrow_device_info(self._h, byref(sm), byref(fr), byref(tot)))
        return sm.value, fr.value, tot.value

    def set_tuning(self, long_row_threshold: int, long_row_segment: int):
        self._check(self.lib.arrow_set_tuning(self._h, int(long_row_threshold), int(long_row_segment)))

    OPT_L2_HINTS_PLAIN, OPT_L2_HINTS_FUSED, OPT_BIG_TILES, OPT_SPMM_CTAS_PER_SM, OPT_PREFETCH = 1, 2, 3, 4, 5
    OPT_ROWS_PER_GROUP, OPT_SPMM_SM_LIMIT, OPT_PUSH_CTAS, OPT_BARRIER_TIMEOUT_MS, OPT_SMEM_CARVEOUT = 6, 7, 8, 9, 10
    OPT_FORCE_PREDICATED, OPT_TILE_KERNEL, OPT_PUSH_INTERLEAVE, OPT_TILE_ROWS = 11, 12, 13, 14

    def set_option(self, option: int, value: int):
        self._check(self.lib.arrow_set_option(self._h, int(option), int(value)))

    def tile_rows(self, k: int, dtype=np.float32) -> int:
        """rows per CSR tile of this context's tile-kernel launches at feature width ``k`` (``arrow_tile_rows``)"""
        rows = c_int()
        self._check(self.lib.arrow_tile_rows(self._h, int(k), _DTYPE_CODE[element_type(dtype)], byref(rows)))
        return rows.value

    # -- sparse -----------------------------------------------------------------------------
    def csr_upload(self, n_rows: int, n_cols: int, indptr: np.ndarray, indices: np.ndarray,
                   data: Optional[np.ndarray], dtype=np.float32) -> "Csr":
        """`indptr` may be a slice of a larger row pointer; indices/data are the matching slices.  ``dtype`` is the
        precision of the block's values and of every launch on it (float32 or float64)."""
        dtype = element_type(dtype)
        indptr = np.ascontiguousarray(indptr)
        if indptr.dtype not in (np.int32, np.int64):
            indptr = indptr.astype(np.int64)
        nnz = int(indptr[-1] - indptr[0]) if indptr.size else 0
        indices = np.ascontiguousarray(indices)
        if indices.dtype not in (np.int32, np.int64):
            indices = indices.astype(np.int64)
        if indices.size != nnz:
            raise ValueError(f"indices has {indices.size} entries, indptr spans {nnz}")
        if data is not None:
            data = np.ascontiguousarray(data, dtype=dtype)
            if data.size != nnz:
                raise ValueError(f"data has {data.size} entries, indptr spans {nnz}")
        upload = self.lib.arrow_csr_upload_f64 if dtype == np.float64 else self.lib.arrow_csr_upload
        h = c_int()
        self._check(upload(self._h, int(n_rows), int(n_cols), nnz, _ptr(indptr), indptr.dtype.itemsize,
                           _ptr(indices), indices.dtype.itemsize, _ptr(data), byref(h)))
        return Csr(self, h.value, int(n_rows), int(n_cols), nnz, dtype)

    def csr_from_scipy(self, A) -> "Csr":
        from scipy import sparse
        A = sparse.csr_matrix(A)
        return self.csr_upload(A.shape[0], A.shape[1], A.indptr, A.indices, A.data.astype(np.float32, copy=False))

    # -- maps -------------------------------------------------------------------------------
    def map_upload(self, m: np.ndarray, limit: int) -> "RowMap":
        m = np.ascontiguousarray(m, dtype=np.int64)
        h = c_int()
        self._check(self.lib.arrow_map_upload(self._h, _ptr(m), m.size, int(limit), byref(h)))
        return RowMap(self, h.value, m.size, int(limit))

    # -- dense ------------------------------------------------------------------------------
    def dense_alloc(self, rows: int, k: int, dtype=np.float32) -> "Dense":
        """a zero-filled tile of float32 / float64 features, of int32 labels (``arrow_spmm_sr_witness``) or, with
        ``dtype=BITS``, of ``k`` bit columns (``ARROW_B1``: host rows of ``b1_words(k)`` uint32 words; ``np.uint32``
        itself is not a tile type)"""
        if isinstance(dtype, str) and dtype == BITS:
            h = c_int()
            self._check(self.lib.arrow_dense_alloc_dtype(self._h, int(rows), int(k), B1, byref(h)))
            return Dense(self, h.value, int(rows), int(k), owned=True, dtype=BITS)
        dtype = np.dtype(np.int32) if np.dtype(dtype) == np.int32 else element_type(dtype)
        h = c_int()
        if dtype == np.float32:
            self._check(self.lib.arrow_dense_alloc(self._h, int(rows), int(k), byref(h)))
        else:
            self._check(self.lib.arrow_dense_alloc_dtype(self._h, int(rows), int(k), _TILE_CODE[dtype], byref(h)))
        return Dense(self, h.value, int(rows), int(k), owned=True, dtype=dtype)

    def dense_wrap(self, device_ptr: int, rows: int, k: int) -> "Dense":
        h = c_int()
        self._check(self.lib.arrow_dense_wrap(self._h, c_void_p(device_ptr), int(rows), int(k), byref(h)))
        return Dense(self, h.value, int(rows), int(k), owned=False)

    def dense_from_host(self, X: np.ndarray, dtype=np.float32) -> "Dense":
        X = np.ascontiguousarray(X, dtype=element_type(dtype))
        d = self.dense_alloc(X.shape[0], X.shape[1], X.dtype)
        d.h2d(X)
        self.sync()
        return d

    def ipc_import(self, handle: bytes, rows: int, k: int) -> "Dense":
        assert len(handle) == IPC_HANDLE_BYTES
        buf = ctypes.create_string_buffer(handle, IPC_HANDLE_BYTES)
        h = c_int()
        self._check(self.lib.arrow_ipc_import(self._h, buf, int(rows), int(k), byref(h)))
        return Dense(self, h.value, int(rows), int(k), owned=False)

    # -- hot path ---------------------------------------------------------------------------
    def spmm(self, A: "Csr", X: "Dense", C: "Dense", rowmap: Optional["RowMap"] = None,
             accumulate: bool = False, variant: int = VARIANT_AUTO):
        self._check(self.lib.arrow_spmm(self._h, A.h, X.h, C.h, rowmap.h if rowmap is not None else -1,
                                        ACCUMULATE if accumulate else 0, int(variant)))

    def spmm_add(self, A: "Csr", X: "Dense", C: "Dense", add: "Dense", add_map: "RowMap", variant: int = VARIANT_AUTO):
        """C[r] = (A X)[r] + add[add_map[r]] (where add_map[r] >= 0)"""
        self._check(self.lib.arrow_spmm_add(self._h, A.h, X.h, C.h, add.h, add_map.h, int(variant)))

    def spmm_sr(self, A: "Csr", X: "Dense", C: "Dense", add: Optional["Dense"] = None,
                add_map: Optional["RowMap"] = None, semiring: int = SR_PLUS_TIMES):
        """C[r] = (⊕_p A[r,p] ⊗ X[col_p]) ⊕ add[add_map[r]] in the semiring ``SR_*`` (``arrow_spmm_sr``)"""
        self._check(self.lib.arrow_spmm_sr(self._h, A.h, X.h, C.h, add.h if add is not None else -1,
                                           add_map.h if add_map is not None else -1, int(semiring)))

    def spmm_sr_witness(self, A: "Csr", X: "Dense", labels: "Dense", values: Optional["Dense"] = None,
                        add_values: Optional["Dense"] = None, add_labels: Optional["Dense"] = None,
                        add_map: Optional["RowMap"] = None, dist: Optional["Dense"] = None,
                        row_labels: Optional["RowMap"] = None, semiring: int = SR_MIN_PLUS):
        """The product of ``spmm_sr`` over (value, label) pairs (``arrow_spmm_sr_witness``): the lexicographic ⊕ of the
        candidates (fl(A[r,p] + X[c]), c) with c != row_labels[r] (the row index when ``row_labels`` is None), ⊕ the
        addend pair at add_map[r].  Without ``dist`` the pair goes to ``values`` / ``labels``; with it ``labels``
        receives the parents (the witness label where dist[r] is not the ⊕ identity and equals the witness value, else
        -1) and ``values``, when given, the witness values."""
        h = lambda o: o.h if o is not None else -1
        self._check(self.lib.arrow_spmm_sr_witness(self._h, A.h, X.h, h(row_labels), h(values), labels.h, h(add_values),
                                                   h(add_labels), h(add_map), h(dist), int(semiring)))

    def spmm_ex(self, A: "Csr", X: "Dense", C: Optional["Dense"] = None, X2: Optional["Dense"] = None, x_split: int = 0,
                out_table: Optional["PtrTable"] = None, add: Optional["Dense"] = None, add_map: Optional["RowMap"] = None,
                variant: int = VARIANT_AUTO):
        """Generalised product (``arrow_spmm_ex``): two-part X operand, row-pointer epilogue, gather-add."""
        self._check(self.lib.arrow_spmm_ex(self._h, A.h, X.h, X2.h if X2 is not None else -1, int(x_split),
                                           C.h if C is not None else -1, out_table.h if out_table is not None else -1,
                                           add.h if add is not None else -1, add_map.h if add_map is not None else -1,
                                           int(variant)))

    def ptrtable_upload(self, tiles: Sequence["Dense"], which: np.ndarray, row: np.ndarray) -> "PtrTable":
        which = np.ascontiguousarray(which, dtype=np.int32)
        row = np.ascontiguousarray(row, dtype=np.int64)
        assert which.shape == row.shape and which.ndim == 1
        n = len(tiles)
        hs = (c_int * n)(*[t.h for t in tiles])
        h = c_int()
        self._check(self.lib.arrow_ptrtable_upload(self._h, hs, n, _ptr(which), _ptr(row), which.size, byref(h)))
        return PtrTable(self, h.value, which.size)

    def push_rows(self, dsts: Sequence[Optional["Dense"]], item_bounds: Sequence[int], src: "Dense", m: "RowMap"):
        n = len(dsts)
        hs = (c_int * n)(*[(d.h if d is not None else -1) for d in dsts])
        bd = (c_int64 * (n + 1))(*[int(b) for b in item_bounds])
        self._check(self.lib.arrow_push_rows(self._h, hs, bd, n, src.h, m.h))

    def reduce_rows(self, srcs: Sequence["Dense"], rows: int, dst: Optional["Dense"] = None,
                    out_table: Optional["PtrTable"] = None):
        n = len(srcs)
        hs = (c_int * n)(*[s.h for s in srcs])
        self._check(self.lib.arrow_reduce_rows(self._h, dst.h if dst is not None else -1,
                                               out_table.h if out_table is not None else -1, hs, n, int(rows)))

    # -- graphs -----------------------------------------------------------------------------
    def graph_begin(self):
        self._check(self.lib.arrow_graph_begin(self._h))

    def graph_end(self) -> int:
        h = c_int()
        self._check(self.lib.arrow_graph_end(self._h, byref(h)))
        return h.value

    def graph_launch(self, g: int):
        self._check(self.lib.arrow_graph_launch(self._h, int(g)))

    def graph_free(self, g: int):
        self._check(self.lib.arrow_graph_free(self._h, int(g)))

    def gather_rows(self, dst: "Dense", src: "Dense", m: "RowMap", accumulate: bool = False):
        self._check(self.lib.arrow_gather_rows(self._h, dst.h, src.h, m.h, ACCUMULATE if accumulate else 0))

    def gather_rows_sr(self, dst: "Dense", src: "Dense", m: "RowMap", semiring: int = SR_PLUS_TIMES):
        """dst[r] = dst[r] ⊕ src[m[r]] where m[r] >= 0 (``arrow_gather_rows_sr``)"""
        self._check(self.lib.arrow_gather_rows_sr(self._h, dst.h, src.h, m.h, int(semiring)))

    def bits_mark_new(self, new: "Dense", old: "Dense", dist: "Dense", level: int) -> int:
        """dist[r, c] = level where the bit (r, c) is set in ``new`` and clear in ``old`` (``arrow_bits_mark_new``); returns
        the number of such bits; synchronises"""
        n = c_int64()
        self._check(self.lib.arrow_bits_mark_new(self._h, new.h, old.h, dist.h, int(level), byref(n)))
        return int(n.value)

    def adj_build(self, parts: Sequence[tuple], n_vertices: int, weighted: bool = False,
                  direction: str = "out") -> "Adjacency":
        """The push adjacency of a BFS (``arrow_adj_build``): ``parts`` is a sequence of ``(Csr, RowMap or None)``; entry
        (r, c) of a block gives the edge map(c) -> map(r) (None: the identity), edges with an end at -1 and u == v are
        dropped.  ``weighted`` (``arrow_adj_build_weighted``): every edge carries its entry's fp32 value and the edges
        u == v are kept -- the adjacency of the min-plus / max-plus push.  ``direction="in"`` (``arrow_adj_build_in``):
        the same edges stored by destination, row v listing its sources u in ascending order -- the adjacency of
        ``bits_parents``.  Synchronises."""
        if direction not in ("out", "in"):
            raise ValueError(f"direction must be 'out' or 'in', got {direction!r}")
        if direction == "in" and weighted:
            raise ValueError("the in-adjacency carries no weights")
        n = len(parts)
        csrs = (c_int * max(n, 1))(*[A.h for A, _ in parts])
        maps = (c_int * max(n, 1))(*[m.h if m is not None else -1 for _, m in parts])
        h = c_int()
        build = self.lib.arrow_adj_build_weighted if weighted else \
            self.lib.arrow_adj_build_in if direction == "in" else self.lib.arrow_adj_build
        self._check(build(self._h, n, csrs, maps, int(n_vertices), byref(h)))
        return Adjacency(self, h.value)

    def bits_mark_frontier(self, adj: "Adjacency", new: "Dense", old: "Dense", dist: "Dense", level: int):
        """``bits_mark_new`` that also records in ``adj`` the rows with a fresh bit (``arrow_bits_mark_frontier``); returns
        (fresh bits, frontier rows, frontier edges); synchronises"""
        n, rows, edges = c_int64(), c_int64(), c_int64()
        self._check(self.lib.arrow_bits_mark_frontier(self._h, adj.h, new.h, old.h, dist.h, int(level), byref(n),
                                                      byref(rows), byref(edges)))
        return int(n.value), int(rows.value), int(edges.value)

    def bits_push_frontier(self, adj: "Adjacency", x: "Dense", out: "Dense"):
        """out = x, then out[v] |= x[u] along the adjacency's edges of the recorded frontier rows u
        (``arrow_bits_push_frontier``); ``x`` must be the tile of the last ``bits_mark_frontier`` on ``adj``"""
        self._check(self.lib.arrow_bits_push_frontier(self._h, adj.h, x.h, out.h))

    def bits_parents(self, in_adj: "Adjacency", adj: "Adjacency", new: "Dense", old: "Dense", parent: "Dense",
                     count: bool = False) -> Optional[int]:
        """parent[v, s] = the smallest u of ``in_adj``'s row v whose bit s is set in ``old``, for every bit (v, s) set in
        ``new`` and clear in ``old`` of the rows recorded in ``adj`` by the last ``bits_mark_frontier(adj, new, old, ...)``
        (``arrow_bits_parents``); other elements of the int32 tile ``parent`` are left alone.  With ``count`` returns the
        in-edges gathered (synchronises), else None (stream-ordered)."""
        n = c_int64()
        self._check(self.lib.arrow_bits_parents(self._h, in_adj.h, adj.h, new.h, old.h, parent.h,
                                                byref(n) if count else None))
        return int(n.value) if count else None

    def bits_path_counts(self, in_adj: "Adjacency", adj: "Adjacency", new: "Dense", old: "Dense", sigma: "Dense",
                         count: bool = False) -> Optional[int]:
        """sigma[v, s] = the sum of sigma[u, s] over the distinct u of ``in_adj``'s row v whose bit s is set in ``old``,
        for every bit (v, s) set in ``new`` and clear in ``old`` of the rows recorded in ``adj`` by the last
        ``bits_mark_frontier(adj, new, old, ...)`` (``arrow_bits_path_counts``); other elements of the float64 tile
        ``sigma`` are left alone.  With ``count`` returns the in-list entries read (synchronises), else None."""
        n = c_int64()
        self._check(self.lib.arrow_bits_path_counts(self._h, in_adj.h, adj.h, new.h, old.h, sigma.h,
                                                    byref(n) if count else None))
        return int(n.value) if count else None

    def adj_keep_record(self, adj: "Adjacency", level: int):
        """copies ``adj``'s frontier record into its history as ``level`` (0 restarts it; otherwise the next level)
        (``arrow_adj_keep_record``)"""
        self._check(self.lib.arrow_adj_keep_record(self._h, adj.h, int(level)))

    def bits_dependencies(self, adj: "Adjacency", level: int, dist: "Dense", sigma: "Dense", delta: "Dense",
                          count: bool = False) -> Optional[int]:
        """delta[u, s] = sigma[u, s] * sum of (1 + delta[w, s]) / sigma[w, s] over the distinct w of ``adj``'s row u
        with dist[w, s] == level + 1, for the rows u of the history's ``level`` and the columns with dist[u, s] == level
        (``arrow_bits_dependencies``).  With ``count`` returns the out-list entries read (synchronises), else None."""
        n = c_int64()
        self._check(self.lib.arrow_bits_dependencies(self._h, adj.h, int(level), dist.h, sigma.h, delta.h,
                                                     byref(n) if count else None))
        return int(n.value) if count else None

    def bits_fill_f64(self, new: "Dense", old: "Dense", out: "Dense", value: float):
        """out[r, s] = value for every bit set in ``new`` and clear in ``old`` (float64 ``out``; ``arrow_bits_fill_f64``)"""
        self._check(self.lib.arrow_bits_fill_f64(self._h, new.h, old.h, out.h, float(value)))

    def row_sum(self, x: "Dense", out: "Dense"):
        """out[r, 0] = x[r, 0] + ... + x[r, k - 1], left to right (float64 tiles; ``arrow_dense_row_sum``)"""
        self._check(self.lib.arrow_dense_row_sum(self._h, x.h, out.h))

    def adj_build_loopfree(self, parts: Sequence[tuple], n_vertices: int, direction: str = "out") -> "Adjacency":
        """The weighted adjacency of ``adj_build`` without the edges u == v (``arrow_adj_build_loopfree``): the lists of
        ``adj_build(parts, n)`` (``direction="out"``) or ``adj_build(parts, n, direction="in")``, every entry carrying its
        fp32 weight -- the lists of the weighted path passes.  Synchronises."""
        if direction not in ("out", "in"):
            raise ValueError(f"direction must be 'out' or 'in', got {direction!r}")
        n = len(parts)
        csrs = (c_int * max(n, 1))(*[A.h for A, _ in parts])
        maps = (c_int * max(n, 1))(*[m.h if m is not None else -1 for _, m in parts])
        h = c_int()
        self._check(self.lib.arrow_adj_build_loopfree(self._h, n, csrs, maps, int(n_vertices), int(direction == "in"),
                                                      byref(h)))
        return Adjacency(self, h.value)

    def wpaths_counts(self, in_adj: "Adjacency", out_adj: "Adjacency", x0: "Dense", dist: "Dense", state: "Dense",
                      sigma: "Dense", count: bool = False) -> Tuple[int, Optional[int]]:
        """sigma[v, s] = [v in S_s] + the sum of sigma[u, s] over the distinct tight pairs u -> v of the fixed point
        ``dist`` started from ``x0``, by Kahn rounds over the tight pairs; ``state`` (int32) receives -(depth + 2), -1
        where ``dist`` is not finite, and ``out_adj`` keeps every round's rows (``arrow_wpaths_counts``).  Returns (rounds,
        list entries read with ``count``, else None); synchronises."""
        rounds, n = c_int64(), c_int64()
        self._check(self.lib.arrow_wpaths_counts(self._h, in_adj.h, out_adj.h, x0.h, dist.h, state.h, sigma.h, byref(rounds),
                                                 byref(n) if count else None))
        return int(rounds.value), (int(n.value) if count else None)

    def wpaths_dependencies(self, out_adj: "Adjacency", x0: "Dense", dist: "Dense", state: "Dense", sigma: "Dense",
                            delta: "Dense", count: bool = False) -> Optional[int]:
        """delta[v, s] = 0 for v in S_s, else sigma[v, s] * the sum of fl((1 + delta[w, s]) / sigma[w, s]) over the
        distinct tight pairs v -> w, over the rounds of the last ``wpaths_counts`` (``arrow_wpaths_dependencies``).  With
        ``count`` returns the out-list entries read (synchronises), else None."""
        n = c_int64()
        self._check(self.lib.arrow_wpaths_dependencies(self._h, out_adj.h, x0.h, dist.h, state.h, sigma.h, delta.h,
                                                       byref(n) if count else None))
        return int(n.value) if count else None

    def sr_mark_frontier(self, adj: "Adjacency", new: "Dense", old: "Dense"):
        """(rows changed by value -- ``count_diff``'s figure --, frontier rows, frontier edges) of two fp32 tiles; records
        in ``adj`` the rows that differ in bits (``arrow_sr_mark_frontier``); synchronises"""
        n, rows, edges = c_int64(), c_int64(), c_int64()
        self._check(self.lib.arrow_sr_mark_frontier(self._h, adj.h, new.h, old.h, byref(n), byref(rows), byref(edges)))
        return int(n.value), int(rows.value), int(edges.value)

    def sr_push_frontier(self, adj: "Adjacency", x: "Dense", out: "Dense", semiring: int):
        """out = canon(x), then out[v] ⊕= a ⊗ x[u] along the weighted adjacency's edges of the recorded frontier rows u
        (``arrow_sr_push_frontier``, ``semiring`` SR_MIN_PLUS, SR_MAX_PLUS, SR_MAX_MIN or SR_MIN_MAX); ``x`` must be the
        tile of the last ``sr_mark_frontier`` on ``adj``"""
        self._check(self.lib.arrow_sr_push_frontier(self._h, adj.h, x.h, out.h, int(semiring)))

    def sr_mark_frontier_steps(self, adj: "Adjacency", new: "Dense", old: "Dense", steps: "Dense", level: int):
        """``sr_mark_frontier``, and in the same pass steps[r, c] = ``level`` where ``new`` and ``old`` differ in bits
        (level 0: 0 everywhere) in the int32 tile ``steps`` (``arrow_sr_mark_frontier_steps``); synchronises"""
        n, rows, edges = c_int64(), c_int64(), c_int64()
        self._check(self.lib.arrow_sr_mark_frontier_steps(self._h, adj.h, new.h, old.h, steps.h, int(level), byref(n),
                                                          byref(rows), byref(edges)))
        return int(n.value), int(rows.value), int(edges.value)

    def sr_tree_parents(self, in_adj: "Adjacency", dist: "Dense", steps: "Dense", parent: "Dense", semiring: int,
                        count: bool = False) -> Optional[int]:
        """parent[v, s] = the smallest u of the loop-free in-adjacency's row v with a ⊗ D[u, s] == D[v, s] in bits and D[u, s]
        strictly better than D[v, s] or equal to it with T[u, s] < T[v, s]; -1 where T[v, s] == 0, D[v, s] is the ⊕
        identity or no such u exists (``arrow_sr_tree_parents``, ``semiring`` SR_MAX_MIN or SR_MIN_MAX; ``dist`` fp32,
        ``steps`` T and ``parent`` int32).  With ``count`` returns the in-list entries read (synchronises), else None."""
        n = c_int64()
        self._check(self.lib.arrow_sr_tree_parents(self._h, in_adj.h, dist.h, steps.h, parent.h, int(semiring),
                                                   byref(n) if count else None))
        return int(n.value) if count else None

    def out_weights(self, parts: Sequence[tuple], n_vertices: int, w: "Dense", inv: "Dense") -> Tuple[int, int, int]:
        """Out-weights of the operator of ``adj_build(parts, n_vertices)`` with its self-loops (``arrow_out_weights``):
        ``w`` (float64 [n x 1]) receives the float64 sum of each source's edge values in (part, entry) order, ``inv`` (the
        blocks' type, [n x 1]) fl(1 / w), 0 where w == 0.  Returns (edges with a negative, NaN or +-inf value, dangling
        vertices, other vertices whose inverse is not finite or 0); synchronises."""
        n = len(parts)
        csrs = (c_int * max(n, 1))(*[A.h for A, _ in parts])
        maps = (c_int * max(n, 1))(*[m.h if m is not None else -1 for _, m in parts])
        bad, dangling, bad_inv = c_int64(), c_int64(), c_int64()
        self._check(self.lib.arrow_out_weights(self._h, n, csrs, maps, int(n_vertices), w.h, inv.h, byref(bad), byref(dangling),
                                               byref(bad_inv)))
        return int(bad.value), int(dangling.value), int(bad_inv.value)

    def pagerank_restart(self, x: "Dense", inv: "Dense", s: "Dense", scratch: "Dense", state: "Dense") -> Tuple[np.ndarray, int, int]:
        """sigma = the chunked float64 column sums of ``x``; when no column is bad (a negative, NaN or +-inf value, or a
        sigma that is not positive and finite) ``s`` = fl(x / sigma) and state row 0 the dangling mass of ``s``
        (``arrow_pagerank_restart``).  Returns (sigma, bad columns, first bad column or -1); synchronises."""
        sums = np.zeros(x.k, np.float64)
        bad, first = c_int64(), c_int64()
        self._check(self.lib.arrow_pagerank_restart(self._h, x.h, inv.h, s.h, scratch.h, state.h,
                                                    sums.ctypes.data_as(POINTER(c_double)), byref(bad), byref(first)))
        return sums, int(bad.value), int(first.value)

    def pagerank_update(self, y: "Dense", p: "Dense", s: "Dense", inv: "Dense", scratch: "Dense", state: "Dense",
                        alpha: float) -> np.ndarray:
        """p_{t+1} = fl(fl(alpha Y) + fl(c S)) over ``y`` in place, c = fl(fl(1 - alpha) + fl(alpha m_t)); returns the
        float64 residuals sum |p_{t+1} - p_t| per column (``arrow_pagerank_update``); synchronises"""
        res = np.zeros(y.k, np.float64)
        self._check(self.lib.arrow_pagerank_update(self._h, y.h, p.h, s.h, inv.h, scratch.h, state.h, float(alpha),
                                                   res.ctypes.data_as(POINTER(c_double))))
        return res

    def connected_components(self, parts: Sequence[tuple], n_vertices: int, labels: "Dense",
                             sizes: Optional["Dense"] = None) -> int:
        """Weakly connected components of the operator of ``adj_build(parts, n_vertices)`` (``arrow_connected_components``):
        ``labels`` (int32 [n x 1]) receives the smallest vertex of each vertex's component, ``sizes`` (int32 [n x 1]) the
        member count at each label's row and 0 elsewhere.  Returns the number of components; synchronises."""
        n = len(parts)
        csrs = (c_int * max(n, 1))(*[A.h for A, _ in parts])
        maps = (c_int * max(n, 1))(*[m.h if m is not None else -1 for _, m in parts])
        count = c_int64()
        self._check(self.lib.arrow_connected_components(self._h, n, csrs, maps, int(n_vertices), labels.h,
                                                        sizes.h if sizes is not None else -1, byref(count)))
        return int(count.value)

    def count_diff(self, a: "Dense", b: "Dense") -> int:
        """rows in which two equally shaped tiles differ in some element (-0 == +0, NaN != NaN); synchronises"""
        n = c_int64()
        self._check(self.lib.arrow_dense_count_diff(self._h, a.h, b.h, byref(n)))
        return int(n.value)

    def count_diff_bits(self, a: "Dense", b: "Dense") -> int:
        """rows in which two equally shaped fp32 tiles differ in some element's bits (-0 != +0)
        (``arrow_dense_count_diff_bits``); synchronises"""
        n = c_int64()
        self._check(self.lib.arrow_dense_count_diff_bits(self._h, a.h, b.h, byref(n)))
        return int(n.value)

    def gather_rows_multi(self, dst: "Dense", srcs: Sequence["Dense"], row_bounds: Sequence[int], m: "RowMap",
                          accumulate: bool = False):
        n = len(srcs)
        hs = (c_int * n)(*[s.h for s in srcs])
        bd = (c_int64 * (n + 1))(*[int(b) for b in row_bounds])
        self._check(self.lib.arrow_gather_rows_multi(self._h, dst.h, hs, bd, n, m.h, ACCUMULATE if accumulate else 0))

    def peer_barrier(self, flag_tiles: Sequence["Dense"], rank: int):
        n = len(flag_tiles)
        hs = (c_int * n)(*[s.h for s in flag_tiles])
        self._check(self.lib.arrow_peer_barrier(self._h, hs, int(rank), n))

    # -- copy lanes -------------------------------------------------------------------------
    LANE_MAIN, LANE_H2D, LANE_D2H = 0, 1, 2

    def h2d_lane(self, lane: int, dst: "Dense", X: np.ndarray, row0: int = 0):
        assert X.dtype == dst.dtype and X.flags.c_contiguous and X.shape[1] == dst.cols
        self._check(self.lib.arrow_dense_h2d_lane(self._h, lane, dst.h, int(row0), X.shape[0], _ptr(X)))

    def d2h_lane(self, lane: int, src: "Dense", out: np.ndarray, row0: int = 0):
        assert out.dtype == src.dtype and out.flags.c_contiguous and out.shape[1] == src.cols
        self._check(self.lib.arrow_dense_d2h_lane(self._h, lane, src.h, int(row0), out.shape[0], _ptr(out)))

    def lane_wait(self, waiting_lane: int, signalling_lane: int):
        self._check(self.lib.arrow_lane_wait(self._h, waiting_lane, signalling_lane))

    def lane_sync(self, lane: int):
        self._check(self.lib.arrow_lane_sync(self._h, lane))

    def set_lane(self, lane: int):
        self._check(self.lib.arrow_set_lane(self._h, lane))

    def event_record(self, event: int, lane: int):
        self._check(self.lib.arrow_event_record(self._h, event, lane))

    def event_wait(self, event: int, lane: int):
        self._check(self.lib.arrow_event_wait(self._h, event, lane))

    # -- timing -----------------------------------------------------------------------------
    def timer_start(self, slot: int = 0):
        self._check(self.lib.arrow_timer_start(self._h, slot))

    def timer_stop(self, slot: int = 0):
        self._check(self.lib.arrow_timer_stop(self._h, slot))

    def timer_ms(self, slot: int = 0) -> float:
        ms = c_float()
        self._check(self.lib.arrow_timer_elapsed_ms(self._h, slot, byref(ms)))
        return float(ms.value)

    def launch_count(self) -> int:
        n = c_int64()
        self._check(self.lib.arrow_launch_count(self._h, byref(n)))
        return int(n.value)

    def l2_flush(self):
        self._check(self.lib.arrow_l2_flush(self._h))


class _Handle:
    def __init__(self, ctx: Context, h: int):
        self.ctx, self.h = ctx, h

    def _free(self, fn_name: str):
        if self.h >= 0 and self.ctx is not None and self.ctx._h:
            self.ctx._check(getattr(self.ctx.lib, fn_name)(self.ctx._h, self.h))     # a refused free keeps the handle
        self.h = -1


class Csr(_Handle):
    def __init__(self, ctx, h, n_rows, n_cols, nnz, dtype=np.float32):
        super().__init__(ctx, h)
        self.n_rows, self.n_cols, self.nnz = n_rows, n_cols, nnz
        self.dtype = np.dtype(dtype)

    def info(self):
        v = [c_int64() for _ in range(5)]
        self.ctx._check(self.ctx.lib.arrow_csr_info(self.ctx._h, self.h, *[byref(x) for x in v]))
        return dict(zip(("n_rows", "n_cols", "nnz", "max_row_nnz", "n_long_rows"), (x.value for x in v)))

    def remap_columns(self, m: "RowMap", new_n_cols: int) -> "Csr":
        h = c_int()
        self.ctx._check(self.ctx.lib.arrow_csr_remap_columns(self.ctx._h, self.h, m.h, int(new_n_cols), byref(h)))
        out = Csr(self.ctx, h.value, self.n_rows, int(new_n_cols), self.nnz, self.dtype)
        out._parent = self           # shares indptr/values: keep the source alive
        return out

    def scale_columns(self, scale: "Dense", m: Optional["RowMap"] = None) -> "Csr":
        """a values-only copy whose entry (r, c) holds fl(a * scale[m(c)]) (``arrow_csr_scale_columns``; ``m`` None: the
        identity); it shares this block's structure, so this block cannot be freed while the copy lives"""
        h = c_int()
        self.ctx._check(self.ctx.lib.arrow_csr_scale_columns(self.ctx._h, self.h, m.h if m is not None else -1, scale.h,
                                                             byref(h)))
        out = Csr(self.ctx, h.value, self.n_rows, self.n_cols, self.nnz, self.dtype)
        out._parent = self
        return out

    def free(self):
        self._free("arrow_csr_free")


class RowMap(_Handle):
    def __init__(self, ctx, h, n, limit):
        super().__init__(ctx, h)
        self.n, self.limit = n, limit

    def compose(self, outer: "RowMap") -> "RowMap":
        h = c_int()
        self.ctx._check(self.ctx.lib.arrow_map_compose(self.ctx._h, self.h, outer.h, byref(h)))
        return RowMap(self.ctx, h.value, self.n, outer.limit)

    def invert(self, n_out: int) -> "RowMap":
        h = c_int()
        self.ctx._check(self.ctx.lib.arrow_map_invert(self.ctx._h, self.h, int(n_out), byref(h)))
        return RowMap(self.ctx, h.value, int(n_out), self.n)

    def to_host(self) -> np.ndarray:
        out = np.empty(self.n, dtype=np.int32)
        self.ctx._check(self.ctx.lib.arrow_map_d2h(self.ctx._h, self.h, _ptr(out), self.n))
        return out

    def free(self):
        self._free("arrow_map_free")


class Adjacency(_Handle):
    """push adjacency (``arrow_adj_build``): a CSR, row u listing the destinations v of u; without values, or with the
    edges' fp32 weights (``arrow_adj_build_weighted``); or the in-adjacency (``arrow_adj_build_in``), row v listing the
    sources u of v"""

    def info(self):
        n, m = c_int64(), c_int64()
        self.ctx._check(self.ctx.lib.arrow_adj_info(self.ctx._h, self.h, byref(n), byref(m)))
        return {"n_vertices": int(n.value), "n_edges": int(m.value)}

    def d2h(self):
        """(indptr, indices) as int32 host arrays"""
        inf = self.info()
        indptr = np.empty(inf["n_vertices"] + 1, np.int32)
        indices = np.empty(inf["n_edges"], np.int32)
        self.ctx._check(self.ctx.lib.arrow_adj_d2h(self.ctx._h, self.h, _ptr(indptr), _ptr(indices)))
        return indptr, indices

    def values_d2h(self):
        """the weights as a float32 host array, in the order of ``d2h()``'s indices (weighted adjacency only)"""
        values = np.empty(self.info()["n_edges"], np.float32)
        self.ctx._check(self.ctx.lib.arrow_adj_values_d2h(self.ctx._h, self.h, _ptr(values)))
        return values

    def free(self):
        self._free("arrow_adj_free")


class PtrTable(_Handle):
    def __init__(self, ctx, h, n):
        super().__init__(ctx, h)
        self.n = n

    def free(self):
        self._free("arrow_ptrtable_free")


class Dense(_Handle):
    def __init__(self, ctx, h, rows, k, owned, dtype=np.float32):
        super().__init__(ctx, h)
        self.rows, self.k, self.owned = rows, k, owned
        self.bits = isinstance(dtype, str) and dtype == BITS
        self.dtype = np.dtype(np.uint32) if self.bits else np.dtype(dtype)       # host element type (words of a bit tile)
        self.cols = b1_words(k) if self.bits else k                              # host elements per row

    def device_dtype(self) -> np.dtype:
        """the element type the library holds for this tile (``arrow_dense_dtype``; ``BITS`` for a bit tile)"""
        code = c_int()
        self.ctx._check(self.ctx.lib.arrow_dense_dtype(self.ctx._h, self.h, byref(code)))
        return _CODE_TILE[code.value]

    def h2d(self, X: np.ndarray, row0: int = 0):
        """upload rows, converted to the tile's element type"""
        X = np.ascontiguousarray(X, dtype=self.dtype)
        if X.ndim != 2 or X.shape[1] != self.cols:
            raise ValueError(f"expected [rows x {self.cols}] {self.dtype}, got {X.shape}")
        self.ctx._check(self.ctx.lib.arrow_dense_h2d(self.ctx._h, self.h, int(row0), X.shape[0], _ptr(X)))
        self._keep = X                  # async copy: keep the host array alive until the next sync

    def d2h(self, out: Optional[np.ndarray] = None, row0: int = 0, rows: Optional[int] = None, sync: bool = True) -> np.ndarray:
        rows = self.rows - row0 if rows is None else rows
        if out is None:
            out = np.empty((rows, self.cols), dtype=self.dtype)
        assert out.dtype == self.dtype and out.flags.c_contiguous and out.shape == (rows, self.cols)
        self.ctx._check(self.ctx.lib.arrow_dense_d2h(self.ctx._h, self.h, int(row0), int(rows), _ptr(out)))
        if sync:
            self.ctx.sync()
        return out

    def fill(self, v: float = 0.0):
        self.ctx._check(self.ctx.lib.arrow_dense_fill(self.ctx._h, self.h, float(v)))

    def copy_from(self, src: "Dense", dst_row0: int = 0, src_row0: int = 0, rows: Optional[int] = None):
        rows = min(self.rows - dst_row0, src.rows - src_row0) if rows is None else rows
        self.ctx._check(self.ctx.lib.arrow_dense_copy(self.ctx._h, self.h, int(dst_row0), src.h, int(src_row0), int(rows)))

    def device_ptr(self) -> int:
        p = c_void_p()
        self.ctx._check(self.ctx.lib.arrow_dense_ptr(self.ctx._h, self.h, byref(p), None, None))
        return int(p.value)

    def ipc_export(self) -> bytes:
        buf = ctypes.create_string_buffer(IPC_HANDLE_BYTES)
        self.ctx._check(self.ctx.lib.arrow_ipc_export(self.ctx._h, self.h, buf))
        return buf.raw

    def free(self):
        self._free("arrow_dense_free")
