"""ctypes binding of the C ABI in include/kb_b200.h (libkbb200.so).

There is no CPU fallback anywhere in this package: if the shared library is missing, or no CUDA device
is present, every entry point raises.  The library is built in-tree by ``__graft_entry__.build()`` /
``make -C kubebrain_b200/csrc``.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence, Tuple

import numpy as np

from .packed import PackedEvents, PackedStore, PackedWatchers, Slab

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libkbb200.so")

KB_OUT_HOST, KB_OUT_DEVICE, KB_OUT_COUNT = 0, 1, 2
KB_WIRE_ETCD_KVS, KB_WIRE_ETCD_EVENTS = 0x10, 0x20  # OR-ed into KB_OUT_HOST / KB_OUT_DEVICE
KB_OK, KB_EINVAL, KB_ECUDA, KB_ENOMEM, KB_EUNSORTED, KB_ECOMPACTED, KB_ESTATE, KB_ENCCL, KB_ELIMIT = (
    0, -1, -2, -3, -4, -5, -6, -7, -8)
NCCL_ID_BYTES = 128

u8p = C.POINTER(C.c_uint8)
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)

# every symbol include/kb_b200.h declares (tests/test_abi.py checks the .so exports all of them)
KB_OP_PUT, KB_OP_DEL = 0, 1
KB_DIFF_MISSING, KB_DIFF_EXTRA, KB_DIFF_CHANGED = 1, 2, 3

ABI_SYMBOLS = [
    "kb_abi_version", "kb_open", "kb_close", "kb_last_error", "kb_stream", "kb_sync",
    "kb_load_sorted", "kb_store_info", "kb_store_mem", "kb_dump", "kb_restore", "kb_apply_batch", "kb_expire", "kb_set_compact_revision",
    "kb_reconcile", "kb_reconcile_view_get",
    "kb_range_batch", "kb_range_prefetch", "kb_range_submit", "kb_range_collect", "kb_pending_free", "kb_range_view_get", "kb_result_wait",
    "kb_range_stream_open", "kb_range_stream_next", "kb_range_stream_close", "kb_range_partitions", "kb_partition_view_get",
    "kb_wire_range_head", "kb_wire_range_tail", "kb_wire_watch_head",
    "kb_get_batch", "kb_get_view_get", "kb_get_submit", "kb_get_collect", "kb_get_elem_off",
    "kb_compact_sweep", "kb_compact_view_get", "kb_compact_stream_open", "kb_compact_stream_info", "kb_compact_stream_next",
    "kb_compact_stream_close", "kb_compact_page_view_get",
    "kb_watch_add", "kb_watch_del", "kb_watch_count", "kb_watch_match", "kb_events_upload", "kb_events_free",
    "kb_watch_match_dev", "kb_match_view_get", "kb_result_free",
    "kb_nccl_unique_id", "kb_nccl_init", "kb_cursor_allgather", "kb_cursor_transport", "kb_cursor_force_nccl",
    "kb_prof_enable", "kb_prof_reset", "kb_prof_read", "kb_launch_count",
]


class PendingRange:
    """a submitted range batch (kb_pending): collect() exactly once, or close() to give it up"""

    def __init__(self, eng, handle, keepalive):
        self._eng, self._h, self._keep = eng, handle, keepalive

    def collect(self) -> "RangeResult":
        if self._h is None:
            raise KbError(KB_ESTATE, "pending batch already collected")
        h, self._h = self._h, None
        r = C.c_void_p()
        self._eng._check(lib().kb_range_collect(self._eng._ctx, h, C.byref(r)))  # the C side ends the pending either way
        return RangeResult(self._eng, r)

    def close(self):
        if self._h is not None and self._eng._ctx:
            lib().kb_pending_free(self._eng._ctx, self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PendingGet(PendingRange):
    """a submitted batch of point reads (kb_get_submit): collect() exactly once, or close() to give it up"""

    def collect(self) -> "GetResult":
        if self._h is None:
            raise KbError(KB_ESTATE, "pending batch already collected")
        h, self._h = self._h, None
        r = C.c_void_p()
        self._eng._check(lib().kb_get_collect(self._eng._ctx, h, C.byref(r)))  # the C side ends the pending either way
        return GetResult(self._eng, r)


class RangeStream:
    """an open kb_range_stream: next(max_bytes) returns the next page as a RangeResult, None once exhausted"""

    def __init__(self, eng, handle):
        self._eng, self._h = eng, handle

    def next(self, max_bytes: int) -> Optional["RangeResult"]:
        if self._h is None:
            raise KbError(KB_ESTATE, "range stream already closed")
        r = C.c_void_p()
        self._eng._check(lib().kb_range_stream_next(self._eng._ctx, self._h, int(max_bytes), C.byref(r)))
        return RangeResult(self._eng, r) if r.value else None

    def close(self):
        if self._h is not None and self._eng._ctx:
            lib().kb_range_stream_close(self._eng._ctx, self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class KbError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"kb_b200 error {code}: {msg}")
        self.code = code


KB_CFG_HIGH_PRIORITY = 1
KB_CFG_HOST_VALUES = 2  # the value heap in mapped pinned host memory instead of HBM


class KbConfig(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("flags", C.c_uint32)]


class KbRangeReq(C.Structure):
    _fields_ = [("start", C.c_char_p), ("start_len", C.c_uint64), ("end", C.c_char_p), ("end_len", C.c_uint64),
                ("read_rev", C.c_uint64), ("limit", C.c_int64)]


class KbRangeView(C.Structure):
    _fields_ = [("n_req", C.c_uint64), ("req_first", u64p), ("req_count", u64p), ("req_examined", u64p),
                ("n_kvs", C.c_uint64), ("rec_idx", u32p), ("rev", u64p), ("key_off", u64p), ("key_len", u32p),
                ("val_off", u64p), ("val_len", u32p), ("bytes", C.c_void_p), ("n_bytes", C.c_uint64),
                ("on_device", C.c_int), ("elem_off", u64p), ("wire", C.c_int)]


class KbPartitionView(C.Structure):
    _fields_ = [("n_parts", C.c_uint64), ("key_off", u64p), ("kv_first", u64p), ("arena_first", u64p),
                ("bytes", C.c_void_p), ("n_bytes", C.c_uint64)]


class KbWriteOp(C.Structure):
    _fields_ = [("type", C.c_uint32), ("key", C.c_char_p), ("key_len", C.c_uint64), ("val", C.c_char_p),
                ("val_len", C.c_uint64), ("expire_unix", C.c_uint64)]


class KbReconcileView(C.Structure):
    _fields_ = [("n_engine", C.c_uint64), ("n_mirror", C.c_uint64), ("n_missing", C.c_uint64), ("n_extra", C.c_uint64),
                ("n_changed", C.c_uint64), ("n_diff", C.c_uint64), ("kind", u8p), ("src_idx", u64p), ("key_off", u64p),
                ("bytes", C.c_void_p), ("n_bytes", C.c_uint64)]


class KbGetReq(C.Structure):
    _fields_ = [("key", C.c_char_p), ("key_len", C.c_uint64), ("revision", C.c_uint64)]


class KbGetView(C.Structure):
    _fields_ = [("n", C.c_uint64), ("status", u8p), ("mod_rev", u64p), ("rec_idx", u32p), ("val_off", u64p),
                ("val_len", u32p), ("bytes", C.c_void_p), ("n_bytes", C.c_uint64), ("on_device", C.c_int)]


class KbCompactView(C.Structure):
    _fields_ = [("n_victims", C.c_uint64), ("victim_idx", C.c_void_p), ("victim_class", C.c_void_p),
                ("count", C.c_uint64), ("examined", C.c_uint64), ("on_device", C.c_int)]


class KbCompactPageView(C.Structure):
    _fields_ = [("first", C.c_uint64), ("n", C.c_uint64), ("rec_idx", u32p), ("victim_class", u8p),
                ("key_off", u64p), ("key_len", u32p), ("guard_off", u64p), ("guard_len", u32p),
                ("bytes", C.c_void_p), ("n_bytes", C.c_uint64)]


class KbEvents(C.Structure):
    _fields_ = [("keys", u8p), ("key_off", u64p), ("rev", u64p), ("n", C.c_uint64),
                ("batch_off", u64p), ("n_batches", C.c_uint64)]


class KbMatchView(C.Structure):
    _fields_ = [("n_watchers", C.c_uint64), ("start", u64p), ("event_idx", C.c_void_p),
                ("n_deliveries", C.c_uint64), ("on_device", C.c_int)]


class KbProfEntry(C.Structure):
    _fields_ = [("name", C.c_char * 32), ("launches", C.c_uint64), ("total_ms", C.c_double),
                ("alg_bytes", C.c_uint64)]


_lib = None
_rt = None


def _cudart():
    """the CUDA runtime libkbb200.so itself is linked against (tests read device-resident results through it)"""
    global _rt
    if _rt is None:
        lib()
        for name in ("libcudart.so.12", "libcudart.so"):
            try:
                _rt = C.CDLL(name)
                break
            except OSError:
                continue
        if _rt is None:
            raise RuntimeError("libcudart not loadable")
        _rt.cudaMemcpy.restype = C.c_int
        _rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    return _rt


def lib():
    """Load libkbb200.so; fail loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: the CUDA extension has not been built (run __graft_entry__.build() or "
            "`make -C kubebrain_b200/csrc`). kubebrain_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    L.kb_abi_version.restype = C.c_int
    L.kb_open.restype = C.c_int
    L.kb_open.argtypes = [C.c_int, vp, C.POINTER(vp)]
    L.kb_close.argtypes = [vp]
    L.kb_close.restype = None
    L.kb_last_error.restype = C.c_char_p
    L.kb_last_error.argtypes = [vp]
    L.kb_stream.restype = vp
    L.kb_stream.argtypes = [vp]
    L.kb_sync.restype = C.c_int
    L.kb_sync.argtypes = [vp]
    L.kb_load_sorted.restype = C.c_int
    L.kb_load_sorted.argtypes = [vp, u8p, u64p, u8p, u64p, C.c_uint64]
    L.kb_store_info.restype = C.c_int
    L.kb_store_info.argtypes = [vp, u64p, u64p, u64p]
    L.kb_store_mem.restype = C.c_int
    L.kb_store_mem.argtypes = [vp, u64p, u64p]
    L.kb_set_compact_revision.restype = C.c_int
    L.kb_dump.restype = C.c_int
    L.kb_dump.argtypes = [vp, C.c_char_p]
    L.kb_restore.restype = C.c_int
    L.kb_restore.argtypes = [vp, C.c_char_p]
    L.kb_apply_batch.argtypes = [vp, C.POINTER(KbWriteOp), C.c_uint64]
    L.kb_apply_batch.restype = C.c_int
    L.kb_expire.restype = C.c_int
    L.kb_expire.argtypes = [vp, C.c_uint64, u64p]
    L.kb_set_compact_revision.argtypes = [vp, C.c_int, C.c_uint64]
    L.kb_reconcile.restype = C.c_int
    L.kb_reconcile.argtypes = [vp, C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64, u8p, u64p, u8p, u64p, C.c_uint64,
                               C.c_int, C.POINTER(vp)]
    L.kb_reconcile_view_get.restype = C.c_int
    L.kb_reconcile_view_get.argtypes = [vp, C.POINTER(KbReconcileView)]
    L.kb_range_batch.restype = C.c_int
    L.kb_range_batch.argtypes = [vp, C.POINTER(KbRangeReq), C.c_uint64, C.c_int, C.POINTER(vp)]
    L.kb_range_prefetch.restype = C.c_int
    L.kb_range_prefetch.argtypes = [vp, C.POINTER(KbRangeReq), C.c_uint64]
    L.kb_range_submit.restype = C.c_int
    L.kb_range_submit.argtypes = [vp, C.POINTER(KbRangeReq), C.c_uint64, C.c_int, C.POINTER(vp)]
    L.kb_range_collect.restype = C.c_int
    L.kb_range_collect.argtypes = [vp, vp, C.POINTER(vp)]
    L.kb_pending_free.restype = None
    L.kb_pending_free.argtypes = [vp, vp]
    L.kb_range_view_get.restype = C.c_int
    L.kb_range_view_get.argtypes = [vp, C.POINTER(KbRangeView)]
    L.kb_range_stream_open.restype = C.c_int
    L.kb_range_stream_open.argtypes = [vp, C.POINTER(KbRangeReq), C.c_int, C.c_uint64, C.POINTER(vp)]
    L.kb_range_stream_next.restype = C.c_int
    L.kb_range_stream_next.argtypes = [vp, vp, C.c_uint64, C.POINTER(vp)]
    L.kb_range_stream_close.restype = None
    L.kb_range_stream_close.argtypes = [vp, vp]
    L.kb_range_partitions.restype = C.c_int
    L.kb_range_partitions.argtypes = [vp, C.POINTER(KbRangeReq), C.c_uint64, C.c_uint64, C.POINTER(vp)]
    L.kb_partition_view_get.restype = C.c_int
    L.kb_partition_view_get.argtypes = [vp, C.POINTER(KbPartitionView)]
    L.kb_result_wait.restype = C.c_int
    L.kb_result_wait.argtypes = [vp, vp, vp]
    L.kb_wire_range_head.restype = C.c_uint64
    L.kb_wire_range_head.argtypes = [C.c_uint64, u8p]
    L.kb_wire_range_tail.restype = C.c_uint64
    L.kb_wire_range_tail.argtypes = [C.c_int, C.c_int64, u8p]
    L.kb_wire_watch_head.restype = C.c_uint64
    L.kb_wire_watch_head.argtypes = [C.c_uint64, C.c_int, C.c_char_p, C.c_uint64, u8p]
    L.kb_get_batch.restype = C.c_int
    L.kb_get_batch.argtypes = [vp, C.POINTER(KbGetReq), C.c_uint64, C.c_int, C.POINTER(vp)]
    L.kb_get_view_get.restype = C.c_int
    L.kb_get_view_get.argtypes = [vp, C.POINTER(KbGetView)]
    L.kb_get_submit.restype = C.c_int
    L.kb_get_submit.argtypes = [vp, C.POINTER(KbGetReq), C.c_uint64, C.c_int, C.POINTER(vp)]
    L.kb_get_collect.restype = C.c_int
    L.kb_get_collect.argtypes = [vp, vp, C.POINTER(vp)]
    L.kb_get_elem_off.restype = C.c_int
    L.kb_get_elem_off.argtypes = [vp, C.POINTER(u64p)]
    L.kb_compact_sweep.restype = C.c_int
    L.kb_compact_sweep.argtypes = [vp, C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64, C.c_uint64, C.c_uint64,
                                   C.c_int, C.c_int, C.POINTER(vp)]
    L.kb_compact_view_get.restype = C.c_int
    L.kb_compact_view_get.argtypes = [vp, C.POINTER(KbCompactView)]
    L.kb_compact_stream_open.restype = C.c_int
    L.kb_compact_stream_open.argtypes = [vp, C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64, C.c_uint64, C.c_uint64,
                                         C.c_int, C.c_uint64, C.POINTER(vp)]
    L.kb_compact_stream_info.restype = C.c_int
    L.kb_compact_stream_info.argtypes = [vp, u64p, u64p, u64p]
    L.kb_compact_stream_next.restype = C.c_int
    L.kb_compact_stream_next.argtypes = [vp, vp, C.c_uint64, C.POINTER(vp)]
    L.kb_compact_stream_close.restype = None
    L.kb_compact_stream_close.argtypes = [vp, vp]
    L.kb_compact_page_view_get.restype = C.c_int
    L.kb_compact_page_view_get.argtypes = [vp, C.POINTER(KbCompactPageView)]
    L.kb_watch_add.restype = C.c_int
    L.kb_watch_add.argtypes = [vp, C.c_char_p, C.c_uint64, C.c_uint64, u32p]
    L.kb_watch_del.restype = C.c_int
    L.kb_watch_del.argtypes = [vp, C.c_uint32]
    L.kb_watch_count.restype = C.c_int
    L.kb_watch_count.argtypes = [vp, u64p]
    L.kb_watch_match.restype = C.c_int
    L.kb_watch_match.argtypes = [vp, C.POINTER(KbEvents), C.c_int, C.POINTER(vp)]
    L.kb_events_upload.restype = C.c_int
    L.kb_events_upload.argtypes = [vp, C.POINTER(KbEvents), C.POINTER(vp)]
    L.kb_events_free.restype = None
    L.kb_events_free.argtypes = [vp, vp]
    L.kb_watch_match_dev.restype = C.c_int
    L.kb_watch_match_dev.argtypes = [vp, vp, C.c_int, C.POINTER(vp)]
    L.kb_match_view_get.restype = C.c_int
    L.kb_match_view_get.argtypes = [vp, C.POINTER(KbMatchView)]
    L.kb_result_free.restype = None
    L.kb_result_free.argtypes = [vp, vp]
    L.kb_nccl_unique_id.restype = C.c_int
    L.kb_nccl_unique_id.argtypes = [u8p]
    L.kb_nccl_init.restype = C.c_int
    L.kb_nccl_init.argtypes = [vp, u8p, C.c_int, C.c_int]
    L.kb_cursor_allgather.restype = C.c_int
    L.kb_cursor_allgather.argtypes = [vp, C.c_uint64, u64p, u64p]
    L.kb_cursor_transport.restype = C.c_int
    L.kb_cursor_transport.argtypes = [vp]
    L.kb_cursor_force_nccl.restype = C.c_int
    L.kb_cursor_force_nccl.argtypes = [vp, C.c_int]
    L.kb_prof_enable.restype = C.c_int
    L.kb_prof_enable.argtypes = [vp, C.c_int]
    L.kb_prof_reset.restype = C.c_int
    L.kb_prof_reset.argtypes = [vp]
    L.kb_prof_read.restype = C.c_int
    L.kb_prof_read.argtypes = [vp, C.POINTER(KbProfEntry), C.c_int, C.POINTER(C.c_int)]
    L.kb_launch_count.restype = C.c_uint64
    L.kb_launch_count.argtypes = [vp]
    _lib = L
    return L


def _np(ptr, n: int, dtype) -> np.ndarray:
    if n == 0 or not ptr:
        return np.zeros(0, dtype=dtype)
    addr = ptr if isinstance(ptr, int) else C.cast(ptr, C.c_void_p).value
    buf = (C.c_uint8 * (n * np.dtype(dtype).itemsize)).from_address(addr)
    return np.frombuffer(buf, dtype=dtype, count=n)


def _slab_ptrs(s: Slab):
    data = s.data if s.data.size else np.zeros(1, np.uint8)
    data = np.ascontiguousarray(data)
    off = np.ascontiguousarray(s.off, dtype=np.uint64)
    return data, off, data.ctypes.data_as(u8p), off.ctypes.data_as(u64p)


class RangeResult:
    """One batch of scanner.Range answers (copies taken out of the library-owned arena on demand)."""

    def __init__(self, eng: "Engine", handle):
        self._eng, self._h = eng, handle
        v = KbRangeView()
        eng._check(lib().kb_range_view_get(handle, C.byref(v)))
        self.n_req = int(v.n_req)
        self.req_first = _np(v.req_first, self.n_req + 1, np.uint64).copy()
        self.req_count = _np(v.req_count, self.n_req, np.uint64).copy()
        self.req_examined = _np(v.req_examined, self.n_req, np.uint64).copy()
        self.n_kvs = int(v.n_kvs)
        self.n_bytes = int(v.n_bytes)
        self.on_device = bool(v.on_device)
        self.bytes_ptr = v.bytes
        self.wire = int(v.wire)
        n = self.n_kvs
        self.elem_off = None
        if self.on_device:
            # KB_OUT_DEVICE: the arena and the per-kv arrays stay in HBM (device pointers, kept as integers)
            self.arena = None
            self.rec_idx = self.rev = self.key_off = self.key_len = self.val_off = self.val_len = None
            self.dev_ptrs = {name: (C.cast(getattr(v, name), C.c_void_p).value or 0)
                             for name in ("rec_idx", "rev", "key_off", "key_len", "val_off", "val_len", "elem_off")}
        else:
            if self.wire:
                self.elem_off = _np(v.elem_off, n + 1, np.uint64) if n else np.zeros(1, np.uint64)
            self.rec_idx = _np(v.rec_idx, n, np.uint32)
            self.rev = _np(v.rev, n, np.uint64)
            self.key_off = _np(v.key_off, n, np.uint64)
            self.key_len = _np(v.key_len, n, np.uint32)
            self.val_off = _np(v.val_off, n, np.uint64)
            self.val_len = _np(v.val_len, n, np.uint32)
            self.arena = _np(v.bytes, self.n_bytes, np.uint8) if v.bytes else np.zeros(0, np.uint8)

    def device_array(self, name: str, dtype) -> np.ndarray:
        """KB_OUT_DEVICE answers: one of the per-kv arrays copied to the host (after waiting for the answer)"""
        assert self.on_device
        self.wait()
        n = self.n_kvs + (1 if name == "elem_off" else 0)
        raw = self._eng.read_device(self.dev_ptrs[name], n * np.dtype(dtype).itemsize, sync=False)
        return np.frombuffer(raw, dtype=dtype).copy()

    def kvs(self, q: int = 0) -> List[Tuple[bytes, bytes, int]]:
        assert self.arena is not None, "results were left on the device"
        a, b = int(self.req_first[q]), int(self.req_first[q + 1])
        out = []
        for k in range(a, b):
            ko, kl, vo, vl = int(self.key_off[k]), int(self.key_len[k]), int(self.val_off[k]), int(self.val_len[k])
            out.append((self.arena[ko : ko + kl].tobytes(), self.arena[vo : vo + vl].tobytes(), int(self.rev[k])))
        return out

    def wait(self, cuda_stream: int = 0):
        """KB_OUT_DEVICE answers: order `cuda_stream` behind the copy into the arena (0: block the host instead)"""
        self._eng._check(lib().kb_result_wait(self._eng._ctx, self._h, C.c_void_p(cuda_stream or None)))

    def rec_indices(self, q: int = 0) -> np.ndarray:
        return self.rec_idx[int(self.req_first[q]) : int(self.req_first[q + 1])].copy()

    def elements(self, q: int = 0, first: int = 0, count: Optional[int] = None) -> memoryview:
        """wire modes: the protobuf elements [first, first+count) of request q, as one contiguous slice of the arena"""
        assert self.wire and self.arena is not None
        a, b = int(self.req_first[q]), int(self.req_first[q + 1])
        lo = min(a + first, b)
        hi = b if count is None else min(lo + count, b)
        return memoryview(self.arena)[int(self.elem_off[lo]) : int(self.elem_off[hi])]

    def close(self):
        if self._h:
            lib().kb_result_free(self._eng._ctx, self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


GET_FOUND, GET_NOT_FOUND, GET_TOMBSTONE = 0, 1, 2


class GetResult:
    """answers of one batch of point reads (backend.get, pkg/backend/range.go:81-121).  In the wire mode
    (KB_WIRE_ETCD_KVS) the arena holds one RangeResponse.kvs element per FOUND read: element(i), bounded by elem_off."""

    def __init__(self, eng: "Engine", handle):
        self._eng, self._h = eng, handle
        v = KbGetView()
        eng._check(lib().kb_get_view_get(handle, C.byref(v)))
        n = int(v.n)
        self.n = n
        self.status = _np(v.status, n, np.uint8).copy()
        self.mod_rev = _np(v.mod_rev, n, np.uint64).copy()
        self.rec_idx = _np(v.rec_idx, n, np.uint32).copy()
        self.val_off = _np(v.val_off, n, np.uint64).copy()
        self.val_len = _np(v.val_len, n, np.uint32).copy()
        self.n_bytes = int(v.n_bytes)
        self.on_device = bool(v.on_device)
        self.arena = None if self.on_device else (_np(v.bytes, self.n_bytes, np.uint8) if v.bytes else np.zeros(0, np.uint8))
        self.bytes_ptr = v.bytes or 0
        eo = u64p()
        self.wire = lib().kb_get_elem_off(handle, C.byref(eo)) == KB_OK
        self.elem_off = _np(eo, n + 1, np.uint64).copy() if self.wire else None

    def value(self, i: int) -> Optional[bytes]:
        if self.status[i] != GET_FOUND:
            return None
        o, l = int(self.val_off[i]), int(self.val_len[i])
        return self.arena[o : o + l].tobytes()

    def element(self, i: int) -> bytes:
        """wire mode: the RangeResponse.kvs element of read i (empty unless it is FOUND)"""
        assert self.wire and self.arena is not None
        return self.arena[int(self.elem_off[i]) : int(self.elem_off[i + 1])].tobytes()

    def close(self):
        if self._h:
            lib().kb_result_free(self._eng._ctx, self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ReconcileResult:
    """The diff of one kb_reconcile, copied out of the library-owned result: counts, `kinds` (KB_DIFF_* per diff, in key
    order), `src_idx` (input index of a MISSING / CHANGED diff, 2**64 - 1 for EXTRA) and keys()."""

    def __init__(self, v: "KbReconcileView"):
        self.n_engine, self.n_mirror = int(v.n_engine), int(v.n_mirror)
        self.n_missing, self.n_extra, self.n_changed = int(v.n_missing), int(v.n_extra), int(v.n_changed)
        self.n_diff = int(v.n_diff)
        self.kinds = _np(v.kind, self.n_diff, np.uint8).copy()
        self.src_idx = _np(v.src_idx, self.n_diff, np.uint64).copy()
        self._key_off = _np(v.key_off, self.n_diff + 1, np.uint64).astype(np.int64)
        self._bytes = _np(v.bytes, int(v.n_bytes), np.uint8).tobytes() if v.bytes else b""

    def keys(self) -> List[bytes]:
        """the internal key of every diff, in key order"""
        o = self._key_off
        return [self._bytes[o[k]: o[k + 1]] for k in range(self.n_diff)]


class CompactResult:
    def __init__(self, eng: "Engine", handle):
        self._eng, self._h = eng, handle
        v = KbCompactView()
        eng._check(lib().kb_compact_view_get(handle, C.byref(v)))
        self.n_victims = int(v.n_victims)
        self.count = int(v.count)
        self.examined = int(v.examined)
        self.on_device = bool(v.on_device)
        self.dev_ptrs = {}
        if not self.on_device and v.victim_idx:
            self.victim_idx = _np(v.victim_idx, self.n_victims, np.uint32).copy()
            self.victim_class = _np(v.victim_class, self.n_victims, np.uint8).copy()
        else:
            self.victim_idx = np.zeros(0, np.uint32)
            self.victim_class = np.zeros(0, np.uint8)
            if self.on_device and v.victim_idx:
                # KB_OUT_DEVICE: both arrays stay in HBM (device pointers, kept as integers)
                self.dev_ptrs = {"victim_idx": v.victim_idx, "victim_class": v.victim_class}

    def device_array(self, name: str) -> np.ndarray:
        """KB_OUT_DEVICE answers: victim_idx (u32) or victim_class (u8) copied to the host"""
        assert self.on_device
        dtype = np.uint32 if name == "victim_idx" else np.uint8
        if not self.n_victims:
            return np.zeros(0, dtype)
        raw = self._eng.read_device(self.dev_ptrs[name], self.n_victims * np.dtype(dtype).itemsize)
        return np.frombuffer(raw, dtype=dtype).copy()

    def close(self):
        if self._h:
            lib().kb_result_free(self._eng._ctx, self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CompactPage:
    """one page of a compaction stream: victims [first, first + n) of the sweep's ordered delete-call list, with the
    internal key of every delete call and, for classes 3 / 4 (DelCurrent), the value the sweep read (the guard).  The
    arrays are copies: the page owns nothing after __init__."""

    def __init__(self, eng: "Engine", handle):
        v = KbCompactPageView()
        try:
            eng._check(lib().kb_compact_page_view_get(handle, C.byref(v)))
            n = int(v.n)
            self.first, self.n = int(v.first), n
            self.rec_idx = _np(v.rec_idx, n, np.uint32).copy()
            self.victim_class = _np(v.victim_class, n, np.uint8).copy()
            self.key_off = _np(v.key_off, n, np.uint64).copy()
            self.key_len = _np(v.key_len, n, np.uint32).copy()
            self.guard_off = _np(v.guard_off, n, np.uint64).copy()
            self.guard_len = _np(v.guard_len, n, np.uint32).copy()
            self.n_bytes = int(v.n_bytes)
            self.arena = _np(v.bytes, self.n_bytes, np.uint8).copy() if v.bytes else np.zeros(0, np.uint8)
        finally:
            lib().kb_result_free(eng._ctx, handle)

    def key(self, i: int) -> bytes:
        o = int(self.key_off[i])
        return self.arena[o : o + int(self.key_len[i])].tobytes()

    def guard(self, i: int) -> bytes:
        o = int(self.guard_off[i])
        return self.arena[o : o + int(self.guard_len[i])].tobytes()

    def keys(self) -> List[bytes]:
        return [self.key(i) for i in range(self.n)]

    def guards(self) -> List[bytes]:
        return [self.guard(i) for i in range(self.n)]


class CompactStream:
    """an open kb_compact_stream: the sweep's count / examined / n_victims, and next(max_bytes) -> CompactPage, None once
    every victim has been handed out"""

    def __init__(self, eng, handle):
        self._eng, self._h = eng, handle
        n, c, x = C.c_uint64(), C.c_uint64(), C.c_uint64()
        eng._check(lib().kb_compact_stream_info(handle, C.byref(n), C.byref(c), C.byref(x)))
        self.n_victims, self.count, self.examined = n.value, c.value, x.value

    def next(self, max_bytes: int) -> Optional[CompactPage]:
        if self._h is None:
            raise KbError(KB_ESTATE, "compaction stream already closed")
        r = C.c_void_p()
        self._eng._check(lib().kb_compact_stream_next(self._eng._ctx, self._h, int(max_bytes), C.byref(r)))
        return CompactPage(self._eng, r) if r.value else None

    def close(self):
        if self._h is not None and self._eng._ctx:
            lib().kb_compact_stream_close(self._eng._ctx, self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class MatchResult:
    def __init__(self, eng: "Engine", handle):
        self._eng, self._h = eng, handle
        v = KbMatchView()
        eng._check(lib().kb_match_view_get(handle, C.byref(v)))
        self.n_watchers = int(v.n_watchers)
        self.n_deliveries = int(v.n_deliveries)
        self.on_device = bool(v.on_device)
        self.start = _np(v.start, self.n_watchers + 1, np.uint64).copy()
        self.event_idx = (_np(v.event_idx, self.n_deliveries, np.uint32).copy()
                          if not self.on_device else np.zeros(0, np.uint32))
        # KB_OUT_DEVICE: the delivery lists stay in HBM and may still be being written when the call returns (on the
        # context's second stream): wait() / kb_sync before reading them
        self.event_idx_ptr = int(v.event_idx or 0) if self.on_device else 0

    def wait(self, cuda_stream: int = 0):
        """KB_OUT_DEVICE answers: order `cuda_stream` behind the delivery lists (0: block the host instead)"""
        self._eng._check(lib().kb_result_wait(self._eng._ctx, self._h, C.c_void_p(cuda_stream or None)))

    def device_event_idx(self) -> np.ndarray:
        self.wait()
        raw = self._eng.read_device(self.event_idx_ptr, self.n_deliveries * 4, sync=False)
        return np.frombuffer(raw, dtype=np.uint32).copy()

    def deliveries(self, watcher_id: int) -> np.ndarray:
        return self.event_idx[int(self.start[watcher_id]) : int(self.start[watcher_id + 1])]

    def close(self):
        if self._h:
            lib().kb_result_free(self._eng._ctx, self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PackedRangeReqs:
    """A kb_range_req[] built once; keeps the bound keys alive."""

    def __init__(self, reqs: Sequence[Tuple[bytes, bytes, int, int]]):
        self.n = len(reqs)
        self._keep = list(reqs)
        self.arr = (KbRangeReq * max(self.n, 1))()
        for i, (s, e, rev, lim) in enumerate(self._keep):
            self.arr[i] = KbRangeReq(s, len(s), e, len(e), rev, lim)


class Engine:
    """A kb_ctx: one HBM-resident snapshot + watcher table on one GPU.  host_values=True keeps the snapshot's value heap
    in mapped pinned host memory instead of HBM (KB_CFG_HOST_VALUES), for the life of the context."""

    def __init__(self, device: int = 0, high_priority: bool = False, host_values: bool = False):
        self._ctx = C.c_void_p()
        cfg = KbConfig(C.sizeof(KbConfig), Engine.config_flags(high_priority, host_values))
        rc = lib().kb_open(device, C.byref(cfg), C.byref(self._ctx))
        if rc != 0:
            raise KbError(rc, "kb_open failed: no usable CUDA device (kubebrain_b200 has no CPU fallback)")
        self.device = device
        self.host_values = host_values
        self._keep = []

    @staticmethod
    def config_flags(high_priority: bool = False, host_values: bool = False) -> int:
        """kb_config.flags for the options of Engine()"""
        return (KB_CFG_HIGH_PRIORITY if high_priority else 0) | (KB_CFG_HOST_VALUES if host_values else 0)

    def _check(self, rc: int):
        if rc != 0:
            raise KbError(rc, (lib().kb_last_error(self._ctx) or b"").decode("utf-8", "replace"))

    def close(self):
        if self._ctx:
            lib().kb_close(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- store ----
    def load_sorted(self, store: PackedStore):
        kd, ko, kp, kop = _slab_ptrs(store.keys)
        vd, vo, vp, vop = _slab_ptrs(store.vals)
        self._check(lib().kb_load_sorted(self._ctx, kp, kop, vp, vop, store.n))

    def apply_batch(self, ops: Sequence[tuple]):
        """One committed BatchWrite (pkg/storage/interface.go:62-84): (internal_key, value) puts, (internal_key, None)
        deletes, applied in order (the last op on a key wins).  A put may carry a third element: the wall-clock second at
        which the key expires (BatchWrite.Put(key, val, ttl) of a TTL engine)."""
        arr = (KbWriteOp * max(len(ops), 1))()
        for i, op in enumerate(ops):
            k, v = op[0], op[1]
            arr[i].type = KB_OP_DEL if v is None else KB_OP_PUT
            arr[i].key, arr[i].key_len = k, len(k)
            if v is not None:
                arr[i].val, arr[i].val_len = v, len(v)
                arr[i].expire_unix = int(op[2]) if len(op) > 2 and op[2] else 0
        self._check(lib().kb_apply_batch(self._ctx, arr, len(ops)))

    def expire(self, now_unix: int) -> int:
        """drop every TTL record whose time has come (kb_expire); returns the number of records removed"""
        n = C.c_uint64()
        self._check(lib().kb_expire(self._ctx, int(now_unix), C.byref(n)))
        return n.value

    def dump(self, path: str):
        """write the snapshot (directory, slabs, compact revision) to `path` (atomically: tmp file + rename)"""
        self._check(lib().kb_dump(self._ctx, os.fsencode(path)))

    def restore(self, path: str):
        """replace the snapshot with the one in `path` (validated: header, checksums, directory, key order)"""
        self._check(lib().kb_restore(self._ctx, os.fsencode(path)))

    def store_info(self) -> Tuple[int, int, int]:
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self._check(lib().kb_store_info(self._ctx, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    def store_mem(self) -> Tuple[int, int]:
        """(device_bytes, host_bytes) the context holds for its snapshot -- key slab, value heap, both directory sets --
        by placement, as allocated capacity (kb_store_mem)"""
        d, h = C.c_uint64(), C.c_uint64()
        self._check(lib().kb_store_mem(self._ctx, C.byref(d), C.byref(h)))
        return d.value, h.value

    def reconcile(self, start: bytes, end: bytes, items, dry_run: bool = False) -> ReconcileResult:
        """Compare the engine's records of [start, end) -- `items`: a PackedStore or (internal_key, value) pairs, passed
        in the order given (the library refuses one that is not strictly ascending) -- with the snapshot's, and unless
        dry_run commit the difference as one batch (kb_reconcile)."""
        if not isinstance(items, PackedStore):
            items = list(items)
            items = PackedStore(Slab.from_list([k for k, _ in items]), Slab.from_list([v for _, v in items]))
        store = items
        kd, ko, kp, kop = _slab_ptrs(store.keys)
        vd, vo, vp, vop = _slab_ptrs(store.vals)
        h = C.c_void_p()
        self._check(lib().kb_reconcile(self._ctx, start, len(start), end, len(end), kp, kop, vp, vop, store.n,
                                       int(bool(dry_run)), C.byref(h)))
        try:
            v = KbReconcileView()
            self._check(lib().kb_reconcile_view_get(h, C.byref(v)))
            return ReconcileResult(v)
        finally:
            lib().kb_result_free(self._ctx, h)

    def set_compact_revision(self, rev: Optional[int]):
        self._check(lib().kb_set_compact_revision(self._ctx, int(rev is not None), rev or 0))

    # ---- scans ----
    @staticmethod
    def pack_range_reqs(reqs: Sequence[Tuple[bytes, bytes, int, int]]) -> "PackedRangeReqs":
        """marshal once what a C / cgo caller passes directly: a kb_range_req array (reusable across calls)"""
        return PackedRangeReqs(reqs)

    def range_batch(self, reqs, out_mode: int = KB_OUT_HOST) -> RangeResult:
        """reqs: sequence of (start_internal_key, end_internal_key, read_rev, limit), or a PackedRangeReqs"""
        pk = reqs if isinstance(reqs, PackedRangeReqs) else PackedRangeReqs(reqs)
        h = C.c_void_p()
        self._check(lib().kb_range_batch(self._ctx, pk.arr, pk.n, out_mode, C.byref(h)))
        return RangeResult(self, h)

    def range_submit(self, reqs, out_mode: int = KB_OUT_HOST) -> "PendingRange":
        """first half of range_batch: the batch is laid out and its kernels launched; .collect() returns the RangeResult.
        Submit batch n+1 before collecting batch n to keep two batches in flight (kb_range_submit / kb_range_collect)."""
        pk = reqs if isinstance(reqs, PackedRangeReqs) else PackedRangeReqs(reqs)
        h = C.c_void_p()
        self._check(lib().kb_range_submit(self._ctx, pk.arr, pk.n, out_mode, C.byref(h)))
        return PendingRange(self, h, pk)

    def range_stream(self, req: Tuple[bytes, bytes, int, int], out_mode: int = KB_OUT_HOST,
                     group_kvs: int = 300) -> RangeStream:
        """req = (start_internal_key, end_internal_key, read_rev, limit <= 0): one unlimited range scanned once, then
        handed out by RangeStream.next(max_bytes) in pages of whole groups of group_kvs kvs (kb_range_stream_open)"""
        pk = PackedRangeReqs([req])
        h = C.c_void_p()
        self._check(lib().kb_range_stream_open(self._ctx, pk.arr, out_mode, int(group_kvs), C.byref(h)))
        return RangeStream(self, h)

    def range_partitions(self, start: bytes, end: bytes, read_rev: int, part_bytes: int,
                         max_parts: int) -> Tuple[List[bytes], np.ndarray, np.ndarray]:
        """[start, end) at read_rev cut into at most max_parts answer-balanced partitions of about part_bytes raw-arena
        bytes each (kb_range_partitions): (borders, kv_first, arena_first) -- len(borders) = partitions + 1, partition k
        is [borders[k], borders[k+1]) and holds kvs [kv_first[k], kv_first[k+1]) of the unlimited answer"""
        pk = PackedRangeReqs([(start, end, read_rev, 0)])
        h = C.c_void_p()
        self._check(lib().kb_range_partitions(self._ctx, pk.arr, int(part_bytes), int(max_parts), C.byref(h)))
        try:
            v = KbPartitionView()
            self._check(lib().kb_partition_view_get(h, C.byref(v)))
            n = int(v.n_parts)
            key_off = _np(v.key_off, n + 2, np.uint64).astype(np.int64)
            raw = _np(v.bytes, int(v.n_bytes), np.uint8).tobytes() if v.bytes else b""
            borders = [raw[key_off[k] : key_off[k + 1]] for k in range(n + 1)]
            return borders, _np(v.kv_first, n + 1, np.uint64).copy(), _np(v.arena_first, n + 1, np.uint64).copy()
        finally:
            lib().kb_result_free(self._ctx, h)

    def range_prefetch(self, reqs):
        """start the bound search of a batch that a later range_batch(reqs) will ask for (kb_range_prefetch)"""
        pk = reqs if isinstance(reqs, PackedRangeReqs) else PackedRangeReqs(reqs)
        self._check(lib().kb_range_prefetch(self._ctx, pk.arr, pk.n))

    def get_batch(self, reqs: Sequence[Tuple[bytes, int]], out_mode: int = KB_OUT_HOST) -> GetResult:
        """reqs: (user_key, revision) -- revision 0 means latest"""
        arr = (KbGetReq * max(len(reqs), 1))()
        for i, (k, rev) in enumerate(reqs):
            arr[i] = KbGetReq(k, len(k), rev)
        h = C.c_void_p()
        self._check(lib().kb_get_batch(self._ctx, arr, len(reqs), out_mode, C.byref(h)))
        return GetResult(self, h)

    def get_submit(self, reqs: Sequence[Tuple[bytes, int]], out_mode: int = KB_OUT_HOST) -> "PendingGet":
        """first half of get_batch: the point reads are launched on a lane beside the range batches in flight; .collect()
        returns the GetResult (kb_get_submit / kb_get_collect).  out_mode may carry KB_WIRE_ETCD_KVS."""
        arr = (KbGetReq * max(len(reqs), 1))()
        keep = [k for k, _ in reqs]
        for i, (k, rev) in enumerate(reqs):
            arr[i] = KbGetReq(k, len(k), rev)
        h = C.c_void_p()
        self._check(lib().kb_get_submit(self._ctx, arr, len(reqs), out_mode, C.byref(h)))
        return PendingGet(self, h, keep)

    def compact_sweep(self, start: bytes, end: bytes, rev: int, timeout_rev: int = 0, support_ttl: bool = True,
                      out_mode: int = KB_OUT_HOST) -> CompactResult:
        h = C.c_void_p()
        self._check(lib().kb_compact_sweep(self._ctx, start, len(start), end, len(end), rev, timeout_rev,
                                           int(support_ttl), out_mode, C.byref(h)))
        return CompactResult(self, h)

    def compact_stream(self, start: bytes, end: bytes, rev: int, timeout_rev: int = 0, support_ttl: bool = True,
                       group_victims: int = 1024) -> CompactStream:
        """compact_sweep's victims handed out as internal keys (+ guards) by CompactStream.next(max_bytes), in pages of
        whole groups of group_victims victims (kb_compact_stream_open)"""
        h = C.c_void_p()
        self._check(lib().kb_compact_stream_open(self._ctx, start, len(start), end, len(end), rev, timeout_rev,
                                                 int(support_ttl), int(group_victims), C.byref(h)))
        return CompactStream(self, h)

    # ---- watch ----
    def watch_add(self, prefix: bytes, min_rev: int) -> int:
        wid = C.c_uint32()
        self._check(lib().kb_watch_add(self._ctx, prefix, len(prefix), min_rev, C.byref(wid)))
        return wid.value

    def watch_add_many(self, w: PackedWatchers) -> List[int]:
        return [self.watch_add(w.prefixes[i], int(w.min_rev[i])) for i in range(w.n)]

    def watch_del(self, wid: int):
        self._check(lib().kb_watch_del(self._ctx, wid))

    def watch_count(self) -> int:
        n = C.c_uint64()
        self._check(lib().kb_watch_count(self._ctx, C.byref(n)))
        return n.value

    @staticmethod
    def _events_c(ev: PackedEvents):
        kd, ko, kp, kop = _slab_ptrs(ev.keys)
        rev = np.ascontiguousarray(ev.rev, dtype=np.uint64)
        bo = np.ascontiguousarray(ev.batch_off, dtype=np.uint64)
        c = KbEvents(kp, kop, rev.ctypes.data_as(u64p), ev.n, bo.ctypes.data_as(u64p), len(bo) - 1)
        return c, (kd, ko, rev, bo)

    def watch_match(self, ev: PackedEvents, out_mode: int = KB_OUT_HOST) -> MatchResult:
        c, keep = self._events_c(ev)
        h = C.c_void_p()
        self._check(lib().kb_watch_match(self._ctx, C.byref(c), out_mode, C.byref(h)))
        return MatchResult(self, h)

    def events_upload(self, ev: PackedEvents):
        c, keep = self._events_c(ev)
        h = C.c_void_p()
        self._check(lib().kb_events_upload(self._ctx, C.byref(c), C.byref(h)))
        return h

    def events_free(self, h):
        lib().kb_events_free(self._ctx, h)

    def watch_match_dev(self, ev_handle, out_mode: int = KB_OUT_DEVICE) -> MatchResult:
        h = C.c_void_p()
        self._check(lib().kb_watch_match_dev(self._ctx, ev_handle, out_mode, C.byref(h)))
        return MatchResult(self, h)

    # ---- multi-GPU cursor ----
    @staticmethod
    def nccl_unique_id() -> bytes:
        buf = (C.c_uint8 * NCCL_ID_BYTES)()
        rc = lib().kb_nccl_unique_id(buf)
        if rc != 0:
            raise KbError(rc, "ncclGetUniqueId failed (libnccl.so.2 not loadable?)")
        return bytes(buf)

    def nccl_init(self, uid: bytes, rank: int, nranks: int):
        buf = (C.c_uint8 * NCCL_ID_BYTES).from_buffer_copy(uid)
        self._check(lib().kb_nccl_init(self._ctx, buf, rank, nranks))
        self._nranks = nranks

    def cursor_allgather(self, local_rev: int) -> Tuple[np.ndarray, int]:
        out = np.zeros(self._nranks, np.uint64)
        mn = C.c_uint64()
        self._check(lib().kb_cursor_allgather(self._ctx, local_rev, out.ctypes.data_as(u64p), C.byref(mn)))
        return out, mn.value

    def cursor_mode(self) -> str:
        return {0: "none", 1: "single", 2: "nccl", 3: "p2p"}[lib().kb_cursor_transport(self._ctx)]

    def cursor_force_nccl(self, on: bool):
        """collective: every rank switches before the next exchange"""
        self._check(lib().kb_cursor_force_nccl(self._ctx, int(on)))

    # ---- measurement ----
    def stream(self) -> int:
        return lib().kb_stream(self._ctx) or 0

    def sync(self):
        self._check(lib().kb_sync(self._ctx))

    def read_device(self, ptr: int, nbytes: int, sync: bool = True) -> bytes:
        """copy `nbytes` of a KB_OUT_DEVICE result to the host, after kb_sync (sync=False: the caller has already waited
        for the answer with RangeResult.wait)"""
        if sync:
            self.sync()
        if nbytes == 0:
            return b""
        rt = _cudart()
        buf = (C.c_uint8 * nbytes)()
        rc = rt.cudaMemcpy(buf, C.c_void_p(ptr), C.c_size_t(nbytes), 2)  # cudaMemcpyDeviceToHost
        if rc != 0:
            raise KbError(KB_ECUDA, f"cudaMemcpy failed with {rc}")
        return bytes(buf)

    def prof_enable(self, level: int):
        """0 off, 1 every kernel, 2 only the two HBM-bound kernels"""
        self._check(lib().kb_prof_enable(self._ctx, int(level)))

    def prof_reset(self):
        self._check(lib().kb_prof_reset(self._ctx))

    def prof_read(self):
        arr = (KbProfEntry * 64)()
        n = C.c_int()
        self._check(lib().kb_prof_read(self._ctx, arr, 64, C.byref(n)))
        return [dict(name=arr[i].name.decode(), launches=int(arr[i].launches), total_ms=float(arr[i].total_ms),
                     alg_bytes=int(arr[i].alg_bytes)) for i in range(min(n.value, 64))]

    def launch_count(self) -> int:
        return int(lib().kb_launch_count(self._ctx))
