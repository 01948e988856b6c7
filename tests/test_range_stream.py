"""CPU tests of the paged range stream (kb_range_stream_open / _next / _close): the symbols cross the boundary, the
argument checks answer KB_EINVAL before any CUDA call, and Scanner.range_stream_paged sends exactly the messages of
Scanner.range_stream over a stub engine that cuts pages the way the library does."""
from __future__ import annotations

import ctypes

import pytest

from kubebrain_b200 import _lib
from kubebrain_b200._lib import (KB_EINVAL, KB_ECOMPACTED, KB_OUT_COUNT, KB_OUT_DEVICE, KB_OUT_HOST,
                                 KB_WIRE_ETCD_EVENTS, KB_WIRE_ETCD_KVS, KbError)
from kubebrain_b200.scanner import RANGE_STREAM_BATCH, Scanner
from tests.test_abi import _declared

NAMES = ["kb_range_stream_open", "kb_range_stream_next", "kb_range_stream_close"]


def test_symbols_declared_exported_and_bound():
    assert set(NAMES) <= set(_declared())
    assert set(NAMES) <= set(_lib.ABI_SYMBOLS)
    L = ctypes.CDLL(_lib.LIB_PATH)
    for n in NAMES:
        assert hasattr(L, n)
    assert L.kb_abi_version() == 2


def test_invalid_arguments_need_no_device():
    L = _lib.lib()
    req = (_lib.KbRangeReq * 1)()
    h = ctypes.c_void_p()
    assert L.kb_range_stream_open(None, req, KB_OUT_HOST, 300, ctypes.byref(h)) == KB_EINVAL
    assert L.kb_range_stream_next(None, None, 1 << 20, ctypes.byref(h)) == KB_EINVAL
    L.kb_range_stream_close(None, None)
    # the mode, group and limit checks come before the context is touched: a placeholder handle never gets read
    fake = ctypes.create_string_buffer(64)
    ctx = ctypes.cast(fake, ctypes.c_void_p)
    assert L.kb_range_stream_open(ctx, None, KB_OUT_HOST, 300, ctypes.byref(h)) == KB_EINVAL
    assert L.kb_range_stream_open(ctx, req, KB_OUT_HOST, 300, None) == KB_EINVAL
    assert L.kb_range_stream_next(ctx, None, 0, ctypes.byref(h)) == KB_EINVAL
    for mode in (KB_OUT_COUNT, KB_OUT_COUNT | KB_WIRE_ETCD_KVS, KB_OUT_HOST | KB_WIRE_ETCD_KVS | KB_WIRE_ETCD_EVENTS, 7):
        assert L.kb_range_stream_open(ctx, req, mode, 300, ctypes.byref(h)) == KB_EINVAL, mode
    assert L.kb_range_stream_open(ctx, req, KB_OUT_DEVICE | KB_WIRE_ETCD_EVENTS, 0, ctypes.byref(h)) == KB_EINVAL
    lim = (_lib.KbRangeReq * 1)()
    lim[0].limit = 5
    assert L.kb_range_stream_open(ctx, lim, KB_OUT_HOST, 300, ctypes.byref(h)) == KB_EINVAL
    bad = (_lib.KbRangeReq * 1)()
    bad[0].start_len = 3  # NULL key with a length
    assert L.kb_range_stream_open(ctx, bad, KB_OUT_HOST, 300, ctypes.byref(h)) == KB_EINVAL
    assert h.value is None


# ---- a stub engine: one answer, handed out whole (range_batch) or in greedy pages of whole groups (range_stream) --
def _answer(n: int):
    return [(b"/k/%06d" % i, bytes([i % 251]) * (i * 37 % 500), 10 + i) for i in range(n)]


def _size(kv) -> int:  # padded [internal key][value] arena bytes of one kv
    return ((len(kv[0]) + 13 + 15) & ~15) + ((len(kv[1]) + 15) & ~15)


class _Page:
    def __init__(self, kvs):
        self._kvs = kvs

    def kvs(self, q=0):
        assert q == 0
        return list(self._kvs)

    def close(self):
        pass


class _Stream:
    def __init__(self, kvs, group):
        self.kvs, self.group, self.a, self.closed = kvs, group, 0, False

    def next(self, max_bytes):
        n, a, g = len(self.kvs), self.a, self.group
        if a >= n:
            return None
        b = min(a + g, n)
        while b < n and sum(_size(kv) for kv in self.kvs[a : min(b + g, n)]) <= max_bytes:
            b = min(b + g, n)
        self.a = b
        return _Page(self.kvs[a:b])

    def close(self):
        self.closed = True


class _StubEngine:
    def __init__(self, kvs, err=None):
        self.kvs, self.err, self.streams = kvs, err, []

    def range_batch(self, reqs, out_mode):
        if self.err:
            raise self.err
        assert len(reqs) == 1 and reqs[0][3] == 0 and out_mode == KB_OUT_HOST
        return _Page(self.kvs)

    def range_stream(self, req, out_mode, group_kvs):
        if self.err:
            raise self.err
        assert req[3] == 0 and out_mode == KB_OUT_HOST and group_kvs == RANGE_STREAM_BATCH
        s = _Stream(self.kvs, group_kvs)
        self.streams.append(s)
        return s


@pytest.mark.parametrize("n", [0, 1, 299, 300, 301, 650])
@pytest.mark.parametrize("budget", [0, 1, 40_000, 150_000, 1 << 40])
def test_paged_messages_equal_one_shot(n, budget):
    eng = _StubEngine(_answer(n))
    sc = Scanner(eng)
    got = list(sc.range_stream_paged(b"a", b"b", 77, budget))
    assert got == list(sc.range_stream(b"a", b"b", 77))
    assert [len(m.kvs) for m in got[:-1]] == [min(300, n - i) for i in range(0, n, 300)]
    assert got[-1].revision == 77 and not got[-1].more and got[-1].err == ""
    assert all(m.revision == 0 and m.more for m in got[:-1])
    assert all(s.closed for s in eng.streams)


def test_open_error_gives_the_end_marker():
    err = KbError(KB_ECOMPACTED, "range stream revision 5 less than compact revision 9")
    sc = Scanner(_StubEngine([], err))
    got = list(sc.range_stream_paged(b"a", b"b", 5, 1 << 20))
    assert got == list(sc.range_stream(b"a", b"b", 5))
    assert len(got) == 1 and got[0].err == str(err) and not got[0].more and got[0].revision == 5
