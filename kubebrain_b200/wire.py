"""etcd wire framing around the protobuf elements the device writes (KB_WIRE_ETCD_KVS / KB_WIRE_ETCD_EVENTS).

A protobuf message is the concatenation of its fields, so a response is  head | elements | tail  where only the few
head / tail bytes are produced on the host (kb_wire_range_head / _tail / kb_wire_watch_head of the C ABI).  Mirrors what
the reference's etcd-compatible server builds per kv on the CPU:
  List          -> etcdserverpb.RangeResponse   (pkg/server/etcd/backendshim.go:269-282)
  range stream  -> etcdserverpb.WatchResponse per 300-kv batch + a cancel message at the end
                   (backendshim.go:329-368; batches receiver.go:119-138; end marker scanner.go:179-192)
"""
from __future__ import annotations

import ctypes as C
from typing import Iterator, Optional

from ._lib import RangeResult, lib, u8p

RANGE_STREAM_BATCH = 300  # receiver.go:36 rangeStreamBatch


def _call(fn, *args, extra: int = 0) -> bytes:
    buf = (C.c_uint8 * (32 + extra))()
    n = fn(*args, C.cast(buf, u8p))
    return bytes(buf[: int(n)])


def range_head(header_rev: int) -> bytes:
    return _call(lib().kb_wire_range_head, header_rev)


def range_tail(more: bool, count: int) -> bytes:
    return _call(lib().kb_wire_range_tail, int(more), count)


def watch_head(header_rev: int, canceled: bool = False, reason: bytes = b"") -> bytes:
    return _call(lib().kb_wire_watch_head, header_rev, int(canceled), reason, len(reason), extra=len(reason) + 16)


def range_response(res: RangeResult, q: int, header_rev: int, more: bool) -> bytes:
    """the serialized etcdserverpb.RangeResponse of request q (count = len(kvs) + (1 if more), backendshim.go:269-277)"""
    n = int(res.req_first[q + 1] - res.req_first[q])
    return range_head(header_rev) + bytes(res.elements(q)) + range_tail(more, n + (1 if more else 0))


def list_response(eng, start: bytes, end: bytes, revision: int, limit: int, header_rev: int) -> bytes:
    """The serialized etcdserverpb.RangeResponse of a List with the USER's limit, as backend.List + backendShim.List build
    it: the scanner is asked for limit + 1 (pkg/backend/range.go:150-170), the first `limit` kvs are kept (the arena is cut
    at elem_off[limit]), More says whether one was dropped and Count = len(kvs) + (1 if More) (backendshim.go:269-277).
    start / end are internal keys."""
    from ._lib import KB_OUT_HOST, KB_WIRE_ETCD_KVS

    res = eng.range_batch([(start, end, revision, limit + 1 if limit > 0 else 0)], KB_OUT_HOST | KB_WIRE_ETCD_KVS)
    try:
        n = res.n_kvs
        more = limit > 0 and n > limit
        if more:
            n = limit
        body = bytes(res.elements(0, 0, n))
        return range_head(header_rev) + body + range_tail(more, n + (1 if more else 0))
    finally:
        res.close()


def get_response(eng, key: bytes, revision: int, current_rev: int) -> bytes:
    """The serialized etcdserverpb.RangeResponse of a Get, as backend.Get + backendShim.Get build it (range.go:45-72,
    backendshim.go:235-254): the kv element of the read when it is FOUND (an empty value is present too), nothing for a
    missing or deleted key; header revision = max(current_rev, mod_revision) when FOUND, else current_rev; Count = 1 or 0.
    key is the USER key; revision 0 reads the latest version."""
    from ._lib import GET_FOUND, KB_OUT_HOST, KB_WIRE_ETCD_KVS

    res = eng.get_submit([(key, revision)], KB_OUT_HOST | KB_WIRE_ETCD_KVS).collect()
    try:
        found = int(res.status[0]) == GET_FOUND
        head = max(current_rev, int(res.mod_rev[0])) if found else current_rev
        return range_head(head) + (res.element(0) if found else b"") + range_tail(False, 1 if found else 0)
    finally:
        res.close()


def stream_messages(res: RangeResult, q: int, revision: int, err: Optional[str] = None) -> Iterator[bytes]:
    """the serialized etcdserverpb.WatchResponse sequence of one range stream: batches of 300 events whose header
    revision is 0 (forked receivers never get readRev, receiver.go:162-166), then the cancel message carrying the read
    revision and, if the scan failed, the error text"""
    n = int(res.req_first[q + 1] - res.req_first[q])
    head0 = watch_head(0)
    for i in range(0, n, RANGE_STREAM_BATCH):
        yield head0 + bytes(res.elements(q, i, RANGE_STREAM_BATCH))
    yield watch_head(revision, True, (err or "").encode())
