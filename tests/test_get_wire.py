"""wire.get_response (the serialized RangeResponse of backendShim.Get, backendshim.go:235-254 + range.go:45-72) against the
protobuf runtime on the restated etcd v3.5.2 schema (tests/golden/etcd_schema.py).  CPU only: a stand-in for the
collected point-read result carries the element bytes the device writes (the oracle's encoder makes them); the device
answer itself is compared with the oracle in tests/test_gpu_get_pipeline.py."""
from __future__ import annotations

import struct

import pytest

from kubebrain_b200 import wire
from kubebrain_b200._lib import GET_FOUND, GET_NOT_FOUND, GET_TOMBSTONE, KB_OUT_HOST, KB_WIRE_ETCD_KVS
from kubebrain_b200.packed import PackedStore
from oracle import binding as ko

MAGIC = b"\x57\xfb\x80\x8b"


class _Result:
    """what GetResult offers get_response: per-read status / mod_rev and the element of a FOUND read"""

    def __init__(self, status, mod_rev, elem):
        self.status, self.mod_rev, self._elem, self.closed = [status], [mod_rev], elem, False

    def element(self, i):
        assert self.status[i] == GET_FOUND
        return self._elem

    def close(self):
        self.closed = True


class _Engine:
    def __init__(self, res):
        self.res, self.calls = res, []

    def get_submit(self, reqs, out_mode):
        self.calls.append((list(reqs), out_mode))
        return self

    def collect(self):
        return self.res


def _element(key: bytes, val: bytes, rev: int) -> bytes:
    st = ko.OracleStore(PackedStore.from_items([(MAGIC + key + b"$" + struct.pack(">Q", rev), val)]))
    el, off = ko.wire_encode(st, [0], ko.WIRE_KVS)
    assert int(off[1]) == len(el)
    return el


@pytest.mark.parametrize("case", ["found", "found_above_current", "found_empty_value", "tombstone", "missing"])
def test_get_response_framing(case):
    pytest.importorskip("google.protobuf")
    from tests.golden import etcd_schema as es

    M = es.build()
    key, cur = b"/registry/pods/ns-1/p", 1700000010
    if case == "tombstone":
        res, kvs = _Result(GET_TOMBSTONE, cur + 5, b""), []
    elif case == "missing":
        res, kvs = _Result(GET_NOT_FOUND, 0, b""), []
    else:
        val = b"" if case == "found_empty_value" else b"\x00value" * 40
        rev = cur + 7 if case == "found_above_current" else cur - 3
        res, kvs = _Result(GET_FOUND, rev, _element(key, val, rev)), [(key, val, rev)]
    eng = _Engine(res)
    got = wire.get_response(eng, key, 0, cur)
    head = max(cur, kvs[0][2]) if kvs else cur  # a missing or deleted key answers with the current revision
    assert got == es.range_response(M, head, kvs, False, len(kvs))
    assert eng.calls == [([(key, 0)], KB_OUT_HOST | KB_WIRE_ETCD_KVS)] and res.closed
