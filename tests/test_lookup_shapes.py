"""The lookup shapes (tests/lookup_shapes.py) reach the boundaries of the bound search, the point-read kernels and the
page cut they are built for, and the references the GPU tests compare with agree with each other: bisect over the keys
with the oracle's examined count, the C oracle's get with the pure-Python one.  The GPU tests in
tests/test_gpu_lookup_shapes.py can only fail on a wrong boundary if a shape puts something on it, so a change to a builder
that stops reaching a class fails here, on any host."""
from __future__ import annotations

import bisect

import pytest

from oracle import binding as ko
from tests import lookup_shapes as ls
from tests import pyref


@pytest.fixture(scope="module")
def classes():
    return ls.lookup_classes()


def test_s1_pivot_rounds(classes):
    for n in ls.S1_SIZES:
        c = classes["S1 n=%d" % n]
        assert c["equal"] and c["below_all"] and c["above_all"], n
        assert {("bound_prefix", len(ls.s1_key(0)) - 1, "byte"), ("record_prefix", len(ls.s1_key(0)), "nul")} <= c["prefix"]
        rounds = 1 + (n > 32) + (n > 32 * 33 + 32) + (n > 33**3 - 1)
        assert max(c["rounds"]) >= rounds, n
        if n > 32:
            assert "r1" in c["at_pivot"], n  # a bound equal to a first-round pivot
        if n >= 33 * 33:
            assert "r2" in c["at_pivot"], n
    for n in (32, 1088, 35936):  # a full final round: the answer may be taken by lane 31
        assert classes["S1 n=%d" % n]["last_lane"], n
    # 33^k records: a bound between two pivots ends one round early, one that is not takes the extra round
    assert {2, 3} <= classes["S1 n=1089"]["rounds"] and {3, 4} <= classes["S1 n=35937"]["rounds"]


def test_s1_large_store():
    keys = ls.s1_store(ls.S1_BIG).keys.tolist()
    c = ls.search_classes(keys, ls.s1_bounds(keys))
    assert c["equal"] and {"r1", "r2"} <= c["at_pivot"] and max(c["rounds"]) >= 4


def test_s2_compare_chunks(classes):
    c = classes["S2"]
    assert set(ls.DIFF_AT) <= c["diff_at"]
    assert {ls.PREFETCH * ls.CHUNK, ls.PREFETCH * ls.CHUNK - 1} <= c["diff_at"]  # first byte of the loop, last prefetched
    for m in ls.PREFIX_AT:
        for who in ("bound_prefix", "record_prefix"):
            for tail in ("byte", "nul"):
                assert (who, m, tail) in c["prefix"], (who, m, tail)
    assert c["max_bound"] == 65535 and c["equal"]


def test_bisect_agrees_with_the_oracle_examined():
    """lower_bound(b) is the examined count of the unlimited request [b"", b): what the GPU tests read k_search by"""
    shapes = [ls.s1_store(n) for n in (1, 33, 1089)]
    st2, b2 = ls.s2_shape()
    for store, bounds in [(s, ls.s1_bounds(s.keys.tolist())) for s in shapes] + [(st2, b2)]:
        keys = store.keys.tolist()
        ost = ko.OracleStore(store)
        for b in bounds:
            x = ko.range_(ost, b"", b, ls.ALL, 0)
            assert x.rc == 0 and x.examined == bisect.bisect_left(keys, b) == ost.lower_bound(b), b[:40]


def test_p1_resolve(classes):
    c = classes["P1"]
    for pre in ls.PRE_TARGETS:
        for ch in ls.NEAR_CHUNKS:
            p = ls._near_pos(pre, ch)
            if p <= pre - 2:  # (chunk 31 of a 511- or 512-byte prefix is its last)
                assert (pre, "last" if p // ls.CHUNK == (pre - 2) // ls.CHUNK else ch) in c["near"], (pre, ch)
    assert {0, 1} <= c["passes"]  # the first and the second 512-byte pass of k_get_resolve
    assert set(ls.PRE_TARGETS) <= c["found_pre"]
    for k in ("ext_dollar", "idx0", "idx_n", "rev_record", "top24", "bound_is_key"):
        assert c[k], k
    assert {"equal", "len8", "len10", *ls.TOMB_OFFSETS} <= c["tomb"]
    assert c["status"] == {"found", "not_found", "tombstone"}


def test_p2_finalize_chunks(classes):
    for n in ls.P2_SIZES:
        cl = {p: classes["P2 n=%d %s" % (n, p)] for p in ls.P2_PATTERNS}
        assert cl["none"]["found"] == 0 and cl["all"]["found"] == n
        assert cl["last"]["found"] == 1
        if n >= ls.FINALIZE_CHUNK:
            assert cl["edge255"]["at"] == {255} and cl["edge0"]["at"] == {0}
        if n > ls.FINALIZE_CHUNK:
            assert cl["all"]["carry"] and cl["edge0"]["carry"] and cl["last"]["carry"]
    assert {classes["P2 n=%d none" % n]["chunks"] for n in ls.P2_SIZES} >= {1, 2, 3, 256, 257}


def test_p2_wire_bodies_and_empty_values():
    store, found, _ = ls.p2_store()
    bodies, empty = set(), 0
    for k, v in zip(store.keys.tolist(), store.vals.tolist()):
        uk, rev = pyref.decode(k)
        if rev:
            b = ls.kv_body(len(uk), len(v), rev)
            assert ls.kvs_elem(len(uk), len(v), rev) == ko.wire_elem_size(len(uk), len(v), rev, ko.WIRE_KVS)
            bodies.add(b)
            empty += len(v) == 0
    assert set(ls.BODY_TARGETS) <= bodies and empty >= 10


def test_p2_one_record_element_exceeds_its_slab_bytes():
    store = ls.p2_one_store()
    k, v = store.keys[0], store.vals[0]
    slab = ls.pad16(len(k)) + ls.pad16(len(v))
    assert len(k) == 16 and len(v) == 16 and slab == 32
    el = ko.wire_elem_size(3, 16, ls.P2_ONE_REV, ko.WIRE_KVS)
    assert el > slab
    reads = [(b"abc", 0)] * 1000
    assert el * 1000 <= ls.get_arena_bound(reads, slab // 16, slab, True)


def test_oracle_get_agrees_with_pyref():
    st, reads = ls.p1_shape()
    s2, found, missing = ls.p2_store()
    for store, rs in ((st, reads), (s2, [(k, r) for k in found[:40] + found[-12:] + missing[:5] for r in (0, 1, 310)])):
        ost = ko.OracleStore(store)
        keys, vals = store.keys.tolist(), store.vals.tolist()
        for uk, rev in rs:
            assert ko.get(ost, uk, rev) == pyref.get(keys, vals, uk, rev), (uk[:40], rev)


def test_cut_search(classes):
    for n in ls.C_SIZES:
        c1 = classes["C n=%d group=1" % n]
        assert c1["pivot_round"] and c1["distinct"] and c1["candidates"] == n
    assert classes["C n=1057 group=7"]["pivot_round"] and classes["C n=1057 group=7"]["candidates"] == 151
    assert not classes["C n=33 group=7"]["pivot_round"]  # the final round alone, for contrast
    for n in ls.C_SIZES:  # the sweep deletes exactly n records
        store = ls.c_compact_store(n)
        x = ko.worker_run(ko.OracleStore(store), ls.MAGIC, b"\xff", 9, compact=True, collect=True)
        assert x.rc == 0 and len(x.victims) == n


def test_x_layouts(classes):
    assert classes["X1 exact"]["starts_at_line"] and classes["X1 exact"]["entry_at_line"] == 4096
    assert classes["X1 straddle"]["straddles"] and classes["X1 straddle"]["entry_at_line"] == 4095
    for name in ("X1 wire", "X2 raw", "X3 stream"):
        assert classes[name]["past"], name
    small = ls.x_store(64, n_objects=5)  # the large stores' layout, at a size any host can build
    assert small.n == 5 and all(small.vals[i][:1] == bytes([i]) and small.vals[i][-1:] == b"\xa5" for i in range(5))
