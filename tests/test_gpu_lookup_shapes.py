"""The bound search, the point reads and the page cut (kb_search.cu: k_search / key_less; kb_scan.cu: k_get_resolve /
k_get_finalize, k_page_cut) against plain references on the lookup shapes (tests/lookup_shapes.py;
tests/test_lookup_shapes.py asserts which classes each shape reaches), and answers past 4 GiB.

  S  k_search's lower bound, read exactly from the ABI: the unlimited request [b"", b) in KB_OUT_COUNT mode examines
     lower_bound(b) records; compared with bisect over the keys as Python bytes.
  P  every point read against the oracle's get in all four out modes (check() of tests/test_gpu_get_pipeline.py).
  C  the first page of a range stream and of a compaction stream at a budget of exactly every cut, and one byte less,
     against the greedy cut of tests/test_gpu_range_stream.py.
  X  one range batch, one point-read batch and one range stream whose arena offsets cross 2^32: every per-kv array and
     the whole arena, read back in windows of 256 MiB."""
from __future__ import annotations

import bisect
import ctypes as C
import resource

import numpy as np
import pytest

from kubebrain_b200._lib import (GET_FOUND, KB_OUT_COUNT, KB_OUT_DEVICE, KB_OUT_HOST, KB_WIRE_ETCD_EVENTS,
                                 KB_WIRE_ETCD_KVS, Engine, _cudart)
from kubebrain_b200.packed import PackedStore
from oracle import binding as ko
from tests import lookup_shapes as ls
from tests import test_gpu_compact_stream as gcs
from tests.test_gpu_get_pipeline import MODES, _all_modes, check
from tests.test_gpu_range_stream import check_stream, expected as stream_expected

pytestmark = pytest.mark.gpu

ALL = ls.ALL
WINDOW = 256 << 20


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


# ---- S: bound search ------------------------------------------------------------------------------------------------
def lower_bounds(eng: Engine, keys, bounds, cap: int = 1 << 26):
    """k_search's answer for every bound (the examined count of [b"", b)) and bisect's, in batches of at most `cap`
    examined records"""
    exp = [bisect.bisect_left(keys, b) for b in bounds]
    got, i = [], 0
    while i < len(bounds):
        j, load = i, 0
        while j < len(bounds) and (j == i or load + exp[j] <= cap):
            load += exp[j]
            j += 1
        res = eng.range_batch([(b"", b, ALL, 0) for b in bounds[i:j]], KB_OUT_COUNT)
        got += res.req_examined.tolist()
        res.close()
        i = j
    return got, exp


def assert_search(eng, store: PackedStore, bounds, what):
    keys = store.keys.tolist()
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    got, exp = lower_bounds(eng, keys, bounds)
    bad = [(i, bounds[i][-12:], g, x) for i, (g, x) in enumerate(zip(got, exp)) if g != x]
    assert not bad, (what, len(bad), bad[:5])


@pytest.mark.parametrize("n", ls.S1_SIZES + (ls.S1_BIG,))
def test_s1_pivots(eng, n):
    store = ls.s1_store(n)
    keys = store.keys.tolist()
    bounds = ls.s1_bounds(keys)
    assert_search(eng, store, bounds, n)
    # the ABI reading once against the oracle's examined count
    st = ko.OracleStore(store)
    for b in bounds[:: max(1, len(bounds) // 50)]:
        res = eng.range_batch([(b"", b, ALL, 0)], KB_OUT_COUNT)
        assert int(res.req_examined[0]) == ko.range_(st, b"", b, ALL, 0).examined, b[-12:]
        res.close()


def test_s1_emptied_store(eng):
    """every record deleted by a write: the search runs on an empty directory"""
    store = ls.s1_store(40)
    eng.load_sorted(store)
    eng.apply_batch([(k, None) for k in store.keys.tolist()])
    bounds = ls.s1_bounds(store.keys.tolist())
    res = eng.range_batch([(b"", b, ALL, 0) for b in bounds], KB_OUT_COUNT)
    assert res.req_examined.tolist() == [0] * len(bounds)
    res.close()


def test_s2_compare_chunks(eng):
    store, bounds = ls.s2_shape()
    assert_search(eng, store, bounds, "S2")
    # the same bounds as range starts over a store of the records around them
    st = ko.OracleStore(store)
    for b in bounds[::7]:
        res = eng.range_batch([(b, b"\xff", ALL, 0)], KB_OUT_COUNT)
        assert int(res.req_examined[0]) == ko.range_(st, b, b"\xff", ALL, 0).examined
        res.close()


# ---- P: point reads -------------------------------------------------------------------------------------------------
def test_p1_resolve(eng):
    store, reads = ls.p1_shape()
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    _all_modes(eng, store, st, reads)
    # tombstones (and near misses) written as new values: the value sits behind the loaded slab, at a non-zero voff16
    items = dict(zip(store.keys.tolist(), store.vals.tolist()))
    tk = [k for k in items if k.startswith(ls.MAGIC + b"/p1/tomb/")]
    ops = [(tk[0], ls.TOMB + b"\x00"), (tk[1], ls.TOMB), (tk[2], b"tombstonf"), (ls.ik(b"/p1/tomb/new", 9), ls.TOMB),
           (ls.ik(b"/p1/tomb/new2", 9), b"uombstone")]
    eng.apply_batch(ops)
    items.update(ops)
    cur = PackedStore.from_items(list(items.items()))
    reads2 = reads + [(b"/p1/tomb/new", 0), (b"/p1/tomb/new", 9), (b"/p1/tomb/new2", 0)]
    _all_modes(eng, cur, ko.OracleStore(cur), reads2)


@pytest.fixture(scope="module")
def p2():
    store, found, missing = ls.p2_store()
    return store, ko.OracleStore(store), found, missing


@pytest.mark.parametrize("n", ls.P2_SIZES)
def test_p2_finalize_chunks(eng, p2, n):
    store, st, found, missing = p2
    eng.load_sorted(store)
    for pat in ls.P2_PATTERNS:
        reads = ls.p2_reads(n, pat, found, missing)
        if n <= 513:
            _all_modes(eng, store, st, reads)
        else:
            for mode in MODES:
                check(eng, eng.get_submit(reads, mode).collect(), store, st, reads, mode)


def test_p2_one_record_read_many_times(eng):
    store = ls.p2_one_store()
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    slab = ls.pad16(len(store.keys[0])) + ls.pad16(len(store.vals[0]))
    for n in (1, 257, 5000):
        reads = [(b"abc", 0)] * n
        for mode in MODES:
            res = eng.get_submit(reads, mode).collect()
            bound = ls.get_arena_bound(reads, slab // 16, slab, bool(mode & KB_WIRE_ETCD_KVS))
            assert res.n_bytes <= bound, (n, mode, res.n_bytes, bound)
            check(eng, res, store, st, reads, mode)


# ---- C: page cut ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", ls.C_SIZES)
@pytest.mark.parametrize("group", ls.C_GROUPS)
def test_c_range_stream_every_cut(eng, n, group):
    store = ls.c_range_store(n)
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    s, e = ls.MAGIC, b"\xff"
    _, _, sizes = stream_expected(store, st, s, e, ALL, KB_OUT_HOST)
    assert len(sizes) == n
    pre = np.concatenate([[0], np.cumsum(sizes)])
    for k in range(1, ls.cut_candidates(n, group) + 1):
        b = min(k * group, n)
        for budget in (int(pre[b]), int(pre[b]) - 1):
            cuts = check_stream(eng, store, st, s, e, ALL, KB_OUT_HOST, group, budget, what=(n, group, b, budget))
            assert cuts[0][1] == (b if budget == pre[b] or k == 1 else (k - 1) * group), (n, group, b, budget)
    for m in (KB_OUT_DEVICE, KB_OUT_HOST | KB_WIRE_ETCD_KVS, KB_OUT_DEVICE | KB_WIRE_ETCD_EVENTS):
        _, _, wsizes = stream_expected(store, st, s, e, ALL, m)
        wpre = np.concatenate([[0], np.cumsum(wsizes)])
        g = ls.cut_candidates(n, group)
        for k in sorted({1, 2, 17, 31, 32, 33, g} & set(range(1, g + 1))):
            b = min(k * group, n)
            check_stream(eng, store, st, s, e, ALL, m, group, int(wpre[b]), what=(n, group, b, m))


@pytest.mark.parametrize("n", ls.C_SIZES)
@pytest.mark.parametrize("group", ls.C_GROUPS)
def test_c_compact_stream_every_cut(eng, n, group):
    store = ls.c_compact_store(n)
    eng.load_sorted(store)
    x = gcs.Expected(store, ls.MAGIC, b"\xff", 9)
    assert len(x.rec) == n
    pre = np.concatenate([[0], np.cumsum(x.sizes)])
    for k in range(1, ls.cut_candidates(n, group) + 1):
        b = min(k * group, n)
        for budget in (int(pre[b]), int(pre[b]) - 1):
            stream = eng.compact_stream(ls.MAGIC, b"\xff", 9, 0, True, group)
            page = stream.next(budget)
            stream.close()
            eng.set_compact_revision(None)
            want = b if budget == pre[b] or k == 1 else (k - 1) * group
            assert want == gcs.greedy_cuts(x.sizes, group, budget)[0][1]
            assert (page.first, page.n) == (0, want), (n, group, b, budget)
            assert page.rec_idx.astype(np.int64).tolist() == x.rec[:want].tolist(), (n, group, b)
            assert page.keys() == x.keys[:want] and page.n_bytes == int(pre[want]), (n, group, b)
            assert page.arena.tobytes() == b"".join(x.entry(i) for i in range(want)), (n, group, b)
    gcs.check_stream(eng, store, ls.MAGIC, b"\xff", 9, group, int(pre[min(group, n)]), what=(n, group))


# ---- X: answers past 4 GiB -------------------------------------------------------------------------------------------
def tiled(unit: np.ndarray, start: int, n: int) -> np.ndarray:
    """bytes [start, start + n) of `unit` repeated without end"""
    s = start % len(unit)
    return np.tile(unit, (s + n + len(unit) - 1) // len(unit))[s: s + n]


def check_arena(eng: Engine, host: np.ndarray, dev_ptr: int, total: int, unit: np.ndarray, what):
    """the whole arena against `unit` tiled, in windows of at most 256 MiB (read back from HBM for KB_OUT_DEVICE)"""
    assert total == ls.X_N * len(unit), what
    for w0 in range(0, total, WINDOW):
        n = min(WINDOW, total - w0)
        got = host[w0: w0 + n] if host is not None else np.frombuffer(eng.read_device(dev_ptr + w0, n, sync=False),
                                                                     np.uint8)
        assert np.array_equal(got, tiled(unit, w0, n)), (what, w0)


def mem_used() -> dict:
    free, total = C.c_size_t(), C.c_size_t()
    _cudart().cudaMemGetInfo(C.byref(free), C.byref(total))
    return dict(device_used=total.value - free.value, host_peak_rss=resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024)


def report(what: str, before: dict):
    after = mem_used()
    print("X-MEM %s device_used_delta=%.2f GB host_peak_rss=%.2f GB" % (
        what, (after["device_used"] - before["device_used"]) / 1e9, after["host_peak_rss"] / 1e9))


def _arr(res, name, dtype):
    return res.device_array(name, dtype) if res.on_device else getattr(res, name)


def _element(st, mode) -> np.ndarray:
    el, off = ko.wire_encode(st, [0], ko.WIRE_KVS if mode & KB_WIRE_ETCD_KVS else ko.WIRE_EVENTS)
    return np.frombuffer(el, np.uint8)


X1_MODES = {"host": KB_OUT_HOST, "device": KB_OUT_DEVICE, "kvs": KB_OUT_HOST | KB_WIRE_ETCD_KVS,
            "events": KB_OUT_DEVICE | KB_WIRE_ETCD_EVENTS}


@pytest.mark.parametrize("vl", [ls.X_VAL_EXACT, ls.X_VAL_STRADDLE], ids=["exact", "straddle"])
def test_x1_range_batch_past_4gib(eng, vl):
    store = ls.x_store(vl)
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    x = ko.range_(st, ls.MAGIC, b"\xff", ALL, 0)
    assert x.emit.tolist() == [0]
    key, val = store.keys[0], store.vals[0]
    reqs = [(ls.MAGIC, b"\xff", ALL, 0)] * ls.X_N
    k = np.arange(ls.X_N, dtype=np.uint64)
    for name, mode in X1_MODES.items():
        before = mem_used()
        res = eng.range_batch(reqs, mode)
        what = (vl, name)
        assert res.req_first.tolist() == list(range(ls.X_N + 1)) and res.req_count.tolist() == [1] * ls.X_N, what
        assert res.req_examined.tolist() == [x.examined] * ls.X_N, what
        assert _arr(res, "rec_idx", np.uint32).tolist() == np.tile(x.emit, ls.X_N).tolist(), what
        assert (_arr(res, "rev", np.uint64) == ls.X_REV).all() and (_arr(res, "val_len", np.uint32) == vl).all(), what
        assert (_arr(res, "key_len", np.uint32) == len(ls.X_KEY)).all(), what
        if mode & (KB_WIRE_ETCD_KVS | KB_WIRE_ETCD_EVENTS):
            unit = _element(st, mode)
            L = len(unit)
            n1 = bytes(unit).find(b"\x0a\x03" + ls.X_KEY) + 2
            eo = _arr(res, "elem_off", np.uint64)
            assert eo.tolist() == (np.arange(ls.X_N + 1, dtype=np.uint64) * np.uint64(L)).tolist(), what
            assert _arr(res, "key_off", np.uint64).tolist() == (k * np.uint64(L) + np.uint64(n1)).tolist(), what
            assert _arr(res, "val_off", np.uint64).tolist() == (k * np.uint64(L) + np.uint64(L - vl)).tolist(), what
        else:
            unit = ls.x_pair(key, val)
            P = np.uint64(len(unit))
            assert _arr(res, "key_off", np.uint64).tolist() == (k * P + np.uint64(4)).tolist(), what
            assert _arr(res, "val_off", np.uint64).tolist() == (k * P + np.uint64(ls.pad16(len(key)))).tolist(), what
        assert res.n_bytes > ls.X_LINE, what
        check_arena(eng, res.arena, res.bytes_ptr if res.on_device else 0, res.n_bytes, unit, what)
        report("X1 %s %s" % ("exact" if vl == ls.X_VAL_EXACT else "straddle", name), before)
        res.close()


def test_x2_point_reads_past_4gib(eng):
    store = ls.x_store(ls.X_VAL_EXACT)
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    idx, mod = ko.get(st, ls.X_KEY, 0)
    assert idx == 0 and mod == ls.X_REV
    vl = ls.X_VAL_EXACT
    reads = [(ls.X_KEY, 0)] * ls.X_N
    i = np.arange(ls.X_N, dtype=np.uint64)
    for name, mode in (("host", KB_OUT_HOST), ("kvs device", KB_OUT_DEVICE | KB_WIRE_ETCD_KVS)):
        before = mem_used()
        res = eng.get_submit(reads, mode).collect()
        what = name
        assert (res.status == GET_FOUND).all() and (res.mod_rev == mod).all() and (res.rec_idx == idx).all(), what
        assert (res.val_len == vl).all(), what
        if mode & KB_WIRE_ETCD_KVS:
            unit = _element(st, mode)
            L = np.uint64(len(unit))
            assert res.elem_off.tolist() == (np.arange(ls.X_N + 1, dtype=np.uint64) * L).tolist(), what
            assert res.val_off.tolist() == (i * L + L - np.uint64(vl)).tolist(), what
        else:
            unit = np.frombuffer(store.vals[0] + b"\x00" * (ls.pad16(vl) - vl), np.uint8)
            assert res.val_off.tolist() == (i * np.uint64(len(unit))).tolist(), what
        assert res.n_bytes == ls.X_N * len(unit) > ls.X_LINE, what
        check_arena(eng, res.arena, res.bytes_ptr if res.on_device else 0, res.n_bytes, unit, what)
        report("X2 %s" % name, before)
        res.close()


@pytest.mark.parametrize("mode", [KB_OUT_HOST, KB_OUT_DEVICE], ids=["host", "device"])
def test_x3_range_stream_past_4gib(eng, mode):
    vl = ls.X_VAL_EXACT
    store = ls.x_store(vl, n_objects=ls.X_N)
    st = ko.OracleStore(store)
    before = mem_used()
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    x = ko.range_(st, ls.MAGIC, b"\xff", ALL, 0)
    emit = x.emit.astype(np.int64)
    assert len(emit) == ls.X_N
    keys = np.frombuffer(b"".join(store.keys.tolist()), np.uint8).reshape(ls.X_N, 16)
    vals = store.vals.data.reshape(ls.X_N, vl)
    P = 16 + vl
    stream = eng.range_stream((ls.MAGIC, b"\xff", ALL, 0), mode, 1)
    a, total = 0, 0
    while True:
        page = stream.next(ls.X_PAGE)
        if page is None:
            break
        m = page.n_kvs
        assert m == min(ls.X_PAGE // P, ls.X_N - a) and page.n_bytes == m * P, (a, m)
        rec = _arr(page, "rec_idx", np.uint32).astype(np.int64)
        assert rec.tolist() == emit[a: a + m].tolist(), a
        j = np.arange(m, dtype=np.uint64)
        assert _arr(page, "key_off", np.uint64).tolist() == (j * np.uint64(P) + np.uint64(4)).tolist(), a
        assert _arr(page, "val_off", np.uint64).tolist() == (j * np.uint64(P) + np.uint64(16)).tolist(), a
        img = np.empty((m, P), np.uint8)
        img[:, :16] = keys[emit[a: a + m]]
        img[:, 16:] = vals[emit[a: a + m]]
        got = (np.frombuffer(eng.read_device(page.bytes_ptr, page.n_bytes, sync=False), np.uint8) if page.on_device
               else page.arena[: page.n_bytes])
        assert np.array_equal(got, img.reshape(-1)), a
        a += m
        total += page.n_bytes
        page.close()
    stream.close()
    assert a == ls.X_N and total == ls.X_N * P > ls.X_LINE
    report("X3 %s" % ("host" if mode == KB_OUT_HOST else "device"), before)
