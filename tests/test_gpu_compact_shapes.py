"""The compaction sweep and the compaction stream (kb_decode.cuh k_decode_lcp's sweep flags; kb_scan.cu k_emit<true>,
k_tile_scan, k_place_victims; kb_compact.cu k_victim_capture, k_victim_jobs) against the C oracle on the compaction shapes
(tests/compact_shapes.py; tests/test_compact_shapes.py asserts which classes each shape reaches).

  sweeps   every sweep's ordered (record, class) list, count and examined in KB_OUT_HOST, KB_OUT_DEVICE (read back through
           kb_compact_view_get's pointers) and KB_OUT_COUNT, exactly;
  streams  every page's records, classes, keys, guards, offsets, lengths and whole arena against the greedy cut
           (check_pages of tests/test_gpu_compact_stream.py), and past 4 GiB every per-victim array and every arena byte,
           256 MiB at a time."""
from __future__ import annotations

import ctypes as C
import gc

import numpy as np
import pytest

from kubebrain_b200 import _lib
from kubebrain_b200._lib import KB_OUT_COUNT, KB_OUT_DEVICE, KB_OUT_HOST, Engine
from oracle import binding as ko
from tests import compact_shapes as cs
from tests import test_gpu_compact_stream as gcs
from tests.test_gpu_lookup_shapes import mem_used

pytestmark = pytest.mark.gpu

ALL = cs.ALL
MODES = {"host": KB_OUT_HOST, "device": KB_OUT_DEVICE, "count": KB_OUT_COUNT}


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def _same(got: np.ndarray, want: np.ndarray, what):
    got, want = got.astype(np.int64), want.astype(np.int64)
    if len(got) != len(want) or not np.array_equal(got, want):
        m = min(len(got), len(want))
        bad = np.nonzero(got[:m] != want[:m])[0]
        i = int(bad[0]) if len(bad) else m
        raise AssertionError((what, "lengths", len(got), len(want), "first difference", i,
                              got[max(0, i - 2): i + 3].tolist(), want[max(0, i - 2): i + 3].tolist()))


def check_sweep(eng: Engine, st, s: bytes, e: bytes, rev: int, timeout_rev: int = 0, support_ttl: bool = True,
                what=None):
    """kb_compact_sweep in every out mode against the oracle's worker_run; returns the oracle's answer"""
    x = ko.worker_run(st, s, e, rev, compact=True, timeout_rev=timeout_rev, support_ttl=support_ttl, collect=True)
    assert x.rc == 0, what
    for name, mode in MODES.items():
        got = eng.compact_sweep(s, e, rev, timeout_rev, support_ttl, mode)
        w = (what, name)
        assert (got.n_victims, got.count, got.examined) == (len(x.victims), x.count, x.examined), w
        if mode == KB_OUT_HOST:
            _same(got.victim_idx, x.victims, w)
            _same(got.victim_class, x.vclass, w)
        elif mode == KB_OUT_DEVICE:
            _same(got.device_array("victim_idx"), x.victims, w)
            _same(got.device_array("victim_class"), x.vclass, w)
        else:
            assert got.victim_idx.size == 0 and not got.dev_ptrs, w
        got.close()
    eng.set_compact_revision(None)
    return x


def loaded(eng: Engine, store):
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    return ko.OracleStore(store)


# ---- K1: classes and their order within a record -----------------------------------------------------------------
def test_k1_classes(eng):
    store = cs.k1_store()
    st = loaded(eng, store)
    seen = set()
    for q in cs.k1_sweeps():
        x = check_sweep(eng, st, *q, what=q)
        seen |= set(x.vclass.tolist())
    assert seen == {1, 2, 3, 4, 5}


@pytest.mark.parametrize("group", [1, 7])
def test_k1_streams(eng, group):
    store = cs.k1_store()
    eng.load_sorted(store)
    for s, e, rev, trev, ttl in cs.k1_sweeps():
        x = gcs.Expected(store, s, e, rev, trev, ttl)
        for budget in gcs.budgets(x.sizes, group):
            gcs.check_stream(eng, store, s, e, rev, group, budget, trev, ttl, (s[4:20], rev, trev, budget))


def test_k1_none_and_every(eng):
    store = cs.k1_none_store()
    st = loaded(eng, store)
    assert len(check_sweep(eng, st, cs.MAGIC, b"\xff", ALL, what="none").victims) == 0
    store = cs.k1_every_store()
    st = loaded(eng, store)
    x = check_sweep(eng, st, cs.MAGIC, b"\xff", ALL, what="every")
    assert sorted(set(x.victims.tolist())) == list(range(store.n))
    gcs.check_stream(eng, store, cs.MAGIC, b"\xff", ALL, 7, 4096, what="every")


# ---- K2: slots and tiles ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("start", cs.K2_STARTS)
def test_k2_tiles(eng, start):
    store = cs.k2_tiles_store()
    st = loaded(eng, store)
    check_sweep(eng, st, store.keys[start], b"\xff", ALL, what=start)
    gcs.check_stream(eng, store, store.keys[start], b"\xff", ALL, 1024, 64 << 10, what=start)


@pytest.mark.parametrize("n", cs.K2_CHAIN_N)
def test_k2_chain_2n_minus_1(eng, n):
    store = cs.chain_store(n)
    st = loaded(eng, store)
    x = check_sweep(eng, st, cs.MAGIC, b"\xff", ALL, what=n)
    assert len(x.victims) == 2 * n - 1
    if n <= 1025:
        gcs.check_stream(eng, store, cs.MAGIC, b"\xff", ALL, 1024, ALL, what=n)


@pytest.mark.parametrize("n", cs.K2_FULL_N)
def test_k2_every_record_two_calls(eng, n):
    store = cs.full_store(n)
    st = loaded(eng, store)
    assert len(check_sweep(eng, st, cs.MAGIC, b"\xff", ALL, what=n).victims) == 2 * n
    assert len(check_sweep(eng, st, cs.MAGIC, b"\xff", cs.T_TOMB - 1, what=n).victims) == n


@pytest.fixture(scope="module")
def big():
    store = cs.big_store()
    return store, ko.OracleStore(store)


def check_stream_vec(eng: Engine, store, x, s: bytes, e: bytes, rev: int, budget: int, group: int = 1024):
    """a stream's pages against the oracle's victims, every array and arena byte compared with numpy"""
    koff, kd = store.keys.off.astype(np.int64), store.keys.data
    voff, vd = store.vals.off.astype(np.int64), store.vals.data
    stream = eng.compact_stream(s, e, rev, 0, True, group)
    assert (stream.n_victims, stream.count, stream.examined) == (len(x.victims), x.count, x.examined)
    pos = 0
    while True:
        p = stream.next(budget)
        if p is None:
            break
        assert p.first == pos and (p.n % group == 0 or pos + p.n == len(x.victims))
        rec = x.victims[pos: pos + p.n].astype(np.int64)
        cls = x.vclass[pos: pos + p.n]
        _same(p.rec_idx, rec, pos)
        _same(p.victim_class, cls, pos)
        klen = koff[rec + 1] - koff[rec]
        glen = np.where(np.isin(cls, gcs.GUARDED), voff[rec + 1] - voff[rec], 0)
        _same(p.key_len, klen, pos)
        _same(p.guard_len, glen, pos)
        kp, gp = (klen + 15) & ~15, (glen + 15) & ~15
        start = np.concatenate([[0], np.cumsum(kp + gp)[:-1]])
        _same(p.key_off, start, pos)
        _same(p.guard_off, start + kp, pos)
        img = np.zeros(int((kp + gp).sum()), np.uint8)
        img[gcs._ranges(start, klen)] = kd[gcs._ranges(koff[rec], klen)]
        img[gcs._ranges(start + kp, glen)] = vd[gcs._ranges(voff[rec], glen)]
        assert p.n_bytes == len(img) and np.array_equal(p.arena, img), pos
        pos += p.n
    assert pos == len(x.victims)
    stream.close()
    eng.set_compact_revision(None)


@pytest.mark.parametrize("start", cs.K2_STARTS)
def test_k2_one_sweep_across_the_tile_scan_chunk(eng, big, start):
    store, st = big
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    s = store.keys[start]
    x = check_sweep(eng, st, s, b"\xff", ALL, what=start)
    assert x.examined > cs.TILE * cs.SCAN_CHUNK
    if start in (0, 1023):
        check_stream_vec(eng, store, x, s, b"\xff", ALL, 16 << 20)


# ---- K3: revision and TTL comparisons --------------------------------------------------------------------------------
def test_k3_comparisons(eng):
    store = cs.k3_store()
    st = loaded(eng, store)
    for q in cs.k3_sweeps():
        check_sweep(eng, st, *q, what=q)


@pytest.mark.parametrize("start", [0, 1])
def test_k3_expired_runs_on_tile_seams(eng, start):
    store = cs.k3_seam_store()
    st = loaded(eng, store)
    s = store.keys[start]
    for trev, ttl in ((cs.K3_SEAM_TIMEOUT, False), (cs.K3_SEAM_TIMEOUT, True), (1024, False), (0, True)):
        check_sweep(eng, st, s, b"\xff", ALL - 1, trev, ttl, what=(start, trev, ttl))
    gcs.check_stream(eng, store, s, b"\xff", ALL - 1, 1024, 32 << 10, cs.K3_SEAM_TIMEOUT, False, what=start)


# ---- K4: capture and pages -------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def k4():
    store = cs.k4_count_store()
    return store, ko.OracleStore(store)


@pytest.mark.parametrize("v", cs.K4_COUNTS)
def test_k4_capture_counts(eng, k4, v):
    store, st = k4
    eng.load_sorted(store)
    e = cs.k4_count_end(store, v)
    x = check_sweep(eng, st, cs.MAGIC, e, ALL, what=v)
    assert len(x.victims) == v
    for group, budget in ((1024, ALL), (1024, 1 << 18), (7, ALL)):
        gcs.check_stream(eng, store, cs.MAGIC, e, ALL, group, budget, what=(v, group, budget))
    if v <= 1025:
        gcs.check_stream(eng, store, cs.MAGIC, e, ALL, 1, 4096, what=(v, 1))


@pytest.mark.parametrize("group", cs.K4_GROUPS)
def test_k4_entries(eng, group):
    store = cs.k4_entry_store()
    st = loaded(eng, store)
    for s, e, rev, trev, ttl in cs.k4_entry_sweeps():
        check_sweep(eng, st, s, e, rev, trev, ttl, what=(trev, group))
        x = gcs.Expected(store, s, e, rev, trev, ttl)
        pre = np.concatenate([[0], np.cumsum(x.sizes)])
        cuts = sorted({int(pre[min(k * group, len(x.sizes))]) for k in range(1, 4)})
        for budget in sorted(set(gcs.budgets(x.sizes, group) + cuts + [c - 1 for c in cuts])):
            gcs.check_stream(eng, store, s, e, rev, group, budget, trev, ttl, (trev, group, budget))


# ---- K5: past 4 GiB --------------------------------------------------------------------------------------------------
def check_k5_page(x, glen: int, a: int, n: int, rec, cls, key_off, key_len, guard_off, guard_len, arena, n_bytes):
    unit = cs.pad16(cs.K5_KEY) + cs.pad16(glen)
    j = np.arange(n, dtype=np.uint64)
    what = (glen, a)
    _same(rec, x.victims[a: a + n], what)
    assert (cls == 4).all() and (key_len == cs.K5_KEY).all() and (guard_len == glen).all(), what
    _same(key_off, j * np.uint64(unit), what)
    _same(guard_off, j * np.uint64(unit) + np.uint64(cs.pad16(cs.K5_KEY)), what)
    assert n_bytes == n * unit, what
    keys = np.frombuffer(b"".join(cs.k5_key(int(i)) for i in x.victims[a: a + n]), np.uint8).reshape(n, cs.K5_KEY)
    ids = np.arange(a, a + n, dtype=np.uint32).view(np.uint8).reshape(n, 4)
    head = np.frombuffer(cs.be(cs.K5_VREV), np.uint8)
    g0 = cs.pad16(cs.K5_KEY)
    for r0 in range(0, n, 256):  # 256 entries (256 MiB) at a time
        r1 = min(n, r0 + 256)
        m = arena[r0 * unit: r1 * unit].reshape(r1 - r0, unit)
        w = (what, r0)
        assert np.array_equal(m[:, : cs.K5_KEY], keys[r0:r1]) and not m[:, cs.K5_KEY: g0].any(), w
        assert (m[:, g0: g0 + 8] == head).all() and np.array_equal(m[:, g0 + 8: g0 + 12], ids[r0:r1]), w
        assert (m[:, g0 + 12] == 0x5A).all() and (m[:, -1] == 0xA5).all() and not m[:, g0 + 13: -1].any(), w


@pytest.mark.parametrize("glen", [cs.K5_GUARD_EXACT, cs.K5_GUARD_STRADDLE], ids=["exact", "straddle"])
def test_k5_stream_past_4gib(glen):
    lay = cs.k5_layout(glen)
    assert lay["past"] and (lay["starts_at_line"] or lay["guard_straddles"])
    before = mem_used()
    eng = Engine(0)  # its own: closing it releases the 4.3 GB page buffers the engine pools
    try:
        _k5(eng, glen, lay, before)
    finally:
        eng.close()


def _k5(eng: Engine, glen: int, lay, before):
    store = cs.k5_store(glen)
    x = ko.worker_run(ko.OracleStore(store), cs.MAGIC, b"\xff", cs.K5_REV, compact=True, timeout_rev=cs.K5_TIMEOUT,
                      support_ttl=False, collect=True)
    assert x.rc == 0 and x.victims.tolist() == list(range(cs.K5_N)) and (x.vclass == 4).all()
    eng.load_sorted(store)
    del store
    gc.collect()
    args = (cs.MAGIC, b"\xff", cs.K5_REV, cs.K5_TIMEOUT, False)
    # pages of 256 MiB, one victim per group
    stream = eng.compact_stream(*args, 1)
    assert (stream.n_victims, stream.count, stream.examined) == (cs.K5_N, x.count, x.examined)
    a = 0
    while True:
        p = stream.next(cs.K5_PAGE)
        if p is None:
            break
        assert p.first == a and p.n == min(cs.K5_PAGE // lay["unit"], cs.K5_N - a), a
        check_k5_page(x, glen, a, p.n, p.rec_idx, p.victim_class, p.key_off, p.key_len, p.guard_off, p.guard_len,
                      p.arena, p.n_bytes)
        a += p.n
        del p
    assert a == cs.K5_N
    stream.close()
    # one page of everything (read in place: the page is not copied out of the library's host arena)
    stream = eng.compact_stream(*args, 1024)
    r = C.c_void_p()
    eng._check(_lib.lib().kb_compact_stream_next(eng._ctx, stream._h, ALL, C.byref(r)))
    try:
        v = _lib.KbCompactPageView()
        eng._check(_lib.lib().kb_compact_page_view_get(r, C.byref(v)))
        n = int(v.n)
        assert (int(v.first), n, int(v.n_bytes)) == (0, cs.K5_N, lay["total"]) and lay["total"] > cs.LINE

        def arr(p, dtype):
            return _lib._np(p, n, dtype)

        check_k5_page(x, glen, 0, n, arr(v.rec_idx, np.uint32), arr(v.victim_class, np.uint8),
                      arr(v.key_off, np.uint64), arr(v.key_len, np.uint32), arr(v.guard_off, np.uint64),
                      arr(v.guard_len, np.uint32), _lib._np(v.bytes, int(v.n_bytes), np.uint8), int(v.n_bytes))
    finally:
        _lib.lib().kb_result_free(eng._ctx, r)
    assert stream.next(ALL) is None
    stream.close()
    after = mem_used()
    print("K5-MEM %s device_used_delta=%.2f GB host_peak_rss=%.2f GB" % (
        "exact" if glen == cs.K5_GUARD_EXACT else "straddle", (after["device_used"] - before["device_used"]) / 1e9,
        after["host_peak_rss"] / 1e9))


# ---- K6: out modes and held answers ----------------------------------------------------------------------------------
def test_k6_device_answers_held_across_sweeps(eng):
    store = cs.k2_tiles_store()
    st = loaded(eng, store)
    mid = store.keys[store.n // 2]
    reqs = [(cs.MAGIC, mid, ALL), (mid, b"\xff", ALL), (cs.MAGIC, b"\xff", cs.T_TOMB - 1)]
    want = [ko.worker_run(st, s, e, r, compact=True, collect=True) for s, e, r in reqs]
    held = [eng.compact_sweep(s, e, r, 0, True, KB_OUT_DEVICE) for s, e, r in reqs]
    ptrs = [h.dev_ptrs["victim_idx"] for h in held]
    assert len(set(ptrs)) == len(ptrs)  # no pooled buffer is handed out twice
    host = eng.compact_sweep(cs.MAGIC, b"\xff", ALL, 0, True, KB_OUT_HOST)  # a fourth sweep while they are held
    _same(host.victim_idx, ko.worker_run(st, cs.MAGIC, b"\xff", ALL, compact=True, collect=True).victims, "host")
    host.close()
    for h, x, q in zip(held, want, reqs):
        assert (h.n_victims, h.count, h.examined) == (len(x.victims), x.count, x.examined), q
        _same(h.device_array("victim_idx"), x.victims, q)
        _same(h.device_array("victim_class"), x.vclass, q)
    held[0].close()
    again = eng.compact_sweep(*reqs[1][:2], ALL, 0, True, KB_OUT_DEVICE)  # may reuse the freed buffer, not the held ones
    assert again.dev_ptrs["victim_idx"] not in ptrs[1:]
    for h, x, q in zip(held[1:] + [again], want[1:] + [want[1]], reqs[1:] + [reqs[1]]):
        _same(h.device_array("victim_idx"), x.victims, q)
        _same(h.device_array("victim_class"), x.vclass, q)
        h.close()
    eng.set_compact_revision(None)
