"""The watch fan-out (kb_watch.cu: k_fanout, k_expand_write) against the C oracle in every group-size class, and across
consecutive bursts on one engine.  Every answer is compared exactly: the W+1 offsets, the delivery count and the full
delivery list, for a host-resident answer and for a device-resident one.

The shapes (tests/fuzz.py; tests/test_fanout_shapes.py asserts which classes each reaches) put groups on both sides of
each size threshold: 16/17 (half-warp / warp), 32/33 (small / medium), big_t / big_t+1 (medium / large, global
bitmap), medium groups inside one shared-memory window and over many, large groups over several bitmap chunks, under
four revision modes and irregular batch cuts.

The sequences keep one engine across bursts.  k_fanout clears the group state of the previous call itself when the
scratch geometry (E, groups, prefix lengths, watchers) is unchanged, and the write of one burst overlaps the next
burst's k_fanout; a burst that reads state another burst left behind differs from the oracle only when the bursts
differ, so every sequence changes the data between calls."""
from __future__ import annotations

import numpy as np
import pytest

from kubebrain_b200._lib import KB_ESTATE, KB_OUT_DEVICE, KB_OUT_HOST, Engine, KbError
from kubebrain_b200.packed import PackedEvents, PackedWatchers, Slab
from oracle import binding as ko
from tests import fuzz
from tests.fuzz import MR_ALL, REV_MODES, Group, tag

pytestmark = pytest.mark.gpu

THREADS = 8  # oracle threads


def expected(ev: PackedEvents, w: PackedWatchers):
    start, idx, _ = ko.fanout(ev, w, threads=THREADS)
    return start, idx


def _first_diff(start, idx, gstart, gidx) -> str:
    """the first watcher whose list differs, and where"""
    for i in range(len(start) - 1):
        a = idx[int(start[i]) : int(start[i + 1])]
        if i + 1 >= len(gstart):
            return "watcher %d missing" % i
        b = gidx[int(gstart[i]) : int(gstart[i + 1])]
        if not np.array_equal(a, b):
            n = min(len(a), len(b))
            j = int(np.argmax(a[:n] != b[:n])) if n and np.any(a[:n] != b[:n]) else n
            return "watcher %d: %d deliveries expected, %d got; from position %d expected %s, got %s" % (
                i, len(a), len(b), j, a[j : j + 6].tolist(), b[j : j + 6].tolist())
    return "lists equal"


def assert_same(got, exp, what: str, device: bool = False):
    start, idx = exp
    gidx = got.device_event_idx() if device else got.event_idx
    ok = (got.n_deliveries == len(idx) and got.start.tolist() == start.tolist()
          and np.array_equal(gidx, idx.astype(np.uint32)))
    assert ok, "%s: D %d vs %d; %s" % (what, got.n_deliveries, len(idx), _first_diff(start, idx, got.start, gidx))


def check_shape(ev: PackedEvents, w: PackedWatchers, what: str):
    exp = expected(ev, w)
    e = Engine(0)
    try:
        assert e.watch_add_many(w) == list(range(w.n))
        got = e.watch_match(ev, KB_OUT_HOST)
        assert_same(got, exp, what + " host")
        got.close()
        h = e.events_upload(ev)
        ds = [e.watch_match_dev(h, KB_OUT_DEVICE) for _ in range(2)]
        for d in ds:
            assert_same(d, exp, what + " device", device=True)
            d.close()
        e.events_free(h)
    finally:
        e.close()


# ---- shapes ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cuts", fuzz.CUT_MODES)
@pytest.mark.parametrize("mode", REV_MODES)
def test_shape_a(mode, cuts):
    """E = 40 001: 1 024 / 1 025, 16 / 17 / 32 / 33, medium in one window and across borders, "", nested, no-match"""
    check_shape(*fuzz.shape_a(mode, cuts), "A %s %s" % (mode, cuts))


@pytest.mark.parametrize("cuts", ["b300", "irregular"])
@pytest.mark.parametrize("mode", REV_MODES)
def test_shape_b(mode, cuts):
    """E = 200 003: 3 125 / 3 126, 17 bitmap chunks per large group, medium groups over 25 windows, 2 001 watchers"""
    check_shape(*fuzz.shape_b(mode, cuts), "B %s %s" % (mode, cuts))


@pytest.mark.parametrize("cuts", ["b300", "irregular"])
@pytest.mark.parametrize("mode", REV_MODES)
def test_shape_c(mode, cuts):
    """E = 20 000, 20 001 watchers in ~12 k groups over 10 lengths: the two-watchers-per-warp pairing with an odd W"""
    check_shape(*fuzz.shape_c(mode, cuts), "C %s %s" % (mode, cuts))


@pytest.mark.parametrize("W", [1, 2])
@pytest.mark.parametrize("E", [1, 31, 32, 33])
def test_shape_tiny(E, W):
    for mode in REV_MODES:
        for cuts in ("one", "irregular"):
            check_shape(*fuzz.shape_tiny(E, W, mode, cuts), "E=%d W=%d %s %s" % (E, W, mode, cuts))


# ---- sequences on one engine ----------------------------------------------------------------------------------------
def test_same_geometry_different_data():
    """S1: six bursts of one scratch geometry (no host reset between them): large groups become medium, their bitmap
    words move and the number of large groups changes; host-resident answers, then device-resident ones"""
    bursts, w = fuzz.seq_rotation()
    exps = [expected(ev, w) for ev in bursts]
    e = Engine(0)
    try:
        e.watch_add_many(w)
        for k, ev in enumerate(bursts):
            got = e.watch_match(ev, KB_OUT_HOST)
            assert_same(got, exps[k], "S1 host burst %d" % k)
            got.close()
        hs = [e.events_upload(ev) for ev in bursts]
        for k, h in enumerate(hs):
            d = e.watch_match_dev(h, KB_OUT_DEVICE)
            assert_same(d, exps[k], "S1 device burst %d" % k, device=True)
            d.close()
        for h in hs:
            e.events_free(h)
    finally:
        e.close()


def test_bursts_in_flight():
    """S2: device-resident bursts issued back to back without waiting (the write of one overlaps the next burst's
    k_fanout), with host-slab matches in between; every answer is held and compared at the end"""
    bursts, w = fuzz.seq_rotation(seed=15)
    exps = [expected(ev, w) for ev in bursts]
    e = Engine(0)
    try:
        e.watch_add_many(w)
        hs = [e.events_upload(ev) for ev in bursts[:4]]
        plan = [("dev", 0), ("dev", 1), ("host", 4), ("dev", 2), ("dev", 3), ("dev", 0), ("host", 5), ("dev", 3),
                ("dev", 1), ("dev", 2)]
        held = []
        for kind, k in plan:
            if kind == "dev":
                held.append((k, True, e.watch_match_dev(hs[k], KB_OUT_DEVICE)))
            else:
                held.append((k, False, e.watch_match(bursts[k], KB_OUT_HOST)))
        for n, (k, dev, r) in enumerate(held):
            assert_same(r, exps[k], "S2 call %d (burst %d, %s)" % (n, k, "device" if dev else "host"), device=dev)
            r.close()
        for h in hs:
            e.events_free(h)
    finally:
        e.close()


def test_output_regrow_in_flight():
    """S3: deliveries small -> large -> small -> large: every large burst outgrows the buffer sized from the previous
    one, in device mode with the bursts in flight, then in host mode"""
    bursts, w = fuzz.seq_regrow()
    exps = [expected(ev, w) for ev in bursts]
    d = [len(x[1]) for x in exps]
    assert d[1] > max(65536, 1.25 * d[0] + 4096) and d[3] > max(65536, 1.25 * d[2] + 4096), d
    e = Engine(0)
    try:
        e.watch_add_many(w)
        hs = [e.events_upload(ev) for ev in bursts]
        held = [e.watch_match_dev(h, KB_OUT_DEVICE) for h in hs]
        for k, r in enumerate(held):
            assert_same(r, exps[k], "S3 device burst %d" % k, device=True)
            r.close()
        for k, ev in enumerate(bursts):
            got = e.watch_match(ev, KB_OUT_HOST)
            assert_same(got, exps[k], "S3 host burst %d" % k)
            got.close()
        for h in hs:
            e.events_free(h)
    finally:
        e.close()


def _expected_live(ev: PackedEvents, live: dict, n_ids: int):
    """the oracle on the live watchers, laid out by watcher id (a deleted id has an empty list)"""
    ids = sorted(live)
    w = PackedWatchers(Slab.from_list([live[i][0] for i in ids]), np.array([live[i][1] for i in ids], np.uint64))
    start, idx = expected(ev, w)
    lists = {i: idx[int(start[j]) : int(start[j + 1])] for j, i in enumerate(ids)}
    parts = [lists.get(i, np.zeros(0, idx.dtype)) for i in range(n_ids)]
    out = np.zeros(n_ids + 1, np.uint64)
    np.cumsum([len(p) for p in parts], out=out[1:])
    return out, (np.concatenate(parts) if parts else np.zeros(0, np.uint32))


def test_watcher_churn_between_bursts():
    """S4: G grows; the only watcher of a prefix is replaced by another prefix (G unchanged, group ids shift, the freed
    id is reused); every watcher deleted (W > 0, G = 0); watchers added back"""
    ev, w0 = fuzz.shape_a("stepback", "irregular", seed=21, n_watchers=61)
    ev2 = fuzz.shape_a("random", "b300", seed=22)[0]
    e = Engine(0)
    live, n_ids = {}, 0

    def add(p, r):
        nonlocal n_ids
        i = e.watch_add(p, r)
        assert i not in live
        live[i] = (p, r)
        n_ids = max(n_ids, i + 1)
        return i

    def drop(i):
        e.watch_del(i)
        del live[i]

    def check(step):
        for burst in (ev, ev2):
            exp = _expected_live(burst, live, n_ids)
            got = e.watch_match(burst, KB_OUT_HOST)
            assert_same(got, exp, "S4 %s host" % step)
            assert got.n_watchers == n_ids and e.watch_count() == len(live)
            for i in range(n_ids):
                if i not in live:
                    assert got.start[i] == got.start[i + 1], (step, i)
            got.close()
            h = e.events_upload(burst)
            d = e.watch_match_dev(h, KB_OUT_DEVICE)
            assert_same(d, exp, "S4 %s device" % step, device=True)
            d.close()
            e.events_free(h)

    try:
        pref, mr = w0.prefixes.tolist(), w0.min_rev.tolist()
        for i in range(41):
            add(pref[i], mr[i])
        check("initial")
        for i in range(41, 61):
            add(pref[i], mr[i])
        only = add(tag(50, 33), 0)  # the only watcher of its prefix
        add(tag(1), 0)
        check("G grows")
        g_before = len({p for p, _ in live.values()})
        drop(only)
        new = add(b"/bg/#1", 0)  # sorts in front of every tag: the group ids behind it shift
        assert new == only and len({p for p, _ in live.values()}) == g_before
        check("prefix replaced, id reused")
        drop(sorted(live)[3])
        check("one id deleted")
        for i in sorted(live):
            drop(i)
        check("every watcher deleted")
        for i in range(0, 61, 3):
            add(pref[i], mr[i])
        check("added back")
    finally:
        e.close()


def test_stride_check_then_reupload():
    """S5: a watcher prefix longer than an uploaded slab's key stride makes matching that slab an error (KB_ESTATE);
    the slab uploaded again matches the oracle"""
    g = [Group(tag(1, 17), 300, "spread", MR_ALL), Group(b"", 0, "spread", ("0",)), Group(tag(2, 40), 50, "cluster")]
    ev = fuzz.burst_events(31, 3001, g, "random", "irregular")
    w = fuzz.burst_watchers(ev, g[:2], 31)
    e = Engine(0)
    try:
        e.watch_add_many(w)
        h = e.events_upload(ev)  # keys stored to 32 bytes: the longest prefix is 17
        d = e.watch_match_dev(h, KB_OUT_DEVICE)
        assert_same(d, expected(ev, w), "S5 before", device=True)
        d.close()
        e.watch_add(tag(2, 40), 0)
        w2 = PackedWatchers(Slab.from_list(w.prefixes.tolist() + [tag(2, 40)]), np.append(w.min_rev, np.uint64(0)))
        exp2 = expected(ev, w2)
        assert int(exp2[0][-1] - exp2[0][-2]) == 50
        with pytest.raises(KbError) as ei:
            e.watch_match_dev(h, KB_OUT_DEVICE)
        assert ei.value.code == KB_ESTATE
        e.events_free(h)
        h = e.events_upload(ev)
        d = e.watch_match_dev(h, KB_OUT_DEVICE)
        assert_same(d, exp2, "S5 re-uploaded", device=True)
        d.close()
        got = e.watch_match(ev, KB_OUT_HOST)
        assert_same(got, exp2, "S5 host slab")
        got.close()
        e.events_free(h)
    finally:
        e.close()


def test_empty_bursts_between():
    """S6: E = 0 bursts (no launch: the host resets the scratch) between device-resident bursts"""
    bursts, w = fuzz.seq_rotation(seed=25, n_bursts=3)
    empty = PackedEvents(Slab.from_list([]), np.zeros(0, np.uint64), np.zeros(1, np.uint64))
    seq = [bursts[0], empty, bursts[1], empty, empty, bursts[2], bursts[0]]
    exps = [expected(ev, w) for ev in seq]
    e = Engine(0)
    try:
        e.watch_add_many(w)
        hs = [e.events_upload(ev) for ev in seq]
        held = [e.watch_match_dev(h, KB_OUT_DEVICE) for h in hs]
        got = e.watch_match(empty, KB_OUT_HOST)
        assert got.n_deliveries == 0 and not got.start.any()
        got.close()
        held += [e.watch_match_dev(hs[2], KB_OUT_DEVICE)]
        for k, r in enumerate(held):
            assert_same(r, exps[k] if k < len(seq) else exps[2], "S6 call %d" % k, device=True)
            r.close()
        for h in hs:
            e.events_free(h)
    finally:
        e.close()
