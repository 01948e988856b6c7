"""kb_range_partitions at its key-order, search, warp, report and snapshot boundaries (tests/partition_shapes.py Q1-Q5):
every call equals the reference helper byte for byte and keeps the invariants checked against the oracle alone
(partition_shapes.check_partitions); on selected shapes the device's range batches (host and count modes) and range
streams over the borders concatenate to the whole answer."""
from __future__ import annotations

import ctypes
import struct

import pytest

from kubebrain_b200 import _lib
from kubebrain_b200._lib import KB_EINVAL, KB_ELIMIT, Engine, KbError
from oracle import binding as ko
from tests import partition_shapes as ps
from tests.range_shapes import TOMB, ik
from tests.test_gpu_partitions import answers_whole

pytestmark = pytest.mark.gpu

ALL = ps.ALL


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def check(eng, store, st, s, e, rev, part_bytes, max_parts, other_revs=(), what="", kv_first=None):
    want = ps.partitions(store, st, s, e, rev, part_bytes, max_parts)
    b, kf, af = eng.range_partitions(s, e, rev, part_bytes, max_parts)
    got = (b, kf.tolist(), af.tolist())
    assert got[1] == want[1], (what, part_bytes, max_parts, "kv_first")
    assert got[2] == want[2], (what, part_bytes, max_parts, "arena_first")
    assert got[0] == want[0], (what, part_bytes, max_parts, "borders")
    split = ps.check_partitions(store, st, s, e, rev, got, other_revs)
    if kv_first is not None:
        kv_first[:] = got[1]
    return got[0], split


def _total(store, st, s, e, rev):
    emit = ko.range_(st, s, e, rev, 0).emit.tolist()
    return sum(ps.pad16(len(store.keys[i])) + ps.pad16(len(store.vals[i])) for i in emit), len(emit)


def _load(eng, store):
    eng.load_sorted(store)
    return ko.OracleStore(store)


# ---- Q1 key order ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rev_records", [True, False])
def test_q1_key_order(eng, rev_records):
    store = ps.q1_store(rev_records)
    st = _load(eng, store)
    dropped = 0
    for name, s, e in ps.q1_intervals(store):
        for rev in ps.Q1_REVS:
            total, n = _total(store, st, s, e, rev)
            for pb in ps.q1_part_bytes(total, n):
                for mp in (2, 3, 64):
                    b, split = check(eng, store, st, s, e, rev, pb, mp, ps.Q1_REVS, (name, rev))
                    dropped += len(b) - 1 < ps.part_count(n, total, pb, mp, s, e)
                    if pb == 1 and mp == 64 and name in ("q", "n", "all", "start_is_revkey_e1") and s < e:
                        answers_whole(eng, st, b, [rev] if split else [rev, 3, ALL])
    assert dropped


# ---- Q2 search --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", ps.Q2_N)
def test_q2_search(eng, n):
    store = ps.sized_store([40] * n)
    st = _load(eng, store)
    T, _ = _total(store, st, b"", b"\xff", ALL)
    assert T == 80 * n
    b, _ = check(eng, store, st, b"", b"\xff", ALL, 1, ps.MAX_PARTS, [5])  # every i in [1, n) a cut
    assert len(b) - 1 == n
    answers_whole(eng, st, b, [ALL], streams=n < 100)
    for k in (2, 7):  # slot[i] * P == k * T exactly where k divides n; T == part_bytes * k and +- 1
        for d in (-1, 0, 1):
            check(eng, store, st, b"", b"\xff", ALL, T // k + d, ps.MAX_PARTS)


def test_q2_equal_bumped_big_and_unreached(eng):
    for vals in ([40] * 34, [40] * 17 + [56] + [40] * 16, [40] * 40 + [24000] + [40] * 59,
                 [40] * 100 + [40000], [40] * 1100 + [400000]):
        store = ps.sized_store(vals)
        st = _load(eng, store)
        T, n = _total(store, st, b"", b"\xff", ALL)
        for pb in (T // 2, T // 20, T // 33, max(T // 1000, 1), 1):
            b, _ = check(eng, store, st, b"", b"\xff", ALL, pb, ps.MAX_PARTS, [5], len(vals))
        b, _ = check(eng, store, st, b"", b"\xff", ALL, T // 20, 64)
        answers_whole(eng, st, b, [ALL, 5])


# ---- Q3 warps and clamps ------------------------------------------------------------------------------------------------
def test_q3_warps_and_clamps(eng):
    store = ps.uniform_store(4200)
    st = _load(eng, store)
    s, e = ik(b"/u/", 0), b"\xff"
    T, n = _total(store, st, s, e, ALL)
    for p in (16, 17, 18, 32, 33, 34):  # P - 1 of 15 .. 17 and 31 .. 33 cuts over 16 warps
        b, _ = check(eng, store, st, s, e, ALL, -(-T // p), 64, [300])
        assert len(b) - 1 == p
    answers_whole(eng, st, b, [ALL, 300], streams=False)
    b, _ = check(eng, store, st, s, e, ALL, 1, 4096)
    assert len(b) - 1 == 4096
    few = ik(b"/u/o%07d" % 5, 0)
    b, _ = check(eng, store, st, s, few, ALL, 1, 64)  # the n clamp
    assert len(b) - 1 == 5
    for pb, mp, code in ((1, 4097, KB_ELIMIT), (0, 64, KB_EINVAL), (1 << 20, 0, KB_EINVAL)):
        with pytest.raises(KbError) as ex:
            eng.range_partitions(s, e, ALL, pb, mp)
        assert ex.value.code == code
    req = eng.pack_range_reqs([(s, e, ALL, 5)])
    h = ctypes.c_void_p()
    assert _lib.lib().kb_range_partitions(eng._ctx, req.arr, 1 << 20, 64, ctypes.byref(h)) == KB_EINVAL  # limit > 0
    assert eng.range_partitions(s, e, ALL, 1 << 40, 64)[0] == [s, e]  # still answers


# ---- Q4 report ---------------------------------------------------------------------------------------------------------
def test_q4_key_lengths(eng):
    store = ps.q4_store()
    st = _load(eng, store)
    b, _ = check(eng, store, st, b"", b"\xff", ALL, 1, 64, [3])
    assert sorted(len(x) for x in b[1:-1]) == [L for L in ps.Q4_KEY_LENS if L != ps.Q4_KEY_LENS[0]]
    answers_whole(eng, st, b, [ALL, 3])
    for pb in (1000, 70_000, 140_000):
        check(eng, store, st, b"", b"\xff", ALL, pb, 64)


def test_q4_report_regrows_on_one_engine(eng):
    """small, large and small P, a write of a 65 535-byte key (the report's key stride grows from 80 bytes to 64 KiB),
    then P = 4096 again: k_partition_cut's pinned report is regrown between calls"""
    store = ps.uniform_store(4200)
    st = _load(eng, store)
    s, e = ik(b"/u/", 0), b"\xff"
    for mp in (8, 4096, 8):
        check(eng, store, st, s, e, ALL, 1, mp)
    eng.apply_batch([(ps.LONG_KEY, b"long")])
    items = dict(zip(store.keys.tolist(), store.vals.tolist()))
    cur = ps.apply_model(items, [(ps.LONG_KEY, b"long")])
    assert ps.max_kv_chunks(cur) == 4097
    cst = ko.OracleStore(cur)
    for mp in (4096, 8, 4096):
        check(eng, cur, cst, s, e, ALL, 1, mp)
    end = ik(b"/u/o0000820", 0)
    T, _ = _total(cur, cst, s, end, ALL)
    b, _ = check(eng, cur, cst, s, end, ALL, -(-T // 2), 64)
    assert b[1] == ps.revision_key(ps.LONG_KEY)
    answers_whole(eng, cst, b, [ALL, 300])


# ---- Q5 snapshots -------------------------------------------------------------------------------------------------------
def test_q5_snapshots(eng, tmp_path):
    store = ps.q5_store()
    st = _load(eng, store)
    s, e = ik(b"/r/", 0), ik(b"/r0", 0)
    items = dict(zip(store.keys.tolist(), store.vals.tolist()))
    revs = [ALL, 250, 120]

    def round_(cur, what):
        """check the partitions of cur at three shares; returns the internal key of the 8-share call's first cut kv"""
        cst = ko.OracleStore(cur)
        T, _ = _total(cur, cst, s, e, ALL)
        for share in (2, 8, 50):
            kf = []
            b, split = check(eng, cur, cst, s, e, ALL, max(T // share, 1), 64, revs, what, kv_first=kf)
            assert not split
            if share == 8:
                cut = cur.keys[ko.range_(cst, s, e, ALL, 0).emit.tolist()[kf[1]]]
                answers_whole(eng, cst, b, revs)
        return cut

    cut = round_(store, "load")
    # a batch that deletes the cut kv
    ops = [(cut, None)]
    eng.apply_batch(ops)
    cut = round_(ps.apply_model(items, ops), "delete")
    # one that tombstones the cut's object
    uk = ps.decode(cut)[0]
    ops = [(ik(uk, 900), TOMB), (ik(uk, 0), struct.pack(">Q", 900))]
    eng.apply_batch(ops)
    cut = round_(ps.apply_model(items, ops), "tombstone")
    # one that inserts an object in front of the cut kv
    uk = ps.decode(cut)[0]
    front = uk[:-1] + bytes([uk[-1] - 1]) + b"~front"
    ops = [(ik(front, 0), struct.pack(">Q", 950)), (ik(front, 950), b"f" * 3000)]
    eng.apply_batch(ops)
    round_(ps.apply_model(items, ops), "insert in front")
    # TTL records due at 1000, dropped by expire
    ttl = [(ik(b"/r/%04d~ttl" % j, 960 + j), b"t" * (100 * j), 1000) for j in range(1, 30)]
    eng.apply_batch(ttl)
    round_(ps.apply_model(items, [op[:2] for op in ttl]), "before expire")
    assert eng.expire(1000) == len(ttl)
    cur = ps.apply_model(items, [(op[0], None) for op in ttl])
    round_(cur, "after expire")
    # restore the image into the engine after another store was loaded
    path = str(tmp_path / "snap")
    eng.dump(path)
    eng.load_sorted(ps.uniform_store(50))
    eng.restore(path)
    round_(cur, "after restore")
