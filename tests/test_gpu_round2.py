"""GPU parity / behaviour tests of the round-2 features, through the C ABI against the CPU oracle:
TTL expiry (kb_write_op.expire_unix + kb_expire), the user-limit RangeResponse helper, the heap + sorted-directory write
path (layout compaction, dump / restore after appends, write rate), the decoupled look-back on its worst case, and
batches in flight."""
from __future__ import annotations

import random
import struct
import time

import numpy as np
import pytest

from kubebrain_b200 import synth, wire
from kubebrain_b200._lib import KB_OUT_COUNT, KB_OUT_DEVICE, KB_OUT_HOST, Engine
from kubebrain_b200.coder import NormalCoder, prefix_end
from kubebrain_b200.packed import PackedStore
from oracle import binding as ko
from tests import fuzz
from tests.test_gpu_parity import check_compact, check_ranges

pytestmark = pytest.mark.gpu

CODER = NormalCoder()
LO, HI = CODER.encode_object_key(b"/registry/", 0), CODER.encode_object_key(b"/registry0", 0)


@pytest.fixture()
def eng():
    e = Engine(0)
    yield e
    e.close()


def _ik(uk: bytes, rev: int) -> bytes:
    return CODER.encode_object_key(uk, rev)


def test_ttl_expire(eng):
    """/events/ keys are written with a ttl (BatchWrite.Put(key, val, ttl), badger WithTTL batch.go:47-93) and never
    deleted explicitly: after kb_expire(now) the mirror answers like an engine that stopped returning the expired keys"""
    now = 1_700_000_000
    items, expire = {}, {}
    rev = 100
    ops = []
    for i in range(300):
        res = (b"pods", b"events")[i % 2]
        uk = b"/registry/%s/ns-%d/o%03d" % (res, i % 4, i)
        rev += 1
        exp = now + 10 + i if res == b"events" else 0
        for k, v in ((_ik(uk, 0), struct.pack(">Q", rev)), (_ik(uk, rev), b"v" * (20 + i))):
            ops.append((k, v, exp))
            items[k] = v
            if exp:
                expire[k] = exp
    eng.load_sorted(PackedStore.from_items([]))
    eng.apply_batch(ops)
    # a later write of the same key WITHOUT ttl cancels the expiry; a delete cancels it too
    k_keep = _ik(b"/registry/events/ns-1/o001", 0)
    eng.apply_batch([(k_keep, struct.pack(">Q", 7777))])
    items[k_keep] = struct.pack(">Q", 7777)
    expire.pop(k_keep)
    k_gone = _ik(b"/registry/events/ns-3/o003", 0)
    eng.apply_batch([(k_gone, None)])
    items.pop(k_gone)
    expire.pop(k_gone)
    for t in (now + 5, now + 100, now + 100, now + 10_000):
        before = len(items)
        for k in [k for k, e in expire.items() if e <= t]:
            items.pop(k)
            expire.pop(k)
        assert eng.expire(t) == before - len(items)
        cur = PackedStore.from_items(list(items.items()))
        assert eng.store_info()[0] == cur.n
        check_ranges(eng, cur, ko.OracleStore(cur), [(LO, HI, 2**62, 0), (LO, HI, 150, 0), (LO, HI, 2**62, 5)])
    assert not expire


def test_range_prefetch(eng):
    """kb_range_prefetch: the bound search of a batch started ahead is picked up by the identical batch on the same
    snapshot and ignored otherwise (other bounds, snapshot changed in between); two submissions may be outstanding"""
    store, meta = synth.gen_store(3000, 3, 64, 80, 9, config_id=2, tomb_frac=0.1)
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    p = b"/registry/pods/ns-00003/"
    a = [(LO, HI, meta.read_rev, 0), (CODER.encode_object_key(p, 0), CODER.encode_object_key(prefix_end(p), 0), meta.last_rev, 5)]
    b = [(LO, HI, meta.last_rev, 7)]
    eng.range_prefetch(a)
    eng.range_prefetch(a)  # the batch after the next one, submitted before the first is consumed
    check_ranges(eng, store, st, a)
    check_ranges(eng, store, st, a)
    eng.range_prefetch(a)
    check_ranges(eng, store, st, b)  # different bounds: own search
    check_ranges(eng, store, st, a)  # the submission from before is still there
    eng.range_prefetch(a)
    k = store.keys[10]
    eng.apply_batch([(k, None)])  # the snapshot changes: the submitted search is void
    items = dict(zip(store.keys.tolist(), store.vals.tolist()))
    items.pop(k)
    cur = PackedStore.from_items(list(items.items()))
    check_ranges(eng, cur, ko.OracleStore(cur), a)


def test_list_response_wire(eng):
    """wire.list_response: user limit -> scan limit + 1 -> cut at elem_off[limit] -> More / Count
    (pkg/backend/range.go:150-170, pkg/server/etcd/backendshim.go:269-277)"""
    store, meta = synth.gen_store(500, 3, 48, 100, 5, config_id=2)
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    p = b"/registry/pods/"
    s, e = CODER.encode_object_key(p, 0), CODER.encode_object_key(prefix_end(p), 0)
    total = len(ko.range_(st, s, e, meta.last_rev, 0).emit)
    assert total > 20
    for limit in (0, 1, 7, total - 1, total, total + 5):
        exp = ko.range_(st, s, e, meta.last_rev, limit + 1 if limit else 0)
        keep = exp.emit[:limit] if limit else exp.emit
        more = bool(limit) and len(exp.emit) > limit
        body, _ = ko.wire_encode(st, keep, ko.WIRE_KVS)
        want = ko.wire_range_head(meta.last_rev) + body + ko.wire_range_tail(more, len(keep) + (1 if more else 0))
        assert wire.list_response(eng, s, e, meta.last_rev, limit, meta.last_rev) == want, limit


def test_heap_layout_compaction_and_dump(eng, tmp_path):
    """appends beyond the thresholds trigger the layout compaction; a dump taken while records are out of place restores
    to the same answers"""
    rng = random.Random(3)
    store, meta = synth.gen_store(4000, 3, 64, 120, 10, config_id=2, tomb_frac=0.1)
    eng.load_sorted(store)
    items = dict(zip(store.keys.tolist(), store.vals.tolist()))
    keys = sorted(items)
    for rnd in range(6):
        ops = []
        for k in rng.sample(keys, 900):
            r = rng.random()
            if r < 0.5:  # new version of the same object: an insert next to it, bytes at the slab tail
                ops.append((k[:-8] + struct.pack(">Q", rng.randint(1, 2**40)), bytes([rnd]) * rng.randint(1, 200)))
            elif r < 0.8:
                ops.append((k, bytes([rnd + 9]) * rng.randint(0, 300)))  # same key, new value: old bytes become garbage
            else:
                ops.append((k, None))
        eng.apply_batch(ops)
        for k, v in ops:
            if v is None:
                items.pop(k, None)
            else:
                items[k] = v
        keys = sorted(items)
        cur = PackedStore.from_items(list(items.items()))
        st = ko.OracleStore(cur)
        assert eng.store_info()[0] == cur.n
        check_ranges(eng, cur, st, [(LO, HI, meta.last_rev, 0), (LO, HI, meta.read_rev, 0), (LO, HI, 2**62, 11)])
        if rnd == 2:  # records are out of place right now
            path = str(tmp_path / "snap.kb")
            eng.dump(path)
            e2 = Engine(0)
            e2.restore(path)
            assert e2.store_info()[0] == cur.n
            check_ranges(e2, cur, st, [(LO, HI, meta.last_rev, 0), (LO, HI, 2**62, 11)])
            check_compact(e2, cur, st, LO, HI, meta.read_rev)
            e2.close()
    check_compact(eng, cur, st, LO, HI, meta.read_rev)


def test_write_rate_300_op_batches(eng):
    """the write path behind the 300-event collector batches on a 200k-record store: the cost of a batch no longer grows
    with the bytes of the store (round 1 rebuilt both slabs per batch)"""
    store, meta = synth.gen_store(40_000, 4, 256, 2048, 200, config_id=2)
    eng.load_sorted(store)
    keys = store.keys.tolist()
    rng = random.Random(11)
    rev = meta.last_rev
    t0 = time.perf_counter()
    n_ops = 0
    for _ in range(20):
        ops = []
        for k in rng.sample(keys, 150):  # an update = CAS of the revision record + Put of the new version
            rev += 1
            uk = k[4:-9]
            ops.append((_ik(uk, 0), struct.pack(">Q", rev)))
            ops.append((_ik(uk, rev), b"w" * 2048))
        eng.apply_batch(ops)
        n_ops += len(ops)
    dt = time.perf_counter() - t0
    assert eng.store_info()[0] == store.n + n_ops // 2
    assert n_ops / dt > 20_000, f"{n_ops / dt:.0f} ops/s"


def test_lookback_worst_case_is_not_quadratic(eng):
    """round 1's k_emit walked the sub-tile aggregates of the request backwards until it met a visible record: with long
    runs of invisible records (a read revision below every version; a compact at an old revision) every tile walked to
    the start of the request.  With decoupled look-back both scans cost what the ordinary ones cost."""
    store, meta = synth.gen_store(8, 400_000, 64, 16, 1, config_id=4, tomb_frac=0.0)  # 3.2M records, 8 objects
    st = ko.OracleStore(store)
    eng.load_sorted(store)

    def timed(fn, reps=5):
        fn()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        return (time.perf_counter() - t0) / reps

    normal = timed(lambda: eng.range_batch([(LO, HI, meta.last_rev, 0)], KB_OUT_COUNT).close())
    old = meta.first_rev  # below every object version: only the 8 revision records are visible
    worst = timed(lambda: eng.range_batch([(LO, HI, old, 0)], KB_OUT_COUNT).close())
    assert worst <= 2.0 * normal + 2e-4, (normal, worst)
    r = eng.range_batch([(LO, HI, old, 0)], KB_OUT_HOST)
    assert r.rec_idx.astype(np.uint64).tolist() == ko.range_(st, LO, HI, old, 0).emit.tolist()
    r.close()
    sweep_n = timed(lambda: eng.compact_sweep(LO, HI, meta.last_rev, out_mode=KB_OUT_COUNT).close())
    sweep_w = timed(lambda: eng.compact_sweep(LO, HI, old, out_mode=KB_OUT_COUNT).close())
    assert sweep_w <= 2.0 * sweep_n + 2e-4, (sweep_n, sweep_w)
    eng.set_compact_revision(None)
    check_compact(eng, store, st, LO, HI, old)
    eng.set_compact_revision(None)
    mid = meta.first_rev + (meta.last_rev - meta.first_rev) // 3
    check_compact(eng, store, st, LO, HI, mid)


def _check_result(res, store, st, reqs):
    for q, (s, e, rev, lim) in enumerate(reqs):
        exp = ko.range_(st, s, e, rev, lim)
        assert res.rec_indices(q).astype(np.uint64).tolist() == exp.emit.tolist(), (q, rev, lim)
        assert int(res.req_count[q]) == exp.count and int(res.req_examined[q]) == exp.examined, q
        assert res.kvs(q) == exp.kvs(store), (q, "kv bytes")


def test_range_submit_collect(eng):
    """kb_range_submit / kb_range_collect: batches in flight on the two lanes answer exactly like kb_range_batch, in any
    collection order, with more submissions than lanes, with other entry points in between (a write sees the submitted
    batches finish on the snapshot they were submitted on), and a pending that is given up frees its buffers"""
    store, meta = synth.gen_store(6000, 4, 64, 90, 9, config_id=2, tomb_frac=0.1)
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    p = b"/registry/pods/ns-00002/"
    a = [(LO, HI, meta.read_rev, 0), (CODER.encode_object_key(p, 0), CODER.encode_object_key(prefix_end(p), 0), meta.last_rev, 5)]
    b = [(LO, HI, meta.last_rev, 7), (LO, HI, meta.first_rev, 0), (HI, HI, meta.last_rev, 0)]
    c = [(LO, HI, meta.last_rev, 0)]
    for mode in (KB_OUT_HOST, KB_OUT_DEVICE):
        # in order, out of order, three submissions before the first collection
        for order in ((0, 1, 2), (2, 0, 1), (1, 2, 0)):
            batches = [a, b, c]
            pend = [eng.range_submit(x, mode) for x in batches]
            for i in order:
                r = pend[i].collect()
                if mode == KB_OUT_DEVICE:
                    h = eng.range_batch(batches[i], KB_OUT_HOST)
                    assert r.req_first.tolist() == h.req_first.tolist()
                    assert r.req_count.tolist() == h.req_count.tolist() and r.req_examined.tolist() == h.req_examined.tolist()
                    assert r.device_array("rec_idx", np.uint32).tolist() == h.rec_idx.tolist()
                    assert r.device_array("rev", np.uint64).tolist() == h.rev.tolist()
                    assert r.n_bytes == h.n_bytes
                    assert eng.read_device(r.bytes_ptr, int(r.n_bytes), sync=False) == bytes(h.arena[: int(r.n_bytes)])
                    h.close()
                else:
                    _check_result(r, store, st, batches[i])
                r.close()
    # the plain call between a submission and its collection
    pa = eng.range_submit(a, KB_OUT_HOST)
    check_ranges(eng, store, st, b)
    pb = eng.range_submit(b, KB_OUT_HOST)
    check_ranges(eng, store, st, c)
    r = pb.collect(); _check_result(r, store, st, b); r.close()
    r = pa.collect(); _check_result(r, store, st, a); r.close()
    # a write between submission and collection: the submitted batches were answered on the old snapshot
    pa = eng.range_submit(a, KB_OUT_HOST)
    pc = eng.range_submit(c, KB_OUT_HOST)
    k = store.keys[17]
    eng.apply_batch([(k, None)])
    r = pa.collect(); _check_result(r, store, st, a); r.close()
    r = pc.collect(); _check_result(r, store, st, c); r.close()
    items = dict(zip(store.keys.tolist(), store.vals.tolist()))
    items.pop(k)
    cur = PackedStore.from_items(list(items.items()))
    cst = ko.OracleStore(cur)
    pa = eng.range_submit(a, KB_OUT_HOST)
    pgone = eng.range_submit(b, KB_OUT_DEVICE)
    pgone.close()  # given up
    with pytest.raises(Exception):
        pgone.collect()
    r = pa.collect(); _check_result(r, cur, cst, a); r.close()
    # many rounds with two in flight
    prev = eng.range_submit(a, KB_OUT_HOST)
    for i in range(20):
        nxt = eng.range_submit(a if i % 2 else c, KB_OUT_HOST)
        r = prev.collect()
        _check_result(r, cur, cst, c if i % 2 else a)
        r.close()
        prev = nxt
    prev.collect().close()
