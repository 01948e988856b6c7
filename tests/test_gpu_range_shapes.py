"""The range scan (kb_scan.cu: k_decode_lcp, k_emit, k_tile_scan, k_place, k_gather, k_wire_copy) against the C oracle on
stores built to put its fixed boundaries on purpose (tests/range_shapes.py; tests/test_range_shapes.py asserts which
classes each shape reaches): tile seams after non-PREVOK runs on both sides of the carry window and of a look-back
step, a batch over more than one k_tile_scan chunk with empty requests sharing a tile, limit probe rounds 0-2 with and
without the reuse of the probe pass, pairs on both sides of k_gather's round and the wire copy's ring room.

Compared exactly: the rows (first kv, count, examined), record indices, revisions, key and value bytes, the whole arena
padding included (host- and device-resident) against the image the oracle's emits imply, both wire modes against the
oracle's encoder, the sweep's ordered victim list, point reads."""
from __future__ import annotations

import numpy as np
import pytest

from kubebrain_b200 import synth
from kubebrain_b200._lib import (KB_ELIMIT, KB_OUT_COUNT, KB_OUT_DEVICE, KB_OUT_HOST, KB_WIRE_ETCD_EVENTS,
                                 KB_WIRE_ETCD_KVS, Engine, KbError)
from kubebrain_b200.packed import PackedStore
from oracle import binding as ko
from tests import fuzz
from tests import range_shapes as rs
from tests.test_gpu_parity import check_compact, check_gets, check_ranges
from tests.test_gpu_round2 import HI, LO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def _pad16(b: bytes) -> bytes:
    return b + b"\x00" * (-len(b) % 16)


def expected(store: PackedStore, st: ko.OracleStore, reqs):
    exps = [ko.range_(st, s, e, rev, lim) for s, e, rev, lim in reqs]
    for x in exps:
        assert x.rc == 0
    return exps


def arena_image(store: PackedStore, emit: np.ndarray) -> bytes:
    """[internal key, zero padded][value, zero padded] per emitted kv, in order"""
    return b"".join(_pad16(store.keys[int(i)]) + _pad16(store.vals[int(i)]) for i in emit)


def check_answer(eng: Engine, store: PackedStore, st: ko.OracleStore, reqs, exps=None, what=""):
    """every field of a batch answer in the arena modes (host and device), both wire modes and the count mode"""
    exps = exps or expected(store, st, reqs)
    first = np.cumsum([0] + [len(x.emit) for x in exps]).tolist()
    emit = np.concatenate([x.emit for x in exps]).astype(np.uint64) if exps else np.zeros(0, np.uint64)
    image = arena_image(store, emit)
    rows = (first, [x.count for x in exps], [x.examined for x in exps])
    res = eng.range_batch(reqs, KB_OUT_HOST)
    assert (res.req_first.tolist(), res.req_count.tolist(), res.req_examined.tolist()) == rows, what
    assert res.rec_idx.astype(np.uint64).tolist() == emit.tolist(), what
    for q, x in enumerate(exps):
        assert res.kvs(q) == x.kvs(store), (what, q)
    assert res.n_bytes == len(image) and res.arena[: res.n_bytes].tobytes() == image, (what, "arena")
    host_rev = res.rev.tolist()
    res.close()
    dev = eng.range_batch(reqs, KB_OUT_DEVICE)
    assert (dev.req_first.tolist(), dev.req_count.tolist(), dev.req_examined.tolist()) == rows, what
    assert dev.device_array("rec_idx", np.uint32).astype(np.uint64).tolist() == emit.tolist(), what
    assert dev.device_array("rev", np.uint64).tolist() == host_rev, what
    assert dev.n_bytes == len(image) and eng.read_device(dev.bytes_ptr, dev.n_bytes, sync=False) == image, (what, "dev")
    dev.close()
    for mode, omode in ((KB_WIRE_ETCD_KVS, ko.WIRE_KVS), (KB_WIRE_ETCD_EVENTS, ko.WIRE_EVENTS)):
        w = eng.range_batch(reqs, KB_OUT_HOST | mode)
        assert (w.req_first.tolist(), w.req_count.tolist(), w.req_examined.tolist()) == rows, (what, mode)
        wexp, woff = ko.wire_encode(st, emit, omode)
        assert w.elem_off.tolist() == woff.tolist() and w.arena.tobytes() == wexp, (what, mode)
        w.close()
    cnt = eng.range_batch([(s, e, r, 0) for s, e, r, _ in reqs], KB_OUT_COUNT)
    for q, (s, e, r, _) in enumerate(reqs):
        if s <= e:
            assert int(cnt.req_count[q]) == ko.scan(st, [s, e], r, collect=False).count, (what, q, "count")
    cnt.close()


# ---- R1: tile seams -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def r1():
    sh = rs.r1_store()
    return sh, ko.OracleStore(sh.store)


def test_r1_seams(eng, r1):
    """one batch over every start (> 1 024 tiles), empty requests at its start, middle and end"""
    sh, st = r1
    eng.load_sorted(sh.store)
    eng.set_compact_revision(None)
    check_answer(eng, sh.store, st, rs.r1_requests(sh), what="R1")
    below = [(s, e, rs.TTL - 50, 0) for s, e, _, _ in rs.r1_requests(sh)[3:6]]  # fewer visible records: longer runs
    check_answer(eng, sh.store, st, below, what="R1 below")


@pytest.mark.parametrize("start", ["s0", "s1", "s255", "reach_back"])
def test_r1_sweep(eng, r1, start):
    """the sweep's ordered victim list on R1: Q5 revision records and expired `/events/` records form the runs"""
    sh, st = r1
    eng.load_sorted(sh.store)
    s = sh.starts[start]
    check_compact(eng, sh.store, st, s, sh.end, rs.READ)
    check_compact(eng, sh.store, st, s, sh.end, rs.READ, timeout_rev=rs.TTL, support_ttl=False)
    check_compact(eng, sh.store, st, s, sh.end, rs.READ, timeout_rev=rs.TTL, support_ttl=True)
    eng.set_compact_revision(None)


# ---- R2: limit probe windows ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("batch", list(rs.R2_BATCHES))
def test_r2_limit_windows(eng, batch):
    store = rs.r2_store()
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    rq = rs.r2_requests(store)
    check_answer(eng, store, st, [rq[n] for n in rs.R2_BATCHES[batch]], what=batch)


# ---- R3: pair sizes, wire room -------------------------------------------------------------------------------------
def test_r3_pairs_and_point_reads(eng):
    store = rs.r3_store()
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    reqs = rs.r3_requests(store)
    for q in reqs:
        check_answer(eng, store, st, [q], what=q[0][:12])
    check_answer(eng, store, st, reqs, what="R3")
    gets = []
    for k in store.keys.tolist():
        uk, rev, err = ko.decode(k)
        gets += [(uk, 0), (uk, rev), (uk, max(rev - 1, 1))]
    check_gets(eng, store, st, gets)  # includes the 65 522-byte user key, the longest a record can hold
    with pytest.raises(KbError) as ei:
        eng.get_batch([(b"h" * (65535 - 12), 0)])
    assert ei.value.code == KB_ELIMIT
    dev = eng.get_batch(gets, KB_OUT_DEVICE)
    host = eng.get_batch(gets, KB_OUT_HOST)
    assert dev.on_device and dev.n_bytes == host.n_bytes
    assert (dev.status.tolist(), dev.mod_rev.tolist()) == (host.status.tolist(), host.mod_rev.tolist())
    found = host.status == 0
    assert dev.rec_idx[found].tolist() == host.rec_idx[found].tolist()
    assert dev.val_len[found].tolist() == host.val_len[found].tolist()
    dev.close(), host.close()


@pytest.mark.parametrize("kind", ["small", "mid", "large"])
def test_wire_room(eng, kind):
    """ring geometries of the wire copy, then a larger pair raises max_kv_chunks through kb_apply_batch"""
    store = rs.wire_store(kind)
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    q = [(rs.MAGIC, b"\xff", 2**63, 0), (rs.MAGIC, b"\xff", 40, 7)]
    check_answer(eng, store, ko.OracleStore(store), q, what=kind)
    bigger = rs.wire_store({"small": "mid", "mid": "large", "large": "large"}[kind], seed=9)
    ops = [(k, v) for k, v in zip(bigger.keys.tolist()[:12], bigger.vals.tolist()[:12])]
    ops.append((rs.ik(b"/w/zzz", 5), b"\x07" * ((1 << 16) + 5)))
    eng.apply_batch(ops)
    items = dict(zip(store.keys.tolist(), store.vals.tolist()))
    items.update(ops)
    cur = PackedStore.from_items(list(items.items()))
    check_answer(eng, cur, ko.OracleStore(cur), q, what=kind + " raised")


# ---- one engine, batches in flight ---------------------------------------------------------------------------------
def test_sequence_two_in_flight(eng, r1):
    """an R1 batch over > 1 024 tiles, an R3 batch of a few tiles, the R1 batch again: two in flight, then collected"""
    sh, _ = r1
    s3 = rs.r3_store()
    items = list(zip(sh.store.keys.tolist(), sh.store.vals.tolist())) + list(zip(s3.keys.tolist(), s3.vals.tolist()))
    store = PackedStore.from_items(items)
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    end = rs.MAGIC + b"/c9"  # the R1 cases end in front of it, R3 starts behind it ('/r' > '/c')
    b1 = [(s, end, rev, lim) for s, e, rev, lim in rs.r1_requests(sh) if s < e]
    b3 = rs.r3_requests(s3)[1:]
    e1, e3 = expected(store, st, b1), expected(store, st, b3)
    for mode in (KB_OUT_HOST, KB_OUT_DEVICE):
        p1 = eng.range_submit(b1, mode)
        p3 = eng.range_submit(b3, mode)
        r1_ = p1.collect()
        p1b = eng.range_submit(b1, mode)
        r3_ = p3.collect()
        r1b = p1b.collect()
        for r, exps in ((r1_, e1), (r3_, e3), (r1b, e1)):
            emit = np.concatenate([x.emit for x in exps]).astype(np.uint64)
            assert r.req_examined.tolist() == [x.examined for x in exps]
            got = r.device_array("rec_idx", np.uint32) if mode == KB_OUT_DEVICE else r.rec_idx
            assert got.astype(np.uint64).tolist() == emit.tolist()
            image = arena_image(store, emit)
            raw = (eng.read_device(r.bytes_ptr, r.n_bytes, sync=False) if mode == KB_OUT_DEVICE
                   else r.arena[: r.n_bytes].tobytes())
            assert r.n_bytes == len(image) and raw == image
            r.close()


# ---- the fuzz stores up to four tiles and short-key synthetics ----------------------------------------------------
@pytest.mark.parametrize("seed", range(4))
def test_fuzz_store_tiles(eng, seed):
    store = fuzz.fuzz_store(200 + seed, n_keys=60 + 400 * seed)
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    reqs = [(s, t, rev, lim) for s, t in fuzz.fuzz_bounds(store, seed) for rev in (0, 23, 2**64 - 1) for lim in (0, 3)]
    check_ranges(eng, store, st, reqs)
    check_compact(eng, store, st, b"\x00", b"\xff" * 4, 35)
    eng.set_compact_revision(None)


@pytest.mark.parametrize("lu,lv,only", [(64, 64, None), (30, 9, b"pods"), (256, 300, None)])
def test_synthetic_key_lengths(eng, lu, lv, only):
    store, meta = synth.gen_store(3000, 5, lu, lv, 7, config_id=4, tomb_frac=0.1, only_resource=only)
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    check_ranges(eng, store, st, [(LO, HI, meta.last_rev, 0), (LO, HI, meta.read_rev, 0), (LO, HI, meta.read_rev, 17)])
    check_compact(eng, store, st, LO, HI, meta.read_rev)
    eng.set_compact_revision(None)
