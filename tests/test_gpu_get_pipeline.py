"""Point reads as lane batches (kb_get_submit / kb_get_collect, and kb_get_batch built on them) against the CPU oracle:
every out mode -- the values-only arena of kb_get_batch, the RangeResponse.kvs elements of the wire mode -- on the
reference's table test, fuzz stores, the R3 extremes and a synthetic store; batches in flight beside range batches on
every lane count, with the other entry points called between submission and collection; the error paths."""
from __future__ import annotations

import ctypes
import os
import random
import struct

import numpy as np
import pytest

from kubebrain_b200 import synth, wire
from kubebrain_b200._lib import (GET_FOUND, GET_NOT_FOUND, GET_TOMBSTONE, KB_EINVAL, KB_ELIMIT, KB_ESTATE,
                                 KB_OUT_COUNT, KB_OUT_DEVICE, KB_OUT_HOST, KB_WIRE_ETCD_EVENTS, KB_WIRE_ETCD_KVS,
                                 Engine, KbError, KbGetReq, lib)
from kubebrain_b200.coder import NormalCoder, prefix_end
from kubebrain_b200.packed import PackedStore
from oracle import binding as ko
from tests import fuzz
from tests.range_shapes import r3_store
from tests.refmodel import MiniBackend
from tests.test_gpu_lanes import _check_any

pytestmark = pytest.mark.gpu

CODER = NormalCoder()
MAGIC = b"\x57\xfb\x80\x8b"
LO, HI = CODER.encode_object_key(b"/registry/", 0), CODER.encode_object_key(b"/registry0", 0)
MODES = [KB_OUT_HOST, KB_OUT_DEVICE, KB_OUT_HOST | KB_WIRE_ETCD_KVS, KB_OUT_DEVICE | KB_WIRE_ETCD_KVS]
WIRE_HOST = KB_OUT_HOST | KB_WIRE_ETCD_KVS


def _pad16(n: int) -> int:
    return (n + 15) & ~15


def expected(st, reqs):
    """[(status, record index or -1, mod_rev)] of every read, by the oracle's backend.get"""
    out = []
    for k, rev in reqs:
        idx, mod = ko.get(st, k, rev)
        out.append((GET_FOUND, idx, mod) if idx >= 0 else (GET_TOMBSTONE, -1, mod) if idx == -2 else (GET_NOT_FOUND, -1, 0))
    return out


def check(eng, res, store, st, reqs, mode):
    """one collected answer against the oracle, in the layout its mode promises"""
    exp = expected(st, reqs)
    is_wire = bool(mode & KB_WIRE_ETCD_KVS)
    assert res.n == len(reqs) and res.wire == is_wire
    if res.on_device:
        # complete at collect: read back on the legacy default stream with no wait on the context's streams
        res.arena = np.frombuffer(eng.read_device(res.bytes_ptr, res.n_bytes, sync=False), np.uint8)
    elif res.n_bytes == 0:
        res.arena = np.zeros(0, np.uint8)
    off = 0
    for i, ((k, rev), (s, idx, mod)) in enumerate(zip(reqs, exp)):
        assert int(res.status[i]) == s and int(res.mod_rev[i]) == mod, (i, k[:40], rev)
        if s == GET_FOUND:
            v = store.vals[idx]
            assert int(res.rec_idx[i]) == idx and int(res.val_len[i]) == len(v)
            assert res.value(i) == v, (i, k[:40], rev)
            if is_wire:
                el, eo = ko.wire_encode(st, [idx], ko.WIRE_KVS)
                assert int(res.elem_off[i]) == off and res.element(i) == el, (i, k[:40], rev)
                assert int(res.val_off[i]) == off + len(el) - len(v)  # the value ends the element
                off += len(el)
            else:
                assert int(res.val_off[i]) == off  # kb_get_batch: exclusive sum of the padded FOUND values before i
                off += _pad16(len(v))
        else:
            assert int(res.val_off[i]) == 0
            assert int(res.val_len[i]) == (9 if s == GET_TOMBSTONE else 0)
            if is_wire:
                assert int(res.elem_off[i]) == off and res.element(i) == b""
    assert res.n_bytes == off
    if is_wire:
        assert int(res.elem_off[len(reqs)]) == off
    res.close()


def reads_for(store: PackedStore, seed: int, cap: int = 4000):
    """every decodable record's user key at revision 0, at its revision, one below and one above, below the first and
    above the last revision; prefixes and extensions of stored keys; keys that are not stored"""
    rng = random.Random(seed)
    out = [(b"", 0), (b"/none", 0), (b"/registry/none", 5)]
    for k in store.keys.tolist():
        if len(k) < 13 or k[:4] != MAGIC or k[-9:-8] != b"$":
            continue
        uk, rev = k[4:-9], struct.unpack(">Q", k[-8:])[0]
        out += [(uk, 0), (uk, rev), (uk, max(rev - 1, 0) or 1), (uk, rev + 1), (uk, 1), (uk, 2**64 - 1)]
        if uk:
            out += [(uk[:-1], 0), (uk + b"\x00", rev)]
    if len(out) > cap:
        out = rng.sample(out, cap)
    return [r for r in out if len(r[0]) <= 65522]


def _all_modes(eng, store, st, reqs):
    for mode in MODES:
        check(eng, eng.get_submit(reqs, mode).collect(), store, st, reqs, mode)
    for mode in (KB_OUT_HOST, KB_OUT_DEVICE):
        check(eng, eng.get_batch(reqs, mode), store, st, reqs, mode)


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def test_backend_table(eng):
    """pkg/backend/backend_test.go:800-823 get cases on the reference's 10-key table, plus an update and a delete"""
    mb = MiniBackend(1000)
    revs = {}
    for i in range(10):
        revs[i], _ = mb.create(b"/registry/test/key/%05d" % i, b"val/%05d" % i)
    mb.update(b"/registry/test/key/00003", b"new", revs[3])
    mb.delete(b"/registry/test/key/00004")
    store = mb.snapshot()
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    reqs = reads_for(store, 1) + [(b"/registry/test/key/%05d" % i, r) for i, r in revs.items()]
    _all_modes(eng, store, st, reqs)
    # the serialized RangeResponse of backendShim.Get
    cur = mb.rev
    for k, rev in [(b"/registry/test/key/00009", 0), (b"/registry/test/key/00004", 0), (b"/nope", 0),
                   (b"/registry/test/key/00003", revs[3])]:
        idx, mod = ko.get(st, k, rev)
        if idx >= 0:
            el, _ = ko.wire_encode(st, [idx], ko.WIRE_KVS)
            want = ko.wire_range_head(max(cur, mod)) + el + ko.wire_range_tail(False, 1)
        else:
            want = ko.wire_range_head(cur) + ko.wire_range_tail(False, 0)
        assert wire.get_response(eng, k, rev, cur) == want
        assert wire.get_response(eng, k, rev, 7) == (ko.wire_range_head(max(7, mod)) + el + ko.wire_range_tail(False, 1)
                                                     if idx >= 0 else ko.wire_range_head(7) + ko.wire_range_tail(False, 0))


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_fuzz_stores(eng, seed):
    store = fuzz.fuzz_store(seed)
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    _all_modes(eng, store, st, reads_for(store, seed))


def test_r3_extremes(eng):
    """the 65 522-byte user key, empty values and a 1 MiB value, also read repeatedly in one batch"""
    store = r3_store()
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    reqs = reads_for(store, 3, cap=3000)
    big = [k[4:-9] for k in store.keys.tolist() if len(k) >= 65535 or b"/r3/big/m" in k]
    assert any(len(u) == 65522 for u in big)
    reqs += [(u, 0) for u in big] * 3
    _all_modes(eng, store, st, reqs)
    huge = max(big, key=len)
    with pytest.raises(KbError) as ei:
        eng.get_submit([(huge + b"x", 0)])
    assert ei.value.code == KB_ELIMIT


def test_synthetic_batches(eng):
    store, meta = synth.gen_store(1500, 3, 64, 90, 9, config_id=2, tomb_frac=0.1)
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    assert store.n >= 6000
    _all_modes(eng, store, st, reads_for(store, 4, cap=6000))
    found = [(u, 0) for u in dict.fromkeys(k[4:-9] for k in store.keys.tolist()) if ko.get(st, u, 0)[0] >= 0]
    rng = random.Random(5)
    shapes = {
        "empty": [],
        "one": found[:1],
        "100k_found": [found[rng.randrange(len(found))] for _ in range(100_000)],
        "all_missing": [(b"/registry/none/%d" % i, 0) for i in range(3000)],
        "repeated": [found[7]] * 5000,
    }
    for name, reqs in shapes.items():
        for mode in MODES:
            check(eng, eng.get_submit(reqs, mode).collect(), store, st, reqs, mode)
        check(eng, eng.get_batch(reqs, KB_OUT_HOST), store, st, reqs, KB_OUT_HOST)


@pytest.mark.parametrize("n_lanes", [1, 2, 3, 4])
def test_in_flight(monkeypatch, n_lanes):
    monkeypatch.setenv("KB_LANES", str(n_lanes))
    store, meta = synth.gen_store(1500, 3, 64, 90, 9, config_id=2, tomb_frac=0.1)
    p = b"/registry/pods/ns-00002/"
    ps, pe = CODER.encode_object_key(p, 0), CODER.encode_object_key(prefix_end(p), 0)
    ranges = [[(LO, HI, meta.read_rev, 0), (ps, pe, meta.last_rev, 5)], [(ps, pe, meta.last_rev, 0)]]
    keys = [k[4:-9] for k in store.keys.tolist()[::37]]
    gets = [[(k, 0) for k in keys], [(k, meta.read_rev) for k in keys[::2]] + [(b"/registry/none", 0)]]
    ev = synth.gen_events(2000, 256, 60, 5000)
    wat = synth.gen_watchers(40, 4, 5000, 6500)
    fan_start, fan_idx, _ = ko.fanout(ev, wat, threads=2)
    m = n_lanes + 1

    eng = Engine(0)
    eng.load_sorted(store)
    eng.watch_add_many(wat)
    items = dict(zip(store.keys.tolist(), store.vals.tolist()))
    cur, st = store, ko.OracleStore(store)
    rng = random.Random(n_lanes)
    # range and get batches interleaved, one more than there are lanes
    specs = [("g", gets[0], MODES[0]), ("r", ranges[0], KB_OUT_HOST), ("g", gets[1], MODES[3]), ("r", ranges[1], WIRE_HOST),
             ("g", gets[0], MODES[2]), ("g", gets[1], MODES[1])]
    orders = (list(range(m)), list(range(m))[::-1], list(range(0, m, 2)) + list(range(1, m, 2)))
    for step, what in enumerate(("watch", "page", "apply", "expire", "compaction", "watch")):
        order = orders[step % 3]
        batch = (specs[step:] + specs[:step])[:m]
        pend = [eng.get_submit(x, mode) if kind == "g" else eng.range_submit(x, mode) for kind, x, mode in batch]
        ops = []
        if what == "watch":
            got = eng.watch_match(ev)
            assert got.start.tolist() == fan_start.tolist() and got.event_idx.tolist() == fan_idx.tolist()
            got.close()
        elif what == "page":
            s = eng.range_stream((LO, HI, meta.last_rev, 0), KB_OUT_HOST, 300)
            page = s.next(1 << 16)
            exp = ko.range_(st, LO, HI, meta.last_rev, 0)
            assert page.rec_idx.astype(np.uint64).tolist() == exp.emit[: page.n_kvs].tolist()
            page.close()
            s.close()
        elif what == "apply":
            ops = [(k, None) for k in rng.sample(sorted(items), 20)] + [(sorted(items)[5], b"rewritten")]
        elif what == "expire":
            k = CODER.encode_object_key(b"/registry/ttl/%d" % step, meta.last_rev + 1)
            eng.apply_batch([(k, b"short-lived", 1000)])  # a write, then expire it: two snapshot changes
            assert eng.expire(2000) == 1
        else:  # new values for a third of the keys: their old bytes become garbage beyond the layout threshold
            ops = [(k, b"c" * rng.randint(0, 200)) for k in rng.sample(sorted(items), len(items) // 3)]
        if ops:
            eng.apply_batch(ops)
        # every pending answers on the snapshot it was submitted on
        for i in order:
            kind, x, mode = batch[i]
            if kind == "g":
                check(eng, pend[i].collect(), cur, st, x, mode)
            else:
                _check_any(eng, pend[i].collect(), cur, st, x, mode)
        for k, v in ops:
            if v is None:
                items.pop(k)
            else:
                items[k] = v
        cur = PackedStore.from_items(list(items.items()))
        st = ko.OracleStore(cur)
        # a get submitted after the write sees it
        reqs = gets[0] + [(k[4:-9], 0) for k, _ in ops]
        check(eng, eng.get_submit(reqs, MODES[step % 4]).collect(), cur, st, reqs, MODES[step % 4])
    # a get pending freed uncollected, then the lanes reused at full depth
    gone = eng.get_submit(gets[0], KB_OUT_DEVICE)
    gone.close()
    with pytest.raises(KbError):
        gone.collect()
    q = []
    for i in range(40):
        q.append(eng.get_submit(gets[i % 2], MODES[i % 4]) if i % 3 else eng.range_submit(ranges[0], KB_OUT_HOST))
        if len(q) > n_lanes:
            j = i - n_lanes
            p_ = q.pop(0)
            if j % 3:
                check(eng, p_.collect(), cur, st, gets[j % 2], MODES[j % 4])
            else:
                _check_any(eng, p_.collect(), cur, st, ranges[0], KB_OUT_HOST)
    for p_ in q:
        p_.close()
    # closed with get and range pendings outstanding; a new context answers
    left = [eng.get_submit(gets[0], KB_OUT_HOST), eng.range_submit(ranges[1], KB_OUT_DEVICE), eng.get_submit(gets[1], WIRE_HOST)]
    eng.close()
    del left
    e2 = Engine(0)
    e2.load_sorted(cur)
    check(e2, e2.get_submit(gets[1], WIRE_HOST).collect(), cur, st, gets[1], WIRE_HOST)
    e2.close()


def test_errors():
    L = lib()
    e = Engine(0)
    arr = (KbGetReq * 1)(KbGetReq(b"/a", 2, 0))
    hv, rv = ctypes.c_void_p(), ctypes.c_void_p()
    h, r = ctypes.byref(hv), ctypes.byref(rv)
    assert L.kb_get_submit(e._ctx, arr, 1, KB_OUT_HOST, h) == KB_ESTATE  # no store loaded
    store = fuzz.fuzz_store(1)
    e.load_sorted(store)
    for bad in (KB_OUT_COUNT, KB_OUT_HOST | KB_WIRE_ETCD_EVENTS, KB_OUT_DEVICE | KB_WIRE_ETCD_KVS | KB_WIRE_ETCD_EVENTS,
                KB_OUT_COUNT | KB_WIRE_ETCD_KVS, 7):
        assert L.kb_get_submit(e._ctx, arr, 1, bad, h) == KB_EINVAL, bad
    for bad in (KB_WIRE_ETCD_KVS, KB_OUT_DEVICE | KB_WIRE_ETCD_KVS, KB_OUT_COUNT):
        assert L.kb_get_batch(e._ctx, arr, 1, bad, r) == KB_EINVAL, bad
    assert L.kb_get_submit(None, arr, 1, KB_OUT_HOST, h) == KB_EINVAL
    assert L.kb_get_collect(None, None, r) == KB_EINVAL
    # cross-type collect is refused and leaves the pending open
    pg = e.get_submit([(b"/a", 0)])
    pr = e.range_submit([(LO, HI, 10, 0)])
    assert L.kb_range_collect(e._ctx, pg._h, r) == KB_EINVAL and not rv.value
    assert L.kb_get_collect(e._ctx, pr._h, r) == KB_EINVAL and not rv.value
    pr.collect().close()
    pg.collect().close()
    # the raw modes have no element offsets
    g = e.get_batch([(b"/a", 0)])
    eo = ctypes.POINTER(ctypes.c_uint64)()
    assert L.kb_get_elem_off(g._h, ctypes.byref(eo)) == KB_EINVAL
    g.close()
    with pytest.raises(KbError) as ei:
        e.get_batch([(b"k" * 65523, 0)])
    assert ei.value.code == KB_ELIMIT
    e.get_batch([(b"k" * 65522, 0)]).close()
    e.close()


def test_get_replay_cpp(tmp_path):
    """tests/cpp/get_replay_test.cpp, compiled here against the in-tree library and the oracle"""
    import shutil
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    gxx = shutil.which("g++")
    assert gxx, "the replay driver needs a C++ compiler"
    libdir, oradir = os.path.join(root, "kubebrain_b200"), os.path.join(root, "oracle")
    ko.build()
    exe = str(tmp_path / "get_replay_test")
    subprocess.check_call([gxx, "-O1", "-std=c++17", "-Wall", "-o", exe,
                           os.path.join(root, "tests", "cpp", "get_replay_test.cpp"),
                           "-L" + libdir, "-lkbb200", "-L" + oradir, "-lkboracle",
                           "-Wl,-rpath," + libdir, "-Wl,-rpath," + oradir])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "get replay OK" in r.stdout, r.stdout + r.stderr
