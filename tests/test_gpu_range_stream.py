"""kb_range_stream_open / _next / _close against the C oracle: the pages of a stream concatenate to the oracle's
unlimited answer in every output mode, each page is the greedy cut of whole groups within the byte budget, a snapshot
change between pages re-scans what has not been handed out yet, and pages interleave with the other work of a context."""
from __future__ import annotations

import os

import numpy as np
import pytest

from kubebrain_b200 import synth
from kubebrain_b200._lib import (KB_ECOMPACTED, KB_OUT_DEVICE, KB_OUT_HOST, KB_WIRE_ETCD_EVENTS, KB_WIRE_ETCD_KVS,
                                 Engine, KbError)
from kubebrain_b200.packed import PackedStore
from kubebrain_b200.scanner import Scanner
from oracle import binding as ko
from tests import fuzz
from tests import range_shapes as rs
from tests.test_gpu_range_shapes import arena_image

pytestmark = pytest.mark.gpu

MODES = {"host": KB_OUT_HOST, "device": KB_OUT_DEVICE, "kvs": KB_OUT_HOST | KB_WIRE_ETCD_KVS,
         "events": KB_OUT_DEVICE | KB_WIRE_ETCD_EVENTS}
ALL = 2**64 - 1
MAX_PAGES = 400


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def _pad16(n: int) -> int:
    return (n + 15) & ~15


def expected(store: PackedStore, st: ko.OracleStore, s: bytes, e: bytes, rev: int, mode: int):
    """the oracle's unlimited answer: emitted records, the answer's bytes, and each kv's arena bytes"""
    x = ko.range_(st, s, e, rev, 0)
    assert x.rc == 0
    emit = x.emit.astype(np.uint64)
    wire = mode & (KB_WIRE_ETCD_KVS | KB_WIRE_ETCD_EVENTS)
    if wire:
        image, off = ko.wire_encode(st, emit, ko.WIRE_KVS if wire == KB_WIRE_ETCD_KVS else ko.WIRE_EVENTS)
        sizes = np.diff(off.astype(np.int64))
    else:
        image = arena_image(store, emit)
        sizes = np.array([_pad16(len(store.keys[int(i)])) + _pad16(len(store.vals[int(i)])) for i in emit], np.int64)
    return emit, image, sizes


def greedy_cuts(sizes: np.ndarray, group: int, budget: int):
    """(a, b) of every page: the most whole groups (or the rest) within the budget, at least one group"""
    pre = np.concatenate([[0], np.cumsum(sizes)]).astype(object)
    n, a, out = len(sizes), 0, []
    while a < n:
        b = min(a + group, n)
        k = 2
        while b < n:
            c = min(a + k * group, n)
            if pre[c] - pre[a] > budget:
                break
            b, k = c, k + 1
        out.append((a, b))
        a = b
    return out


def page_parts(eng: Engine, page, mode: int):
    """(rec_idx, arena bytes, element offsets or None) of one page"""
    assert page.req_first.tolist() == [0, page.n_kvs] and page.req_count.tolist() == [page.n_kvs]
    assert page.req_examined.tolist() == [0]
    wire = mode & (KB_WIRE_ETCD_KVS | KB_WIRE_ETCD_EVENTS)
    if page.on_device:
        rec = page.device_array("rec_idx", np.uint32)
        arena = eng.read_device(page.bytes_ptr, page.n_bytes, sync=False)
        eo = page.device_array("elem_off", np.uint64) if wire else None
    else:
        rec = page.rec_idx.copy()
        arena = page.arena[: page.n_bytes].tobytes()
        eo = page.elem_off.copy() if wire else None
    return rec.astype(np.uint64), arena, eo


def drain(eng: Engine, stream, budget: int, mode: int, limit_pages: int = 1 << 30):
    out = []
    while len(out) < limit_pages:
        page = stream.next(budget)
        if page is None:
            break
        out.append(page_parts(eng, page, mode))
        page.close()
    return out


def check_stream(eng, store, st, s, e, rev, mode, group, budget, what=""):
    emit, image, sizes = expected(store, st, s, e, rev, mode)
    stream = eng.range_stream((s, e, rev, 0), mode, group)
    pages = drain(eng, stream, budget, mode)
    assert stream.next(budget) is None, what  # stays exhausted
    stream.close()
    cuts = greedy_cuts(sizes, group, budget)
    assert [len(r) for r, _, _ in pages] == [b - a for a, b in cuts], (what, "cuts")
    base = 0
    for (a, b), (rec, arena, eo) in zip(cuts, pages):
        assert rec.tolist() == emit[a:b].tolist(), (what, a)
        assert len(arena) == int(sizes[a:b].sum()), (what, a, "bytes")
        if eo is not None:
            assert (eo.astype(np.int64) + base).tolist() == (np.concatenate([[0], np.cumsum(sizes)])[a : b + 1]).tolist()
        base += len(arena)
    assert b"".join(p[1] for p in pages) == image, (what, "image")
    return cuts


def budgets(sizes: np.ndarray, group: int):
    g0 = int(sizes[:group].sum()) if len(sizes) else 16
    return [0, max(g0 - 1, 0), g0, g0 + 1, 3 * g0 + 5, ALL]


# ---- 1, 2: concatenation and cuts on the range-shape and fuzz stores -------------------------------------------------
def _shape_cases():
    r1 = rs.r1_store()
    r3 = rs.r3_store()
    return [("r1", r1.store, [(rs.MAGIC, b"\xff", rs.READ), (rs.MAGIC, b"\xff", rs.TTL - 50)]),
            ("r3", r3, [(rs.MAGIC, b"\xff", 2**63)]),
            ("fuzz0", fuzz.fuzz_store(300, n_keys=400), [(b"\x00", b"\xff" * 4, 0), (b"\x00", b"\xff" * 4, 23)]),
            ("fuzz1", fuzz.fuzz_store(301, n_keys=900), [(b"\x00", b"\xff" * 4, 2**64 - 1)])]


@pytest.fixture(scope="module")
def shapes():
    return [(name, store, ko.OracleStore(store), reqs) for name, store, reqs in _shape_cases()]


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("group", [1, 7, 300])
def test_pages_concatenate_to_the_answer(eng, shapes, mode, group):
    m = MODES[mode]
    for name, store, st, reqs in shapes:
        eng.load_sorted(store)
        eng.set_compact_revision(None)
        for s, e, rev in reqs:
            _, _, sizes = expected(store, st, s, e, rev, m)
            for b in budgets(sizes, group):
                if len(greedy_cuts(sizes, group, b)) > MAX_PAGES:
                    continue  # (near) one page per kv on a large answer: the small stores cover these budgets
                check_stream(eng, store, st, s, e, rev, m, group, b, what=(name, rev, b))


def test_wire_page_starts_on_every_alignment(eng):
    """group 1 and a zero budget: one element per page, so the pages start at every element offset of the answer"""
    store = rs.r3_store()
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    for m in (KB_OUT_HOST | KB_WIRE_ETCD_KVS, KB_OUT_HOST | KB_WIRE_ETCD_EVENTS):
        _, _, sizes = expected(store, st, rs.MAGIC, b"\xff", 2**63, m)
        starts = np.concatenate([[0], np.cumsum(sizes)])[:-1]
        assert set((starts % 16).tolist()) == set(range(16))
        cuts = check_stream(eng, store, st, rs.MAGIC, b"\xff", 2**63, m, 1, 0)
        assert len(cuts) == len(sizes)


def test_single_group_larger_than_the_budget(eng):
    """the 1 MiB value: a page of one group exceeds the budget; the last partial group ends the stream"""
    store = rs.r3_store()
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    for m in MODES.values():
        cuts = check_stream(eng, store, st, rs.MAGIC + b"/r3/big/", rs.MAGIC + b"/r3/big0", 2**63, m, 2, 1024)
        assert [b - a for a, b in cuts] == [2, 1]


def test_config2_full_range_at_16mib(eng):
    """BASELINE config 2 (1M records, 256-byte user keys, 2 KiB values): the whole range in 16 MiB pages"""
    store, meta = synth.gen_store(200000, 4, 256, 2048, 1000, config_id=2)
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    lo, hi = ko.encode_object_key(b"/registry/", 0), ko.encode_object_key(b"/registry0", 0)
    exp = ko.range_(st, lo, hi, meta.read_rev, 0)
    idx_all = exp.emit.astype(np.int64)
    koff, voff = store.keys.off.astype(np.int64), store.vals.off.astype(np.int64)
    assert ((koff[idx_all + 1] - koff[idx_all]) == 269).all() and ((voff[idx_all + 1] - voff[idx_all]) == 2048).all()
    per_kv = 272 + 2048
    stream = eng.range_stream((lo, hi, meta.read_rev, 0), KB_OUT_HOST, 300)
    a, n_pages = 0, 0
    while True:
        page = stream.next(16 << 20)
        if page is None:
            break
        nk = page.n_kvs
        assert nk == min(((16 << 20) // per_kv) // 300 * 300, len(idx_all) - a)
        assert page.rec_idx.astype(np.int64).tolist() == idx_all[a : a + nk].tolist()
        assert page.n_bytes == nk * per_kv
        img = page.arena[: page.n_bytes].reshape(nk, per_kv)
        for c in range(0, nk, 4096):
            sl = slice(c, min(c + 4096, nk))
            idx = idx_all[a + c : a + sl.stop]
            assert np.array_equal(img[sl, :269], store.keys.data[koff[idx][:, None] + np.arange(269)])
            assert not img[sl, 269:272].any()
            assert np.array_equal(img[sl, 272:], store.vals.data[voff[idx][:, None] + np.arange(2048)])
        a += nk
        n_pages += 1
        page.close()
    stream.close()
    assert a == len(idx_all) and n_pages > 20


# ---- 3: writes between pages -----------------------------------------------------------------------------------------
READ = 50


def _write_store(n_keys: int = 900):
    items = []
    for j in range(n_keys):
        uk = b"/w/%05d" % j + b"$x" * (j % 3)  # '$' inside some user keys
        items.append((rs.ik(uk, 0), rs.be(30 + j % 20)))
        for rev in (10 + j % 7, 30 + j % 20, 60 + j % 5):  # the last version is above the read revision
            items.append((rs.ik(uk, rev), bytes([j % 251]) * (1 + (j * 13 + rev) % 90)))
    return dict(items)


def _store_of(items: dict) -> PackedStore:
    return PackedStore.from_items(sorted(items.items()))


def test_writes_above_the_read_revision_leave_the_answer(eng):
    items = _write_store()
    store = _store_of(items)
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    s, e = rs.MAGIC + b"/w/", rs.MAGIC + b"/w0"
    for m in (KB_OUT_HOST, KB_OUT_DEVICE | KB_WIRE_ETCD_EVENTS):
        eng.load_sorted(store)
        emit, image, sizes = expected(store, st, s, e, READ, m)
        stream = eng.range_stream((s, e, READ, 0), m, 7)
        got = drain(eng, stream, 700, m, limit_pages=3)
        rng = np.random.default_rng(5)
        for wave in range(12):  # new versions, new keys, deletes of versions above READ: enough for a layout compaction
            ops = []
            for j in rng.choice(900, 200, replace=False).tolist():
                uk = b"/w/%05d" % j + b"$x" * (j % 3)
                ops.append((rs.ik(uk, 100 + wave), b"n" * (j % 40)))
                ops.append((rs.ik(uk, 60 + j % 5), None))
                ops.append((rs.ik(b"/w/%05d~new%d" % (j, wave), 70 + wave), b"k"))
            eng.apply_batch(ops)
            got += drain(eng, stream, 700, m, limit_pages=1)
        got += drain(eng, stream, 700, m)
        stream.close()
        assert np.concatenate([r for r, _, _ in got]).size == len(emit)
        assert b"".join(p[1] for p in got) == image


@pytest.mark.parametrize("kind", ["below", "expire"])
def test_writes_at_or_below_the_read_revision_show_in_the_rest(eng, kind):
    items = _write_store()
    if kind == "expire":
        ttl = {rs.ik(b"/w/%05d" % j + b"~ttl", 20): b"t" * 5 for j in range(0, 900, 9)}
        base = _store_of(items)
        eng.load_sorted(base)
        eng.apply_batch([(k, v, 1000) for k, v in ttl.items()])
        items.update(ttl)
    else:
        eng.load_sorted(_store_of(items))
    eng.set_compact_revision(None)
    store = _store_of(items)
    s, e = rs.MAGIC + b"/w/", rs.MAGIC + b"/w0"
    stream = eng.range_stream((s, e, READ, 0), KB_OUT_HOST, 7)
    first = drain(eng, stream, 900, KB_OUT_HOST, limit_pages=2)
    last_key = store.keys[int(first[-1][0][-1])]
    if kind == "expire":
        assert eng.expire(2000) == len(ttl)
        for k in ttl:
            del items[k]
    else:
        ops = [(rs.ik(b"/w/%05d" % j + b"~mid", 40), b"m" * 3) for j in range(0, 900, 5)]  # everywhere in the range
        ops += [(rs.ik(b"/w/%05d" % j, 10 + j % 7), None) for j in range(1, 900, 11)]  # visible versions removed
        eng.apply_batch(ops)
        for k, v in ops:
            if v is None:
                items.pop(k, None)
            else:
                items[k] = v
    new = _store_of(items)
    nst = ko.OracleStore(new)
    rest = drain(eng, stream, 900, KB_OUT_HOST)
    stream.close()
    emit, image, _ = expected(new, nst, last_key + b"\x00", e, READ, KB_OUT_HOST)
    assert np.concatenate([r for r, _, _ in rest]).tolist() == emit.tolist()
    assert b"".join(p[1] for p in rest) == image
    old_emit, old_image, _ = expected(store, ko.OracleStore(store), s, e, READ, KB_OUT_HOST)
    n_first = sum(len(r) for r, _, _ in first)
    assert np.concatenate([r for r, _, _ in first]).tolist() == old_emit[:n_first].tolist()


# ---- 4: other work between pages -------------------------------------------------------------------------------------
@pytest.mark.parametrize("lanes", [1, 2, 3, 4])
def test_pages_between_batches_watch_and_a_second_stream(lanes, monkeypatch):
    monkeypatch.setenv("KB_LANES", str(lanes))
    e = Engine(0)
    try:
        store = fuzz.fuzz_store(310, n_keys=1500)
        st = ko.OracleStore(store)
        e.load_sorted(store)
        full = (b"\x00", b"\xff" * 4)
        batch = [(a, b, rev, lim) for a, b in fuzz.fuzz_bounds(store, 3) for rev in (0, 23) for lim in (0, 3)]
        bexp = [ko.range_(st, *q) for q in batch]
        wid = e.watch_add(b"/", 0)
        ev = fuzz.fuzz_events(4)
        mexp = e.watch_match(ev).event_idx.tolist()
        for m in (KB_OUT_HOST, KB_OUT_DEVICE | KB_WIRE_ETCD_KVS):
            emit1, img1, _ = expected(store, st, *full, ALL, m)
            emit2, img2, _ = expected(store, st, *full, 23, m)
            s1 = e.range_stream((*full, ALL, 0), m, 7)
            s2 = e.range_stream((*full, 23, 0), m, 300)
            got1, got2 = [], []
            while True:
                pend = [e.range_submit(batch, KB_OUT_HOST) for _ in range(lanes)]
                a = drain(e, s1, 2000, m, limit_pages=1)
                b = drain(e, s2, 500, m, limit_pages=1)
                got1 += a
                got2 += b
                mr = e.watch_match(ev)
                assert mr.event_idx.tolist() == mexp
                mr.close()
                for p in pend:
                    r = p.collect()
                    for q, x in enumerate(bexp):
                        assert r.rec_indices(q).astype(np.uint64).tolist() == x.emit.tolist()
                    r.close()
                if not a and not b:
                    break
            s1.close()
            s2.close()
            assert len(emit1) > 500 and len(emit2) > 100
            assert np.concatenate([r for r, _, _ in got1]).tolist() == emit1.tolist()
            assert b"".join(p[1] for p in got1) == img1
            assert np.concatenate([r for r, _, _ in got2]).tolist() == emit2.tolist()
            assert b"".join(p[1] for p in got2) == img2
        e.watch_del(wid)
    finally:
        e.close()


# ---- 5: lifecycle ----------------------------------------------------------------------------------------------------
def test_lifecycle(eng):
    store = fuzz.fuzz_store(320, n_keys=300)
    st = ko.OracleStore(store)
    eng.load_sorted(store)
    eng.set_compact_revision(None)
    k0 = store.keys[0]
    for s, e in ((k0, k0), (b"\x7f", b"\x00"), (b"\x02", b"\x03")):  # empty, reversed, no record
        stream = eng.range_stream((s, e, ALL, 0), KB_OUT_HOST, 300)
        assert stream.next(ALL) is None and stream.next(0) is None
        stream.close()
    eng.set_compact_revision(30)
    with pytest.raises(KbError) as ei:
        eng.range_stream((b"\x00", b"\xff", 29, 0), KB_OUT_HOST, 300)
    assert ei.value.code == KB_ECOMPACTED
    assert "range stream revision 29 less than compact revision 30" in str(ei.value)
    msgs = list(Scanner(eng).range_stream_paged(b"\x00", b"\xff", 29))
    assert msgs == list(Scanner(eng).range_stream(b"\x00", b"\xff", 29)) and len(msgs) == 1
    eng.set_compact_revision(None)
    # close before the end, pages outliving their stream
    stream = eng.range_stream((b"\x00", b"\xff" * 4, ALL, 0), KB_OUT_DEVICE, 3)
    p1, p2 = stream.next(64), stream.next(64)
    stream.close()
    emit, _, _ = expected(store, st, b"\x00", b"\xff" * 4, ALL, KB_OUT_DEVICE)
    r = np.concatenate([page_parts(eng, p, KB_OUT_DEVICE)[0] for p in (p1, p2)])
    assert r.tolist() == emit[: len(r)].tolist()
    p1.close(), p2.close()
    # the paged scanner yields the messages of the one-shot one
    for rev in (0, 23):
        assert list(Scanner(eng).range_stream_paged(b"\x00", b"\xff" * 4, rev, 4096)) == \
            list(Scanner(eng).range_stream(b"\x00", b"\xff" * 4, rev))


def test_close_context_with_open_streams():
    e = Engine(0)
    e.load_sorted(fuzz.fuzz_store(321, n_keys=200))
    s1 = e.range_stream((b"\x00", b"\xff" * 4, ALL, 0), KB_OUT_HOST, 1)
    s2 = e.range_stream((b"\x00", b"\xff" * 4, ALL, 0), KB_OUT_DEVICE | KB_WIRE_ETCD_EVENTS, 1)
    p = s1.next(0)
    assert p is not None and p.n_kvs == 1
    p.close()
    e.close()
    s1.close(), s2.close()  # the context already freed them


# ---- 6: the shim's call sequence -------------------------------------------------------------------------------------
def test_stream_replay_cpp(tmp_path):
    """tests/cpp/stream_replay_test.cpp, compiled here against the in-tree library and the oracle"""
    import shutil
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    gxx = shutil.which("g++")
    assert gxx, "the replay driver needs a C++ compiler"
    libdir, oradir = os.path.join(root, "kubebrain_b200"), os.path.join(root, "oracle")
    ko.build()
    exe = str(tmp_path / "stream_replay_test")
    subprocess.check_call([gxx, "-O1", "-std=c++17", "-Wall", "-o", exe,
                           os.path.join(root, "tests", "cpp", "stream_replay_test.cpp"),
                           "-L" + libdir, "-lkbb200", "-L" + oradir, "-lkboracle",
                           "-Wl,-rpath," + libdir, "-Wl,-rpath," + oradir])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "stream replay OK" in r.stdout, r.stdout + r.stderr
