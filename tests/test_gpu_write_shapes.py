"""The write path (kb_store.cu: kb_apply_batch, kb_expire, k_key_exists, k_dir_merge, the fix list, k_summarize,
slab_reserve, store_compact_layout / k_relocate, kb_dump / kb_restore) on sequences built to put its fixed boundaries
on purpose (tests/write_shapes.py; tests/test_write_shapes.py asserts which classes each shape reaches).

After every step of every shape: kb_store_info equals the heap model exactly; ranges over the whole key space at
several read revisions and limits, plus requests that start at the records the batch fixed, the sweep plain and as a
TTL sweep, and point reads of every touched user key equal the C oracle on the model's map.  At chosen steps kb_dump
equals the canonical image byte for byte, and that image restores in a second engine that answers the same.  Batches
also run between a submit and its collect, and invalid batches change nothing."""
from __future__ import annotations

import numpy as np
import pytest

from kubebrain_b200._lib import (KB_EINVAL, KB_ELIMIT, KB_OP_DEL, KB_OP_PUT, KB_OUT_DEVICE, KB_OUT_HOST, Engine,
                                 KbError, KbWriteOp, lib)
from kubebrain_b200.packed import PackedStore
from oracle import binding as ko
from tests import write_shapes as ws
from tests.test_gpu_parity import check_compact, check_gets, check_ranges

pytestmark = pytest.mark.gpu

LO, HI = b"", b"\xff" * 4  # the whole key space: the empty key is a record in W2
SHAPES = {s.name: s for s in ws.all_shapes()}


@pytest.fixture(scope="module")
def engs():
    a, b = Engine(0), Engine(0)
    yield a, b
    a.close()
    b.close()


def _store(m: ws.HeapModel) -> PackedStore:
    return PackedStore.from_items(m.sorted_items())


def check_answers(eng: Engine, m: ws.HeapModel, revs, touched=(), fixed=(), what=""):
    assert eng.store_info() == m.info(), what
    cur = _store(m)
    st = ko.OracleStore(cur)
    eng.set_compact_revision(None)
    reqs = [(LO, HI, rev, lim) for rev in revs for lim in (0, 3)]
    step = max(1, len(fixed) // 48)
    reqs += [(k, HI, revs[0], 5) for k in list(fixed)[::step]] + [(k, HI, revs[-1], 0) for k in list(fixed)[::step * 4]]
    check_ranges(eng, cur, st, reqs)
    check_compact(eng, cur, st, LO, HI, revs[1])
    check_compact(eng, cur, st, LO, HI, revs[1], timeout_rev=revs[1], support_ttl=False)
    eng.set_compact_revision(None)
    uks = sorted({ws.user_key(k) for k in touched} - {None})
    uks = uks[:: max(1, len(uks) // 200)]
    if uks:
        check_gets(eng, cur, st, [(uk, r) for uk in uks for r in (0,) + tuple(revs[1:])])


def check_dump(engs, m: ws.HeapModel, path: str, what=""):
    a, b = engs
    a.set_compact_revision(None)
    a.dump(path)
    m.dump()
    blob = open(path, "rb").read()
    img = ws.dump_image(m.sorted_items())
    got, exp = ws.parse_dump(blob), ws.parse_dump(img)
    assert got.sums_ok, what
    for f in ws.HEADER_FIELDS:
        if f not in ("max_kv_chunks", "sum_dir", "sum_keys", "sum_vals"):
            assert got.header[f] == exp.header[f], (what, f)
    assert got.header["max_kv_chunks"] >= exp.header["max_kv_chunks"], what  # it only grows
    assert (got.koff16, got.klen, got.voff16, got.vlen) == (exp.koff16, exp.klen, exp.voff16, exp.vlen), (what, "dir")
    assert blob[ws.DUMP_HEADER.size:] == img[ws.DUMP_HEADER.size:], (what, "slabs")
    assert a.store_info() == m.info(), what
    with open(path + ".img", "wb") as f:
        f.write(img)
    b.restore(path + ".img")
    check_answers(b, ws.HeapModel(m.sorted_items()), (2**64 - 1, 6, 1), what=what + " restored")


def run_shape(engs, shape: ws.WShape, path: str):
    eng = engs[0]
    eng.load_sorted(PackedStore.from_items(shape.start))
    m = ws.HeapModel(shape.start)
    check_answers(eng, m, shape.revs, what=shape.name + " start")
    stream = None
    for i, s in enumerate(shape.steps):
        what = "%s step %d (%s)" % (shape.name, i, s.what)
        if s.stream == "open":
            stream = eng.compact_stream(LO, HI, shape.revs[1])
            m.pinned = True
        elif s.stream == "close":
            stream.close()
            stream = None
            m.pinned = False
        before = dict(m.items)
        touched = ()
        if s.kind == "apply":
            eng.apply_batch(s.ops)
            m.apply(s.ops)
            touched = {op[0] for op in s.ops}
        elif s.kind == "expire":
            assert eng.expire(s.now) == m.expire(s.now)[0], what
            touched = set(before) - set(m.items)
        elif s.kind == "reload":
            eng.load_sorted(_store(m))
            m.install(m.items)
        else:
            eng.set_compact_revision(None)
            eng.dump(path)
            eng.restore(path)
            m.dump()
            m.install(m.items)
        eng.set_compact_revision(None)
        if stream is None:
            ak = sorted(m.items)
            fixed = [ak[i] for i, _ in ws.fixed_records(before, m.items)]
            check_answers(eng, m, shape.revs, touched, fixed, what)
        else:  # the stream pins the heap: what this step checks is that the trigger waited
            assert eng.store_info() == m.info(), what
        if s.dump:
            check_dump(engs, m, path, what)
            check_answers(eng, m, shape.revs, what=what + " after the dump")
    if stream is not None:
        stream.close()


@pytest.mark.parametrize("name", [n for n, s in SHAPES.items() if not s.slow])
def test_write_shape(engs, tmp_path, name):
    run_shape(engs, SHAPES[name], str(tmp_path / "w.kbd"))


@pytest.mark.parametrize("name", [n for n, s in SHAPES.items() if s.slow])
def test_write_shape_large(engs, tmp_path, name):
    """200 000 inserts into 1 000 records; the displaced trigger over 131 072 records (the N / 32 branch)"""
    run_shape(engs, SHAPES[name], str(tmp_path / "w.kbd"))


def test_empty_value_replacement_dumps_canonically(engs, tmp_path):
    """Put(k, v) over a 0-byte value appends v out of key order but adds to no trigger counter: the dump must still
    be canonical and restore (it used to write a non-contiguous directory that kb_restore refused)"""
    a, b = engs
    items = [(ws.ik(b"/e/%d" % i, 5), b"" if i in (2, 5, 9) else b"val %d" % i) for i in range(10)]
    for ops in ([(items[2][0], b"now longer")], [(items[5][0], b"")], [(items[9][0], b"last")]):
        a.load_sorted(PackedStore.from_items(items))
        m = ws.HeapModel(items)
        a.apply_batch(ops)
        m.apply(ops)
        path = str(tmp_path / "e.kbd")
        a.dump(path)
        b.restore(path)
        assert b.store_info() == m.info()
        assert ws.parse_dump(open(path, "rb").read()).items() == m.sorted_items()


# ---- batches between a submit and its collect -------------------------------------------------------------------------
def test_batches_between_submit_and_collect():
    """range batches (host and device answers) and point reads submitted on the old snapshot, then a batch that grows
    both slabs without compacting and one that grows both and compacts the layout, then the collects: the answers are
    the old snapshot's, and the next ones the new snapshot's"""
    # a fresh engine: its slabs have the capacity a fresh load allocates, which HeapModel restates (dbuf_ensure), so the
    # model's count of slab_reserve growths is the device's.  Growth itself has no observable of its own; what shows
    # it worked is that every answer after batch 1 comes from slabs slab_reserve copied (no compaction rewrote them).
    eng = Engine(0)
    start = [(ws.ik(b"/s/%06d" % (i * 10), 5), b"s%d" % i * (i % 5)) for i in range(3000)]
    m = ws.HeapModel(start)
    old = _store(m)
    st = ko.OracleStore(old)
    reqs = [(LO, HI, 2**64 - 1, 0), (LO, HI, 5, 7), (ws.ik(b"/s/001000", 0), HI, 2**64 - 1, 100)]
    gets = [(b"/s/%06d" % (i * 10), 0) for i in range(0, 3000, 37)] + [(b"/s/000015", 0)]
    batches = [
        [(ws.ik(b"/s/%06d" % (i * 10 + 5), 6), b"merged") for i in range(0, 3000, 3)] +
        [(k, None) for k, _ in start[::7]] + [(k, b"replaced") for k, _ in start[1::7]],
        [(ws.ik(b"/s/%06d" % (i * 10 + 7), 6), b"G" * 300) for i in range(3000)] +
        [(ws.ik(b"/t/%06d" % i, 6), b"H" * 200) for i in range(2000)],
    ]
    try:
        eng.load_sorted(old)
        eng.set_compact_revision(None)
        seen = []
        for ops in batches:
            exps = [ko.range_(st, *q) for q in reqs]
            ph, pd = eng.range_submit(reqs, KB_OUT_HOST), eng.range_submit(reqs, KB_OUT_DEVICE)
            pg = eng.get_submit(gets)
            gk, gv = m.grows_k, m.grows_v
            eng.apply_batch(ops)
            f = m.apply(ops)
            seen.append((f["fired"], m.grows_k - gk, m.grows_v - gv))
            rh, rd, rg = ph.collect(), pd.collect(), pg.collect()
            for q, x in enumerate(exps):
                assert rh.rec_indices(q).astype(np.uint64).tolist() == x.emit.tolist(), q
                assert rh.kvs(q) == x.kvs(old), q
            emit = np.concatenate([x.emit for x in exps]).astype(np.uint64)
            assert rd.device_array("rec_idx", np.uint32).astype(np.uint64).tolist() == emit.tolist()
            image = b"".join(ws.pad16(old.keys[int(i)]) + ws.pad16(old.vals[int(i)]) for i in emit)
            assert rd.n_bytes == len(image) and eng.read_device(rd.bytes_ptr, rd.n_bytes, sync=False) == image
            for i, (k, rev) in enumerate(gets):
                idx, mod = ko.get(st, k, rev)
                assert int(rg.status[i]) == (0 if idx >= 0 else 1), i
                if idx >= 0:
                    assert int(rg.rec_idx[i]) == idx and rg.value(i) == old.vals[idx], i
            rh.close(), rd.close(), rg.close()
            assert eng.store_info() == m.info()  # after batch 2 this is the compacted layout's size
            old = _store(m)
            st = ko.OracleStore(old)
            check_ranges(eng, old, st, reqs)
            check_gets(eng, old, st, gets)
        # what the model says the batches do: batch 1 grows both slabs and leaves them in place, batch 2 grows both
        # again and compacts the layout
        assert seen == [(None, 1, 1), (("displaced",), 1, 1)]
    finally:
        eng.close()


# ---- invalid batches change nothing -------------------------------------------------------------------------------------
def _raw_apply(eng: Engine, ops):
    """kb_apply_batch with raw kb_write_op fields: (type, key, key_len, val, val_len, expire)"""
    arr = (KbWriteOp * len(ops))()
    keep = []
    for i, (t, k, kl, v, vl, ex) in enumerate(ops):
        keep += [k, v]
        arr[i].type, arr[i].key, arr[i].key_len, arr[i].val, arr[i].val_len, arr[i].expire_unix = t, k, kl, v, vl, ex
    return lib().kb_apply_batch(eng._ctx, arr, len(ops))


def test_invalid_ops_change_nothing(engs):
    eng = engs[0]
    T = ws.T0
    start = [(ws.ik(b"/i/%04d" % i, 5), b"i%d" % i) for i in range(200)]
    eng.load_sorted(PackedStore.from_items(start))
    m = ws.HeapModel(start)
    ttl_key = start[10][0]
    eng.apply_batch([(ttl_key, b"due", T)])
    m.apply([(ttl_key, b"due", T)])
    big = b"k" * 65536
    good = [(KB_OP_PUT, start[10][0], len(start[10][0]), b"no ttl any more", 15, 0),  # would cancel the TTL
            (KB_OP_DEL, start[3][0], len(start[3][0]), None, 0, 0),
            (KB_OP_PUT, b"new key", 7, b"x", 1, T)]
    bad = {"65 536-byte key": ((KB_OP_PUT, big, len(big), b"v", 1, 0), KB_ELIMIT),
           "bad type": ((7, b"k", 1, b"v", 1, 0), KB_EINVAL),
           "null value with a length": ((KB_OP_PUT, b"k", 1, None, 5, 0), KB_EINVAL)}
    for name, (op, code) in bad.items():
        for ops in ([op], good + [op], [op] + good):
            assert _raw_apply(eng, ops) == code, name
            check_answers(eng, m, (2**64 - 1, 5, 1), touched=[o[1] for o in good], what=name)
    with pytest.raises(KbError) as ei:
        eng.apply_batch([(big, None)])  # a delete of a key no record can hold is refused too
    assert ei.value.code == KB_ELIMIT
    assert eng.expire(T) == m.expire(T)[0] == 1  # the TTL survived every refused batch
    check_answers(eng, m, (2**64 - 1, 5, 1), touched=[ttl_key], what="after the expiry")
