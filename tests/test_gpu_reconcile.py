"""kb_reconcile (kubebrain_b200/csrc/kb_reconcile.cu) on every shape of tests/reconcile_shapes.py, in both value-heap
placements.  For every call: the dry-run diff equals the merge model's and leaves the snapshot byte for byte as it was,
the real diff equals the model's, kb_store_info equals the heap model after the diff's batch, and ranges, sweeps, point
reads and the dump match the oracle on the model's map.  A walk leaves the snapshot equal to the engine's items.  Open
compaction and range streams, a range batch in flight and TTL keys see exactly the effect of one kb_apply_batch of the
diff; refused calls change nothing."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from kubebrain_b200 import _lib
from kubebrain_b200._lib import KB_OUT_HOST, Engine, KbError
from kubebrain_b200.packed import PackedStore
from oracle import binding as ko
from tests import reconcile_shapes as rs
from tests import write_shapes as ws
from tests.test_gpu_write_shapes import HI, LO, check_answers, check_dump

pytestmark = pytest.mark.gpu

SHAPES = {s.name: s for s in rs.all_shapes()}
REVS = (2**64 - 1, 5, 1)


@pytest.fixture(scope="module", params=[False, True], ids=["hbm", "host_values"])
def engs(request):
    a, b = Engine(0, host_values=request.param), Engine(0, host_values=request.param)
    yield a, b
    a.close()
    b.close()


def _load(eng, sh: rs.RShape) -> ws.HeapModel:
    eng.load_sorted(PackedStore.from_items(sh.mirror))
    eng.set_compact_revision(None)
    m = ws.HeapModel(sh.mirror)
    if sh.ttl:
        ops = [(k, dict(sh.mirror)[k], t) for k, t in sorted(sh.ttl.items())]
        eng.apply_batch(ops)
        m.apply(ops)
    return m


def _got(r):
    return list(zip(r.kinds.tolist(), r.keys(), r.src_idx.tolist()))


def _call(eng, m: ws.HeapModel, s, e, inp, what, dry_first=True):
    """one dry run and one real call over [s, e); the model follows the real one"""
    exp = rs.diff(m.items, inp, s, e)
    span = len([k for k in m.items if s <= k < e]) if s < e else 0
    if dry_first:
        info = eng.store_info()
        r = eng.reconcile(s, e, inp, dry_run=True)
        assert _got(r) == exp, what + " dry"
        assert eng.store_info() == info == m.info(), what
    r = eng.reconcile(s, e, inp)
    assert _got(r) == exp, what
    assert (r.n_engine, r.n_mirror, r.n_diff) == (len(inp), span, len(exp)), what
    assert (r.n_missing, r.n_extra, r.n_changed) == tuple(sum(1 for x in exp if x[0] == k) for k in (1, 2, 3)), what
    m.apply(rs.ops_of(exp, inp))
    assert eng.store_info() == m.info(), what
    return exp


def run_shape(engs, sh: rs.RShape, path: str):
    eng = engs[0]
    m = _load(eng, sh)
    engine = dict(sh.engine)
    if not sh.chunks:
        inp = rs.interval_items(engine, sh.start, sh.end)
        # the dry run leaves the snapshot byte for byte as it was
        eng.dump(path + ".a")
        m.dump()
        r = eng.reconcile(sh.start, sh.end, inp, dry_run=True)
        eng.dump(path + ".b")
        assert open(path + ".a", "rb").read() == open(path + ".b", "rb").read(), sh.name
        assert _got(r) == rs.diff(m.items, inp, sh.start, sh.end)
        d = _call(eng, m, sh.start, sh.end, inp, sh.name, dry_first=False)
        touched = [k for _, k, _ in d]
        check_answers(eng, m, REVS, touched, touched[:: max(1, len(touched) // 64)], sh.name)
    else:
        for ch in sh.chunks:
            m = _load(eng, sh)
            for i, (s, e, inp) in enumerate(rs.walk(engine, sh.start, sh.end, ch)):
                _call(eng, m, s, e, inp, "%s chunk %d call %d" % (sh.name, ch, i), dry_first=i % 5 == 0)
            # after the walk the interval holds the engine's items, the rest is as it was
            assert rs.interval_items(m.items, sh.start, sh.end) == rs.interval_items(engine, sh.start, sh.end)
            check_answers(eng, m, REVS, what="%s after the walk of %d" % (sh.name, ch))
    check_dump(engs, m, path, sh.name)


@pytest.mark.parametrize("name", [n for n, s in SHAPES.items() if not s.interplay and not s.slow])
def test_reconcile_shape(engs, tmp_path, name):
    run_shape(engs, SHAPES[name], str(tmp_path / "r.kbd"))


@pytest.mark.parametrize("name", [n for n, s in SHAPES.items() if not s.interplay and s.slow])
def test_reconcile_shape_large(engs, tmp_path, name):
    run_shape(engs, SHAPES[name], str(tmp_path / "r.kbd"))


# ---- interplay --------------------------------------------------------------------------------------------------------
def _pages(stream, first=None):
    out = []
    while True:
        p = stream.next(1 << 12)
        if p is None:
            return out
        out.append((p.first, p.rec_idx.tolist(), p.victim_class.tolist(), p.keys(), p.guards()))
        if first is not None and len(out) == first:
            return out


def test_reconcile_under_compaction_stream(engs):
    """the stream's later pages equal those taken without the reconcile; the layout compaction waits for the close"""
    a, b = engs
    sh = SHAPES["interplay compact stream"]
    inp = rs.interval_items(dict(sh.engine), sh.start, sh.end)
    _load(b, sh)
    sb = b.compact_stream(LO, HI, 5)
    ref = _pages(sb)
    sb.close()
    m = _load(a, sh)
    st = a.compact_stream(LO, HI, 5)
    m.pinned = True
    got = _pages(st, first=1)
    _call(a, m, sh.start, sh.end, inp, sh.name)
    got += _pages(st)
    assert got == ref
    st.close()
    m.pinned = False
    check_answers(a, m, REVS, what=sh.name)


def _stream_all(eng, st, first=None):
    out = []
    while True:
        p = st.next(1 << 10)
        if p is None:
            return out
        out += p.kvs(0)
        p.close()
        if first is not None:
            return out


@pytest.mark.parametrize("name", ["interplay range stream", "interplay range stream, empty diff"])
def test_reconcile_under_range_stream(engs, name):
    """an open range stream re-scans after a non-empty diff only; what it hands out after that is the new snapshot's"""
    a, b = engs
    sh = SHAPES[name]
    inp = rs.interval_items(dict(sh.engine), sh.start, sh.end)
    req = (LO, HI, 2**64 - 1, 0)
    _load(b, sh)
    sb = b.range_stream(req)
    head_b = _stream_all(b, sb, first=1)
    n0 = b.launch_count()
    tail_b = _stream_all(b, sb)
    plain = b.launch_count() - n0
    sb.close()
    m = _load(a, sh)
    sa = a.range_stream(req)
    head = _stream_all(a, sa, first=1)
    assert head == head_b
    d = _call(a, m, sh.start, sh.end, inp, name, dry_first=False)
    n0 = a.launch_count()
    tail = _stream_all(a, sa)
    sa.close()
    if not d:
        assert tail == tail_b and a.launch_count() - n0 == plain  # no re-scan
    else:
        assert a.launch_count() - n0 > plain
        cur = PackedStore.from_items(m.sorted_items())
        last = ws.ik(head[-1][0], head[-1][2]) + b"\x00"
        exp = ko.range_(ko.OracleStore(cur), last, HI, 2**64 - 1, 0)
        assert tail == exp.kvs(cur)


def test_reconcile_between_submit_and_collect(engs):
    """a range batch submitted before the reconcile answers on the old snapshot"""
    a, _ = engs
    sh = SHAPES["interplay range batch"]
    inp = rs.interval_items(dict(sh.engine), sh.start, sh.end)
    m = _load(a, sh)
    old = PackedStore.from_items(m.sorted_items())
    reqs = [(LO, HI, 2**64 - 1, 0), (LO, HI, 4, 50)]
    exps = [ko.range_(ko.OracleStore(old), *q) for q in reqs]
    p = a.range_submit(reqs, KB_OUT_HOST)
    _call(a, m, sh.start, sh.end, inp, sh.name)
    r = p.collect()
    for q, x in enumerate(exps):
        assert r.rec_indices(q).astype(np.uint64).tolist() == x.emit.tolist() and r.kvs(q) == x.kvs(old)
    r.close()
    check_answers(a, m, REVS, what=sh.name)


def test_reconcile_ttl(engs):
    """a diff key loses its TTL, an unchanged key keeps it"""
    a, _ = engs
    sh = SHAPES["interplay ttl"]
    inp = rs.interval_items(dict(sh.engine), sh.start, sh.end)
    m = _load(a, sh)
    d = _call(a, m, sh.start, sh.end, inp, sh.name)
    dk = {k for _, k, _ in d}
    assert any(k in dk for k in sh.ttl) and any(k not in dk for k in sh.ttl)
    assert a.expire(ws.T0 + 10) == m.expire(ws.T0 + 10)[0] == len([k for k in sh.ttl if k not in dk])
    check_answers(a, m, REVS, what=sh.name)


# ---- refusals -------------------------------------------------------------------------------------------------------
def test_refused_calls_change_nothing(engs):
    a, _ = engs
    sh = SHAPES["edges"]
    m = _load(a, sh)
    for name, code, s, e, items in rs.rejections():
        with pytest.raises(KbError) as ei:
            a.reconcile(s, e, items)
        assert ei.value.code == getattr(_lib, code), name
        assert a.store_info() == m.info(), name
    # NULL arrays with n > 0
    h = C.c_void_p()
    assert _lib.lib().kb_reconcile(a._ctx, b"", 0, b"\xff", 1, None, None, None, None, 1, 0, C.byref(h)) == _lib.KB_EINVAL
    # start >= end with no records: an empty diff
    r = a.reconcile(b"\xff", b"", [])
    assert (r.n_diff, r.n_mirror) == (0, 0)
    check_answers(a, m, REVS, what="after the refusals")
    with _Fresh() as fresh:
        with pytest.raises(KbError) as ei:
            fresh.reconcile(b"", b"\xff", [])
        assert ei.value.code == _lib.KB_ESTATE


class _Fresh:
    def __enter__(self):
        self.e = Engine(0)
        return self.e

    def __exit__(self, *exc):
        self.e.close()


# ---- the storage adaptor's call sequences ---------------------------------------------------------------------------
def test_reconcile_replay_cpp(tmp_path):
    """tests/cpp/reconcile_replay_test.cpp, compiled here against the in-tree library and the oracle"""
    import os
    import shutil
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    gxx = shutil.which("g++")
    assert gxx, "the replay driver needs a C++ compiler"
    libdir, oradir = os.path.join(root, "kubebrain_b200"), os.path.join(root, "oracle")
    ko.build()
    exe = str(tmp_path / "reconcile_replay_test")
    subprocess.check_call([gxx, "-O1", "-std=c++17", "-Wall", "-o", exe,
                           os.path.join(root, "tests", "cpp", "reconcile_replay_test.cpp"),
                           "-L" + libdir, "-lkbb200", "-L" + oradir, "-lkboracle",
                           "-Wl,-rpath," + libdir, "-Wl,-rpath," + oradir])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "reconcile replay OK" in r.stdout, r.stdout + r.stderr
