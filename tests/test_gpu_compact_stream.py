"""kb_compact_stream_open / _next / _close against the C oracle: the pages of a stream concatenate to the oracle's ordered
delete-call list (record, class, the record's internal key, the guard of classes 3 / 4), each page is the greedy cut of
whole groups within the byte budget, pages can be applied as they arrive while other writes land, the layout compaction
waits for the last stream to close, and the heap-rewriting entry points invalidate open streams."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from kubebrain_b200 import _lib, synth
from kubebrain_b200._lib import KB_ECOMPACTED, KB_ESTATE, KB_OUT_HOST, Engine, KbError
from kubebrain_b200.coder import NormalCoder
from kubebrain_b200.packed import PackedStore
from oracle import binding as ko
from tests import fuzz
from tests import range_shapes as rs
from tests.test_gpu_range_stream import greedy_cuts

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL = 2**64 - 1
CODER = NormalCoder()
GUARDED = (3, 4)  # KB_V_REVRECORD, KB_V_TTL_REVREC: DelCurrent


def _pad16(n: int) -> int:
    return (n + 15) & ~15


# ---- ABI (no device) -------------------------------------------------------------------------------------------------
def test_page_view_struct_matches_the_header():
    gcc = shutil.which("gcc")
    if not gcc:
        pytest.skip("no gcc")
    src = '#include <stdio.h>\n#include "kb_b200.h"\nint main(void){printf("%zu\\n",sizeof(kb_compact_page_view));return 0;}\n'
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "s.c"), os.path.join(d, "s")
        with open(c, "w") as f:
            f.write(src)
        subprocess.check_call([gcc, "-std=c99", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        assert int(subprocess.check_output([exe])) == C.sizeof(_lib.KbCompactPageView)


# ---- helpers ---------------------------------------------------------------------------------------------------------
class Expected:
    """the oracle's delete-call list of one sweep and each victim's arena entry"""

    def __init__(self, store: PackedStore, s: bytes, e: bytes, rev: int, timeout_rev: int = 0, support_ttl: bool = True):
        x = ko.worker_run(ko.OracleStore(store), s, e, rev, compact=True, timeout_rev=timeout_rev,
                          support_ttl=support_ttl, collect=True)
        assert x.rc == 0
        self.rec = x.victims.astype(np.int64)
        self.cls = x.vclass.astype(np.uint8)
        self.count, self.examined = x.count, x.examined
        self.keys = [store.keys[int(i)] for i in self.rec]
        self.guards = [store.vals[int(i)] if c in GUARDED else b"" for i, c in zip(self.rec, self.cls)]
        self.sizes = np.array([_pad16(len(k)) + _pad16(len(g)) for k, g in zip(self.keys, self.guards)], np.int64)

    def entry(self, i: int) -> bytes:
        k, g = self.keys[i], self.guards[i]
        return k + b"\0" * (_pad16(len(k)) - len(k)) + g + b"\0" * (_pad16(len(g)) - len(g))


def drain(stream, budget: int, limit_pages: int = 1 << 30):
    pages = []
    while len(pages) < limit_pages:
        p = stream.next(budget)
        if p is None:
            break
        pages.append(p)
    return pages


def check_pages(x: Expected, pages, group: int, budget: int, what=""):
    cuts = greedy_cuts(x.sizes, group, budget)
    assert [(p.first, p.first + p.n) for p in pages] == cuts, (what, "cuts")
    for (a, b), p in zip(cuts, pages):
        assert p.rec_idx.astype(np.int64).tolist() == x.rec[a:b].tolist(), (what, a, "records")
        assert p.victim_class.tolist() == x.cls[a:b].tolist(), (what, a, "classes")
        assert p.keys() == x.keys[a:b], (what, a, "keys")
        assert p.guards() == x.guards[a:b], (what, a, "guards")
        assert p.n_bytes == int(x.sizes[a:b].sum()), (what, a, "bytes")
        assert p.arena.tobytes() == b"".join(x.entry(i) for i in range(a, b)), (what, a, "arena")


def check_stream(eng, store, s, e, rev, group, budget, timeout_rev=0, support_ttl=True, what=""):
    x = Expected(store, s, e, rev, timeout_rev, support_ttl)
    stream = eng.compact_stream(s, e, rev, timeout_rev, support_ttl, group)
    assert (stream.n_victims, stream.count, stream.examined) == (len(x.rec), x.count, x.examined), what
    pages = drain(stream, budget)
    assert stream.next(budget) is None  # stays exhausted
    stream.close()
    check_pages(x, pages, group, budget, what)
    # kb_compact_sweep's answer is the same list
    got = eng.compact_sweep(s, e, rev, timeout_rev, support_ttl, KB_OUT_HOST)
    assert got.victim_idx.astype(np.int64).tolist() == x.rec.tolist() and got.victim_class.tolist() == x.cls.tolist()
    assert (got.count, got.examined) == (x.count, x.examined)
    got.close()
    eng.set_compact_revision(None)
    return x


def budgets(sizes: np.ndarray, group: int):
    g0 = int(sizes[:group].sum()) if len(sizes) else 16
    cut = int(sizes[: 3 * group].sum()) if len(sizes) >= 3 * group else g0
    return [16, g0, cut - 16, cut, cut + 16, 4096, 64 << 20, ALL]


def _g7_store():
    from tests.test_oracle_golden import PREFIX, _g7_backend

    b = _g7_backend()
    lo, hi = ko.compact_borders(PREFIX)
    return b.snapshot(), lo, hi, b.rev - 1


def _config4(n_objects=3000, seed_ns=50):
    store, meta = synth.gen_store(n_objects, 9, 64, 64, seed_ns, config_id=4, tomb_frac=0.05)
    lo, hi = CODER.encode_object_key(b"/registry/", 0), CODER.encode_object_key(b"/registry0", 0)
    mid = meta.first_rev + (meta.last_rev - meta.first_rev) // 2
    return store, meta, lo, hi, mid


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


# ---- 1: concatenation and cuts on every store, budget and group --------------------------------------------------------
def _cases():
    r1 = rs.r1_store()
    g7, glo, ghi, grev = _g7_store()
    c4, meta, lo, hi, mid = _config4()
    return [
        ("fuzz0", fuzz.fuzz_store(400, n_keys=400), [(b"\x00", b"\xff" * 4, 30, 0, True), (b"\x00", b"\xff" * 4, ALL, 0, True)]),
        ("fuzz1", fuzz.fuzz_store(401, n_keys=900), [(b"\x00", b"\xff" * 4, 45, 20, False)]),
        ("g7", g7, [(glo, ghi, grev, 0, True)]),
        ("r1", r1.store, [(rs.MAGIC, r1.end, rs.READ, 0, True), (rs.MAGIC, r1.end, rs.READ, rs.TTL, False)]),
        ("c4", c4, [(lo, hi, meta.last_rev, 0, True), (lo, hi, meta.last_rev, mid, False)]),
    ]


@pytest.fixture(scope="module")
def cases():
    return _cases()


@pytest.mark.gpu
@pytest.mark.parametrize("group", [1, 7, 1024])
def test_pages_concatenate_to_the_victims(eng, cases, group):
    for name, store, sweeps in cases:
        eng.load_sorted(store)
        for s, e, rev, trev, ttl in sweeps:
            x = Expected(store, s, e, rev, trev, ttl)
            assert len(x.rec) > 0, name
            if trev:
                assert set(x.cls.tolist()) & {4, 5}, (name, "ttl classes")
            for budget in budgets(x.sizes, group):
                if len(greedy_cuts(x.sizes, group, budget)) > 3000:
                    continue  # a page per victim or two on the large stores: the small stores cover these budgets
                check_stream(eng, store, s, e, rev, group, budget, trev, ttl, (name, rev, trev, budget))


@pytest.mark.gpu
def test_config4_ttl_sweeps(eng):
    store, meta, lo, hi, mid = _config4(6000)
    eng.load_sorted(store)
    for trev, ttl in ((0, True), (mid, False), (mid, True)):
        x = check_stream(eng, store, lo, hi, meta.last_rev, 1024, 1 << 20, trev, ttl, (trev, ttl))
        assert 3 in x.cls.tolist()
        if not ttl:
            assert 5 in x.cls.tolist()


# ---- 2: apply as you go ------------------------------------------------------------------------------------------------
def _dump_bytes(e: Engine, path: str) -> bytes:
    e.dump(path)
    with open(path, "rb") as f:
        return f.read()


@pytest.mark.gpu
def test_apply_pages_as_they_arrive(eng, tmp_path):
    store, meta, lo, hi, _ = _config4(4000)
    eng.load_sorted(store)
    model = {store.keys[i]: store.vals[i] for i in range(store.n)}  # the engine
    R = meta.last_rev - 5
    x = Expected(store, lo, hi, R)
    group, budget = 64, 48 << 10
    cuts = greedy_cuts(x.sizes, group, budget)
    assert len(cuts) > 4
    # a class-3 victim that a later page hands out: its revision record is rewritten after the first page
    late3 = next(i for i in range(cuts[2][0], len(x.rec)) if x.cls[i] == 3)
    rewritten = x.keys[late3]
    stream = eng.compact_stream(lo, hi, R, 0, True, group)
    deleted = skipped = 0
    for n_page in range(len(cuts)):
        p = stream.next(budget)
        assert p is not None and (p.first, p.first + p.n) == cuts[n_page]
        assert p.rec_idx.astype(np.int64).tolist() == x.rec[p.first : p.first + p.n].tolist()
        ops = []
        for k in range(p.n):
            key = p.key(k)
            if p.victim_class[k] in GUARDED and model.get(key) != p.guard(k):
                skipped += 1  # DelCurrent: the CAS fails, the victim is skipped
                continue
            model.pop(key, None)
            ops.append((key, None))
        eng.apply_batch(ops)
        deleted += len(ops)
        if n_page == 0:
            # the backend keeps writing above the compact revision, and rewrites a revision record not handed out yet
            puts = []
            for j in range(0, 4000, 37):
                uk = b"/registry/pods/new-%05d" % j
                puts.append((CODER.encode_object_key(uk, meta.last_rev + 1 + j), b"v" * (50 + j % 200)))
                puts.append((CODER.encode_object_key(uk, 0), (meta.last_rev + 1 + j).to_bytes(8, "big")))
            new_guard = (meta.last_rev + 7).to_bytes(8, "big") + b"\x00"
            puts.append((rewritten, new_guard))
            for k, v in puts:
                model[k] = v
            eng.apply_batch(puts)
    assert stream.next(budget) is None
    stream.close()
    assert skipped == 1 and model[rewritten] == new_guard
    assert deleted == len(x.rec) - 1
    after = PackedStore.from_items(list(model.items()))
    st = ko.OracleStore(after)
    for rev in (ALL, meta.last_rev):
        got = eng.range_batch([(lo, hi, rev, 0)])
        assert got.rec_indices(0).astype(np.uint64).tolist() == ko.range_(st, lo, hi, rev).emit.tolist()
        got.close()
    ref = Engine(0)
    try:
        ref.load_sorted(after)
        ref.set_compact_revision(R)
        assert _dump_bytes(eng, str(tmp_path / "a")) == _dump_bytes(ref, str(tmp_path / "b"))
    finally:
        ref.close()
    eng.set_compact_revision(None)


@pytest.mark.gpu
def test_backend_compact_apply(eng):
    from kubebrain_b200.backend import Backend

    store, meta, lo, hi, _ = _config4(2000)
    eng.load_sorted(store)
    model = {store.keys[i]: store.vals[i] for i in range(store.n)}
    b = Backend(eng)
    b.set_current_revision(meta.last_rev)
    x = Expected(store, lo, hi, meta.last_rev)

    def engine_del(keys):
        for k in keys:
            model.pop(k, None)

    rev, out = b.compact_apply(0, model.get, engine_del, page_bytes=64 << 10, group=128)
    assert rev == meta.last_rev and len(out) == 1
    assert out[0] == (x.count, x.examined, len(x.rec), 0)
    after = PackedStore.from_items(list(model.items()))
    got = eng.range_batch([(lo, hi, ALL, 0)])
    assert got.rec_indices(0).astype(np.uint64).tolist() == ko.range_(ko.OracleStore(after), lo, hi, ALL).emit.tolist()
    got.close()
    assert eng.store_info()[0] == after.n
    eng.set_compact_revision(None)


# ---- 3: the layout compaction waits for the stream ----------------------------------------------------------------------
def _relocations(e: Engine) -> int:
    return sum(p["launches"] for p in e.prof_read() if p["name"] == "k_relocate")


@pytest.mark.gpu
def test_layout_compaction_deferred_while_open():
    e = Engine(0)
    try:
        store, meta, lo, hi, _ = _config4(500)
        e.load_sorted(store)
        x = Expected(store, lo, hi, meta.last_rev)
        e.prof_enable(1)
        e.prof_reset()
        stream = e.compact_stream(lo, hi, meta.last_rev, 0, True, 16)
        first = stream.next(4096)
        live = [store.keys[i] for i in range(0, store.n, 3)]
        for r in range(4):  # every round replaces a third of the values: the garbage passes a quarter of the slab
            e.apply_batch([(k, bytes([65 + r]) * 3000) for k in live])
        assert _relocations(e) == 0
        rest = drain(stream, 4096)
        check_pages(x, [first] + rest, 16, 4096, "after writes")
        stream.close()
        assert _relocations(e) == 0
        e.apply_batch([(live[0], b"z" * 3000)])  # the first write after the close evaluates the trigger
        assert _relocations(e) == 1
    finally:
        e.close()


# ---- 4: invalidation, cleanup, edge cases -----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("what", ["load", "restore", "dump"])
def test_heap_rewrite_invalidates(what, tmp_path):
    e = Engine(0)
    try:
        store, meta, lo, hi, _ = _config4(500)
        e.load_sorted(store)
        path = str(tmp_path / "snap")
        e.dump(path)
        s1 = e.compact_stream(lo, hi, meta.last_rev, 0, True, 8)
        s2 = e.compact_stream(lo, hi, meta.last_rev, 0, True, 8)
        assert s1.next(1024) is not None
        {"load": lambda: e.load_sorted(store), "restore": lambda: e.restore(path), "dump": lambda: e.dump(path)}[what]()
        for s in (s1, s2):
            with pytest.raises(KbError) as ei:
                s.next(1024)
            assert ei.value.code == KB_ESTATE and "rewrote the snapshot" in str(ei.value)
            s.close()
        # a fresh stream works again
        check_stream(e, store, lo, hi, meta.last_rev, 8, 1024)
    finally:
        e.close()


@pytest.mark.gpu
def test_close_context_with_open_streams():
    e = Engine(0)
    store, meta, lo, hi, _ = _config4(300)
    e.load_sorted(store)
    s1 = e.compact_stream(lo, hi, meta.last_rev, 0, True, 1)
    s2 = e.compact_stream(lo, hi, meta.last_rev, 0, True, 1024)
    p = s1.next(0)
    assert p is not None and p.n == 1
    e.close()
    s1.close(), s2.close()  # the context already freed them


@pytest.mark.gpu
def test_edges(eng):
    store = fuzz.fuzz_store(402, n_keys=300)
    eng.load_sorted(store)
    k0 = store.keys[0]
    for s, e in ((k0, k0), (b"\x7f", b"\x00"), (b"\x02", b"\x03")):  # empty, reversed, no record
        stream = eng.compact_stream(s, e, 30)
        assert stream.n_victims == 0
        assert stream.next(ALL) is None and stream.next(0) is None
        stream.close()
    with pytest.raises(KbError):
        eng.compact_stream(b"\x00", b"\xff", 30, group_victims=0)
    # the open records the compact revision: a range below it is refused
    stream = eng.compact_stream(b"\x00", b"\xff" * 4, 40)
    with pytest.raises(KbError) as ei:
        eng.range_batch([(b"\x00", b"\xff" * 4, 39, 0)])
    assert ei.value.code == KB_ECOMPACTED
    stream.close()
    eng.set_compact_revision(None)


# ---- 5: range batches and point reads in flight around the pages --------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 2, 4])
def test_pages_between_batches_and_point_reads(lanes, monkeypatch):
    monkeypatch.setenv("KB_LANES", str(lanes))
    e = Engine(0)
    try:
        store = fuzz.fuzz_store(403, n_keys=1500)
        st = ko.OracleStore(store)
        e.load_sorted(store)
        batch = [(a, b, ALL, lim) for a, b in fuzz.fuzz_bounds(store, 3) for lim in (0, 3)]
        bexp = [ko.range_(st, *q) for q in batch]
        users = sorted({ko.decode(store.keys[i])[0] for i in range(0, store.n, 11)} - {None})[:50]
        gets = [(u, r) for u in users for r in (0, 25)]
        gexp = []
        for u, r in gets:  # (status, record, mod_rev) as backend.get answers
            idx, mod = ko.get(st, u, r)
            gexp.append((0, idx, mod) if idx >= 0 else (2, -1, mod) if idx == -2 else (1, -1, 0))
        x = Expected(store, b"\x00", b"\xff" * 4, 40)

        def check_inflight(pend):
            for kind, p in pend:
                r = p.collect()
                if kind == "range":
                    for q, ex in enumerate(bexp):
                        assert r.rec_indices(q).astype(np.uint64).tolist() == ex.emit.tolist()
                else:
                    for i, (est, eidx, emod) in enumerate(gexp):
                        assert int(r.status[i]) == est
                        if est != 1:
                            assert int(r.mod_rev[i]) == emod
                        if est == 0:
                            assert int(r.rec_idx[i]) == eidx
                r.close()

        pend = [("range", e.range_submit(batch)) for _ in range(lanes)] + [("get", e.get_submit(gets))]
        stream = e.compact_stream(b"\x00", b"\xff" * 4, 40, 0, True, 7)
        check_inflight(pend)
        pages = []
        while True:
            pend = [("range", e.range_submit(batch)) for _ in range(lanes)] + [("get", e.get_submit(gets))]
            p = stream.next(700)
            check_inflight(pend)
            if p is None:
                break
            pages.append(p)
        stream.close()
        check_pages(x, pages, 7, 700, "in flight")
        e.set_compact_revision(None)
    finally:
        e.close()


# ---- 6: config 4 at full size ---------------------------------------------------------------------------------------------
def _host_ram_gb() -> float:
    try:
        with open("/proc/meminfo") as f:
            for line in f:
                if line.startswith("MemAvailable:"):
                    return int(line.split()[1]) / (1 << 20)
    except OSError:
        pass
    return 0.0


def _ranges(starts: np.ndarray, lens: np.ndarray) -> np.ndarray:
    """the byte indices of the concatenated ranges [starts[i], starts[i] + lens[i])"""
    lens = lens.astype(np.int64)
    tot = int(lens.sum())
    if tot == 0:
        return np.zeros(0, np.int64)
    base = np.repeat(starts.astype(np.int64) - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens)
    return base + np.arange(tot, dtype=np.int64)


@pytest.mark.gpu
def test_config4_full_size_vectorised():
    if _host_ram_gb() < 48:
        pytest.skip("host has less than 48 GB of free RAM")
    store, meta = synth.gen_store(10_000_000, 9, 64, 64, 50000, config_id=4, tomb_frac=0.02)
    lo, hi = CODER.encode_object_key(b"/registry/", 0), CODER.encode_object_key(b"/registry0", 0)
    exp = ko.scan(ko.OracleStore(store), [lo, hi], meta.last_rev, compact=True, collect=False)
    e = Engine(0)
    try:
        e.load_sorted(store)
        stream = e.compact_stream(lo, hi, meta.last_rev)
        assert (stream.n_victims, stream.count, stream.examined) == (len(exp.victims), exp.count, store.n)
        koff, kd = store.keys.off.astype(np.int64), store.keys.data
        voff, vd = store.vals.off.astype(np.int64), store.vals.data
        pos = 0
        while True:
            p = stream.next(64 << 20)
            if p is None:
                break
            assert p.first == pos and (p.n % 1024 == 0 or pos + p.n == len(exp.victims))
            rec = exp.victims[pos : pos + p.n].astype(np.int64)
            cls = exp.vclass[pos : pos + p.n]
            assert np.array_equal(p.rec_idx.astype(np.int64), rec) and np.array_equal(p.victim_class, cls)
            klen = koff[rec + 1] - koff[rec]
            glen = np.where(np.isin(cls, GUARDED), voff[rec + 1] - voff[rec], 0)
            assert np.array_equal(p.key_len.astype(np.int64), klen) and np.array_equal(p.guard_len.astype(np.int64), glen)
            size = ((klen + 15) & ~15) + ((glen + 15) & ~15)
            start = np.concatenate([[0], np.cumsum(size)[:-1]])
            assert np.array_equal(p.key_off.astype(np.int64), start)
            assert np.array_equal(p.guard_off.astype(np.int64), start + ((klen + 15) & ~15))
            assert np.array_equal(p.arena[_ranges(start, klen)], kd[_ranges(koff[rec], klen)])
            assert np.array_equal(p.arena[_ranges(start + ((klen + 15) & ~15), glen)], vd[_ranges(voff[rec], glen)])
            pos += p.n
        assert pos == len(exp.victims)
        stream.close()
    finally:
        e.close()


# ---- 7: the Go shim's call sequence ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_compact_replay_cpp(tmp_path):
    """tests/cpp/compact_replay_test.cpp, compiled here against the in-tree library and the oracle"""
    gxx = shutil.which("g++")
    assert gxx, "the replay driver needs a C++ compiler"
    libdir, oradir = os.path.join(ROOT, "kubebrain_b200"), os.path.join(ROOT, "oracle")
    ko.build()
    exe = str(tmp_path / "compact_replay_test")
    subprocess.check_call([gxx, "-O1", "-std=c++17", "-Wall", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "compact_replay_test.cpp"),
                           "-L" + libdir, "-lkbb200", "-L" + oradir, "-lkboracle",
                           "-Wl,-rpath," + libdir, "-Wl,-rpath," + oradir])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "compact replay OK" in r.stdout, r.stdout + r.stderr
