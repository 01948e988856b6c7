"""Concurrent callers against the oracle (tests/concurrent_plan.py holds the plans and their expected answers).

C1: both halves of the step as bench.py runs them -- a scan context and a fan-out context on one device, each driven
from its own thread, one of them on high-priority streams -- with every range answer and every burst compared exactly.
C2: several threads on one context, interleaving the way the Go binding does: pendings submitted and collected in any
order, point reads, range and compaction streams, partitions and sweeps while a writer commits the plan's versions,
reconciles and expires, and device-resident answers freed by a thread other than the one that made them.
C3: the message kb_last_error gives each thread is the one of its own refused call."""
from __future__ import annotations

import ctypes as C
import queue
import threading
import traceback

import numpy as np
import pytest

from kubebrain_b200 import synth
from kubebrain_b200._lib import (KB_ECOMPACTED, KB_ELIMIT, KB_OUT_DEVICE, KB_OUT_HOST, KB_WIRE_ETCD_EVENTS,
                                 KB_WIRE_ETCD_KVS, Engine, KbError, KbRangeReq, KbWriteOp, lib)
from kubebrain_b200.packed import PackedStore
from oracle import binding as ko
from tests import concurrent_plan as cp
from tests import partition_shapes as ps
from tests import reconcile_shapes as rsh

pytestmark = pytest.mark.gpu

JOIN_S = 120
STEPS = 200
WIRE = KB_WIRE_ETCD_KVS | KB_WIRE_ETCD_EVENTS


# ---- threads ---------------------------------------------------------------------------------------------------------
class Crew:
    """worker threads sharing one stop event: the first exception stops them all and is raised on the main thread with
    the thread's name, its step and what differed; a thread still alive after JOIN_S is reported as a hang, naming the
    call it was in"""

    def __init__(self):
        self.stop = threading.Event()
        self.errors, self.where, self.threads = [], {}, []
        self.barriers = []  # broken on the first error, so no worker waits for one that has stopped

    def at(self, what: str):
        self.where[threading.current_thread().name] = what

    def spawn(self, name: str, fn, *args):
        def run():
            try:
                fn(self, *args)
            except BaseException as e:  # noqa: B902 -- everything a worker raises is reported
                self.errors.append("%s at %s: %r\n%s" % (name, self.where.get(name), e, traceback.format_exc()))
                self.stop.set()
                for b in self.barriers:
                    b.abort()

        self.threads.append(threading.Thread(target=run, name=name, daemon=True))

    def run(self) -> bool:
        """starts and joins every thread; False when one hangs (its engine must then stay open)"""
        for t in self.threads:
            t.start()
        for t in self.threads:
            t.join(JOIN_S)
        alive = [t.name for t in self.threads if t.is_alive()]
        if alive:
            self.stop.set()
            self.errors.append("hang: %s" % ", ".join("%s in %s" % (n, self.where.get(n)) for n in alive))
        return not alive

    def check(self):
        assert not self.errors, "\n".join(self.errors)


def expect(read_exp, got, what, want=None):
    assert cp.digest(got) == (want or cp.digest(read_exp)), "%s: %s" % (what, cp.first_difference(read_exp, got))


# ---- answers read back -----------------------------------------------------------------------------------------------
def range_got(eng: Engine, r, mode: str):
    if mode == "count":
        return {"count": cp._u64(r.req_count)}
    out = {"first": cp._u64(r.req_first), "count": cp._u64(r.req_count), "examined": cp._u64(r.req_examined)}
    wire = cp.MODES[mode] & WIRE
    if r.on_device:
        rec, rev = r.device_array("rec_idx", np.uint32), r.device_array("rev", np.uint64)
        image = eng.read_device(r.bytes_ptr, r.n_bytes, sync=False)
        eo = r.device_array("elem_off", np.uint64) if wire else None
    else:
        rec, rev, image = r.rec_idx, r.rev, r.arena[: r.n_bytes].tobytes()
        eo = r.elem_off if wire else None
    out.update(rec=cp._u64(rec), rev=cp._u64(rev), image=image)
    if wire:
        out["elem_off"] = cp._u64(eo)
    return out


def get_got(g, mode: str):
    st = g.status
    vals = [b"" if st[i] != 0 else g.element(i) if mode == "kvs" else g.value(i) for i in range(g.n)]
    return {"status": st.tobytes(), "mod_rev": cp._u64(g.mod_rev), "rec": cp._u64(np.where(st == 0, g.rec_idx, 0)),
            "vals": b"".join(cp.struct.pack("<I", len(v)) + v for v in vals)}


def stream_got(crew: Crew, s, mode: str):
    rec, image, pages = [], [], []
    while True:
        crew.at("kb_range_stream_next page %d" % len(pages))
        p = s.next(cp.PAGE_BUDGET)
        if p is None:
            break
        rec.append(p.rec_idx.copy())
        image.append(p.arena[: p.n_bytes].tobytes())
        pages.append(p.n_kvs)
        p.close()
    s.close()
    return {"rec": cp._u64(np.concatenate(rec) if rec else []), "image": b"".join(image), "pages": cp._u64(pages)}


# ---- C1: both halves of the step -------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def c1():
    store, meta = synth.gen_store(30000, 4, 64, 2048, 100, config_id=2, tomb_frac=0.1)
    st = ko.OracleStore(store)
    pods = cp.MAGIC + b"/registry/pods/"
    ns = [cp.MAGIC + b"/registry/%s/ns-%05d/" % (r, i) for r, i in ((b"pods", 3), (b"configmaps", 7), (b"pods", 41))]
    specs = []
    for i, mode in enumerate(("device", "host", "kvs", "device", "events", "host", "device", "dev_kvs")):
        reqs = [(ns[i % 3], ns[i % 3][:-1] + b"0", meta.read_rev, 0), (pods, pods + b"\xff", meta.last_rev, 300 + i),
                (cp.MAGIC, cp.MAGIC + b"\xff", meta.first_rev + 5000 * i, 1 + 37 * i)]
        exp = cp.range_parts(store, st, reqs, mode)
        specs.append((Engine.pack_range_reqs(reqs), mode, (exp, cp.digest(exp))))
    return store, specs, cp.gen_bursts()


def scan_worker(crew: Crew, eng: Engine, specs):
    pend, held = [], []
    for step in range(STEPS):
        if crew.stop.is_set():
            return
        for j in (2 * step, 2 * step + 1):
            reqs, mode, exp = specs[j % len(specs)]
            crew.at("step %d: kb_range_submit of batch %d (%s)" % (step, j, mode))
            pend.append((j, mode, exp, eng.range_submit(reqs, cp.MODES[mode])))
            if len(pend) > 2:  # two batches in flight, as bench does
                j0, m0, e0, p = pend.pop(0)
                crew.at("step %d: kb_range_collect of batch %d (%s)" % (step, j0, m0))
                r = p.collect()
                if r.on_device and j0 % 3 == 0:
                    held.append((j0, m0, e0, r))  # read back and freed some steps later
                else:
                    expect(e0[0], range_got(eng, r, m0), "batch %d (%s)" % (j0, m0), e0[1])
                    r.close()
        if step % 4 == 1:
            crew.at("step %d: kb_range_prefetch" % step)
            eng.range_prefetch(specs[(2 * step + 2) % len(specs)][0])
        while len(held) > 3:
            j0, m0, e0, r = held.pop(0)
            crew.at("step %d: reading held batch %d" % (step, j0))
            expect(e0[0], range_got(eng, r, m0), "held batch %d (%s)" % (j0, m0), e0[1])
            r.close()
    for j0, m0, e0, p in pend:
        crew.at("draining batch %d" % j0)
        r = p.collect()
        expect(e0[0], range_got(eng, r, m0), "batch %d (%s)" % (j0, m0), e0[1])
        r.close()
    for j0, m0, e0, r in held:
        expect(e0[0], range_got(eng, r, m0), "held batch %d (%s)" % (j0, m0), e0[1])
        r.close()


def fanout_worker(crew: Crew, weng: Engine, bursts, handles):
    for step in range(STEPS):
        if crew.stop.is_set():
            return
        k = step % len(bursts.events)
        start, idx = bursts.expected[k]
        if step % 3 == 2:
            crew.at("burst %d: kb_watch_match (host) of burst %d" % (step, k))
            m = weng.watch_match(bursts.events[k], KB_OUT_HOST)
            got = m.event_idx
        else:
            crew.at("burst %d: kb_watch_match_dev of burst %d" % (step, k))
            m = weng.watch_match_dev(handles[k], KB_OUT_DEVICE)
            got = m.device_event_idx()
        assert np.array_equal(m.start, start), "burst %d (%d): delivery offsets" % (step, k)
        assert m.n_deliveries == len(idx) and np.array_equal(got, idx), \
            "burst %d (%d): delivery lists differ at %s" % (step, k, np.flatnonzero(got[: len(idx)] != idx[: len(got)])[:1])
        m.close()


@pytest.mark.parametrize("lanes", ["default", "1"])
@pytest.mark.parametrize("host_values", [False, True], ids=["hbm", "host_values"])
@pytest.mark.parametrize("prio", ["fanout", "scan"])
def test_c1_scan_and_fanout_contexts(monkeypatch, c1, prio, host_values, lanes):
    if lanes != "default":
        monkeypatch.setenv("KB_LANES", lanes)  # kb_open reads it every time
    else:
        monkeypatch.delenv("KB_LANES", raising=False)
    store, specs, bursts = c1
    eng = weng = None
    handles = []
    closeable = True
    try:
        eng = Engine(0, high_priority=prio == "scan", host_values=host_values)
        eng.load_sorted(store)
        weng = Engine(0, high_priority=prio == "fanout")
        weng.watch_add_many(bursts.watchers)
        handles = [weng.events_upload(ev) for ev in bursts.events]
        crew = Crew()
        crew.spawn("scan", scan_worker, eng, specs)
        crew.spawn("fanout", fanout_worker, weng, bursts, handles)
        closeable = crew.run()
        crew.check()
    finally:
        if closeable:
            for h in handles:
                weng.events_free(h)
            for e in (eng, weng):
                if e is not None:
                    e.close()


# ---- C2: threads sharing one context ---------------------------------------------------------------------------------
class Shared:
    def __init__(self, plan: cp.Plan, eng: Engine):
        self.plan, self.eng = plan, eng
        self.version = 0                     # the last version whose apply_batch has returned
        self.readers_done = threading.Barrier(5, timeout=JOIN_S)
        self.held = queue.SimpleQueue()      # device answers for the freeing thread
        self.window = {}                     # thread -> the lowest version its window reads may still answer

    def window_check(self, read: cp.Read, got, a: int, b: int, what: str):
        """the answer equals the one of a version in [a, b + 1], and never one older than this thread's last"""
        name = threading.current_thread().name
        lo = max(a, self.window.get(name, 0))
        hi = min(b + 1, len(self.plan.items) - 1)
        d = cp.digest(got)
        match = [v for v in range(lo, hi + 1) if read.answers[v] == d]
        assert match, "%s: answers no version in [%d, %d] (against v0: %s)" % (
            what, lo, hi, cp.first_difference(read.exp, got))
        self.window[name] = match[0]

    def window_in_submit_order(self, window, what: str):
        """a pipelined read answers the version current at its submission, so a thread's window reads go forward in
        the order it submitted them, not in the order it collected them"""
        for i in sorted(window):
            r, got, a, b = window[i]
            self.window_check(r, got, a, b, "%s (%s, submitted %d)" % (what, r.args.get("mode", "-"), i))

    def info_check(self, got, a: int, b: int):
        name = threading.current_thread().name
        lo, hi = max(a, self.window.get(name, 0)), min(b + 1, len(self.plan.items) - 1)
        match = [v for v in range(lo, hi + 1) if cp.info_ok(self.plan, v, got)]
        assert match, "kb_store_info %s is no version's in [%d, %d]" % (got, lo, hi)
        self.window[name] = match[0]


def ranges_worker(crew: Crew, sh: Shared, rounds: int):
    reads = [r for r in sh.plan.reads if r.kind in ("range", "count")]
    for n in range(rounds):
        if crew.stop.is_set():
            break
        pend = []
        for i, r in enumerate(reads[n % 3::3] or reads[:1]):
            a = sh.version
            crew.at("round %d: kb_range_submit (%s)" % (n, r.args["mode"]))
            p = sh.eng.range_submit(r.args["reqs"], cp.MODES[r.args["mode"]])
            pend.append((r, p, a, sh.version))
        window = {}
        for i in range(len(pend) - 1, -1, -1):  # collected in the other order
            r, p, a, b = pend[i]
            crew.at("round %d: kb_range_collect (%s)" % (n, r.args["mode"]))
            res = p.collect()
            if r.invariant and res.on_device and n % 2 == 0:
                sh.held.put((r, res))
                continue
            got = range_got(sh.eng, res, r.args["mode"])
            res.close()
            if r.invariant:
                expect(r.exp, got, "range read (%s)" % r.args["mode"])
            else:
                window[i] = (r, got, a, b)
        sh.window_in_submit_order(window, "count read")
    sh.held.put(None)
    sh.readers_done.wait()


def gets_worker(crew: Crew, sh: Shared, rounds: int):
    reads = [r for r in sh.plan.reads if r.kind == "get"]
    for n in range(rounds):
        if crew.stop.is_set():
            break
        pend = []
        for r in reads:
            a = sh.version
            crew.at("round %d: kb_get_submit (%s)" % (n, r.args["mode"]))
            pend.append((r, sh.eng.get_submit(r.args["reqs"], cp.GET_MODES[r.args["mode"]]), a, sh.version))
        window = {}
        for i in list(range(1, len(pend), 2)) + list(range(0, len(pend), 2)):  # not in submission order
            r, p, a, b = pend[i]
            crew.at("round %d: kb_get_collect (%s)" % (n, r.args["mode"]))
            g = p.collect()
            got = get_got(g, r.args["mode"])
            g.close()
            if r.invariant:
                expect(r.exp, got, "point reads (%s)" % r.args["mode"])
            else:
                window[i] = (r, got, a, b)
        sh.window_in_submit_order(window, "latest point reads")
        a = sh.version
        crew.at("round %d: kb_store_info" % n)
        got = sh.eng.store_info()
        sh.info_check(got, a, sh.version)
    sh.readers_done.wait()


def streams_worker(crew: Crew, sh: Shared, rounds: int):
    streams = [r for r in sh.plan.reads if r.kind == "stream"]
    cs = next(r for r in sh.plan.reads if r.kind == "cstream")
    for n in range(rounds):
        if crew.stop.is_set():
            break
        r = streams[n % len(streams)]
        crew.at("round %d: kb_range_stream_open (%s)" % (n, r.args["mode"]))
        s = sh.eng.range_stream(r.args["req"], cp.MODES[r.args["mode"]], cp.GROUP)
        expect(r.exp, stream_got(crew, s, r.args["mode"]), "range stream (%s)" % r.args["mode"])
        a = cs.args
        crew.at("round %d: kb_compact_stream_open" % n)
        c = sh.eng.compact_stream(a["start"], a["end"], a["rev"], 0, True, cp.GROUP)
        rec, cls, keys, guards = [], [], [], []
        while True:
            crew.at("round %d: kb_compact_stream_next page" % n)
            p = c.next(4096)
            if p is None:
                break
            rec.append(p.rec_idx)
            cls.append(p.victim_class)
            keys += p.keys()
            guards += p.guards()
        c.close()
        got = {"rec": cp._u64(np.concatenate(rec) if rec else []),
               "cls": np.concatenate(cls).tobytes() if cls else b"", "count": cp._u64([c.count]),
               "examined": cp._u64([c.examined]), "keys": b"".join(cp.struct.pack("<I", len(k)) + k for k in keys),
               "guards": b"".join(cp.struct.pack("<I", len(g)) + g for g in guards)}
        expect(cs.exp, got, "compaction stream")
    sh.readers_done.wait()


def partitions_worker(crew: Crew, sh: Shared, rounds: int):
    pr = next(r for r in sh.plan.reads if r.kind == "partitions")
    sw = next(r for r in sh.plan.reads if r.kind == "sweep")
    a = pr.args
    for n in range(rounds):
        if crew.stop.is_set():
            break
        crew.at("round %d: kb_range_partitions" % n)
        borders, kv_first, arena_first = sh.eng.range_partitions(a["start"], a["end"], a["rev"], a["part_bytes"],
                                                                 a["max_parts"])
        if n == 0:
            v0 = sh.plan.stores[0]
            ps.check_partitions(v0, ko.OracleStore(v0), a["start"], a["end"], a["rev"], (borders, kv_first, arena_first))
        got = {"borders": b"".join(cp.struct.pack("<I", len(b)) + b for b in borders), "kv_first": cp._u64(kv_first),
               "arena_first": cp._u64(arena_first)}
        expect(pr.exp, got, "partitions")
        crew.at("round %d: kb_compact_sweep" % n)
        c = sh.eng.compact_sweep(sw.args["start"], sw.args["end"], sw.args["rev"], 0, True, KB_OUT_HOST)
        got = {"rec": cp._u64(c.victim_idx), "cls": c.victim_class.tobytes(), "count": cp._u64([c.count]),
               "examined": cp._u64([c.examined])}
        c.close()
        exp = {k: sw.exp[k] for k in ("rec", "cls", "count", "examined")}
        expect(exp, got, "compaction sweep")
    sh.readers_done.wait()


def free_worker(crew: Crew, sh: Shared):
    """reads back and frees the device answers the range thread collected"""
    n = 0
    while not crew.stop.is_set():
        try:
            x = sh.held.get(timeout=0.05)
        except queue.Empty:
            continue
        if x is None:  # the range thread is done
            return
        r, res = x
        crew.at("freeing held answer %d" % n)
        expect(r.exp, range_got(sh.eng, res, r.args["mode"]), "held range read (%s)" % r.args["mode"])
        res.close()
        n += 1


def writer_worker(crew: Crew, sh: Shared):
    plan, eng = sh.plan, sh.eng
    s, e = plan.reconcile
    for v, batch in enumerate(plan.batches, start=1):
        if crew.stop.is_set():
            return
        crew.at("kb_apply_batch of v%d" % v)
        eng.apply_batch(batch)
        sh.version = v
        crew.at("kb_reconcile dry run at v%d" % v)
        d = eng.reconcile(s, e, rsh.interval_items(plan.items[v], s, e), dry_run=True)
        assert d.n_diff == 0, "dry run at v%d: %d diffs" % (v, d.n_diff)
    crew.at("waiting for the readers")
    sh.readers_done.wait()
    # every reader has stopped: the expiry and the repair make states outside the plan's versions
    latest = plan.items[-1]
    ttl = {op[0] for b in plan.batches for op in b if len(op) > 2 and op[2]}
    crew.at("kb_expire")
    assert eng.expire(cp.EXPIRE_NOW) == len(ttl & set(latest)), "kb_expire"
    after = {k: v for k, v in latest.items() if k not in ttl}
    assert eng.store_info()[0] == len(after), "records after kb_expire"
    gone = sorted(k for k in after if s <= k < e)[:3]
    crew.at("diverging the reconcile interval")
    eng.apply_batch([(k, None) for k in gone])
    inp = rsh.interval_items(after, s, e)
    mirror = {k: v for k, v in after.items() if k not in gone}
    crew.at("kb_reconcile")
    d = eng.reconcile(s, e, inp)
    exp = rsh.diff(mirror, inp, s, e)
    assert (d.kinds.tolist(), d.keys(), d.src_idx.tolist()) == ([x[0] for x in exp], [x[1] for x in exp],
                                                               [x[2] for x in exp]), "reconcile diff"
    assert d.n_missing == len(gone) and eng.reconcile(s, e, inp, dry_run=True).n_diff == 0, "repaired"


@pytest.fixture(scope="module")
def plan():
    return cp.gen_plan(0)


def test_c2_threads_on_one_context(plan):
    eng = Engine(0)
    closeable = True
    try:
        eng.load_sorted(plan.stores[0])
        sh = Shared(plan, eng)
        crew = Crew()
        crew.barriers.append(sh.readers_done)
        crew.spawn("ranges", ranges_worker, sh, 60)
        crew.spawn("gets", gets_worker, sh, 60)
        crew.spawn("streams", streams_worker, sh, 12)
        crew.spawn("partitions", partitions_worker, sh, 20)
        crew.spawn("writer", writer_worker, sh)
        crew.spawn("free", free_worker, sh)
        closeable = crew.run()
        crew.check()
    finally:
        if closeable:
            eng.close()


# ---- C3: error attribution -------------------------------------------------------------------------------------------
def _c3_engine() -> Engine:
    eng = Engine(0)
    eng.load_sorted(PackedStore.from_items([(cp.ik(b"/a", 0), cp.struct.pack(">Q", 5)), (cp.ik(b"/a", 5), b"x")]))
    eng.set_compact_revision(100)
    return eng


def test_c3_each_thread_reads_its_own_message():
    eng = _c3_engine()
    L = lib()
    long_key = b"k" * 65536
    req = (KbRangeReq * 1)(KbRangeReq(cp.MAGIC, 4, cp.MAGIC + b"\xff", 5, 50, 0))
    op = (KbWriteOp * 1)()
    op[0].type, op[0].key, op[0].key_len, op[0].val, op[0].val_len = 0, long_key, len(long_key), b"v", 1
    b1, b2 = threading.Barrier(2, timeout=JOIN_S), threading.Barrier(2, timeout=JOIN_S)
    got = {}

    def a():
        h = C.c_void_p()
        got["a_rc"] = L.kb_range_batch(eng._ctx, req, 1, KB_OUT_HOST, C.byref(h))
        b1.wait()  # B refuses its call now
        b2.wait()
        got["a"] = L.kb_last_error(eng._ctx).decode()

    def b():
        b1.wait()
        got["b_rc"] = L.kb_apply_batch(eng._ctx, op, 1)
        b2.wait()
        got["b"] = L.kb_last_error(eng._ctx).decode()

    try:
        ts = [threading.Thread(target=f, daemon=True) for f in (a, b)]
        for t in ts:
            t.start()
        for t in ts:
            t.join(JOIN_S)
        assert not any(t.is_alive() for t in ts), "hang"
        assert got["a_rc"] == KB_ECOMPACTED and got["b_rc"] == KB_ELIMIT
        assert "less than compact revision" in got["a"], got["a"]
        assert "longer than 65535 bytes" in got["b"], got["b"]
        # a thread that made no refused call reads the context's last message
        other = {}
        t = threading.Thread(target=lambda: other.update(m=L.kb_last_error(eng._ctx).decode()), daemon=True)
        t.start()
        t.join(JOIN_S)
        assert "longer than 65535 bytes" in other["m"], other
    finally:
        eng.close()


def test_c3_refusals_on_two_threads_through_engine():
    eng = _c3_engine()
    crew = Crew()

    def ranges(crew: Crew):
        for i in range(2000):
            crew.at("refused range %d" % i)
            with pytest.raises(KbError) as ei:
                eng.range_batch([(cp.MAGIC, cp.MAGIC + b"\xff", 50, 0)])
            assert ei.value.code == KB_ECOMPACTED and "less than compact revision" in str(ei.value), str(ei.value)

    def writes(crew: Crew):
        for i in range(2000):
            crew.at("refused write %d" % i)
            with pytest.raises(KbError) as ei:
                eng.apply_batch([(b"k" * 65536, b"v")])
            assert ei.value.code == KB_ELIMIT and "longer than 65535 bytes" in str(ei.value), str(ei.value)

    crew.spawn("ranges", ranges)
    crew.spawn("writes", writes)
    closeable = crew.run()
    try:
        crew.check()
    finally:
        if closeable:
            eng.close()
