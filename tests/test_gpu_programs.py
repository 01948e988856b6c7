"""Seeded programs of interleaved entry points on one context (tests/program_model.py) against the model's transcript.

Every op of a program runs on one Engine opened with KB_LANES lanes, and its answer is compared with the model's entry
at that op: emitted records, per-request counts and examined, kv bytes, arena bytes and wire element offsets, page
cuts, partition borders and offsets, victim keys and guards, match lists, error codes, kb_store_info and dump images.
Device-resident answers are held across the later ops that follow them and read back where the program says.  A
mismatch names the seed, the lane count, the op and the 20 ops in front of it; `python -m tests.program_model --seed S
--lanes L` prints the whole program and its expected transcript."""
from __future__ import annotations

import numpy as np
import pytest

from kubebrain_b200._lib import Engine, KbError
from kubebrain_b200.packed import PackedStore
from tests import fuzz
from tests import program_model as pm

pytestmark = pytest.mark.gpu


def _dig(b: bytes) -> str:
    return pm._digest(bytes(b))


class Runner:
    """executes a program's ops on one engine and turns every answer into a transcript entry"""

    def __init__(self, eng: Engine, path: str):
        self.eng, self.path = eng, path
        self.h = {}  # handle name -> pending, stream, result or watcher id

    # -- answers
    def range_entry(self, r, mode: int):
        if pm.base_of(mode) == pm.KB_OUT_COUNT:
            return {"count": r.req_count.tolist()}
        host = {"first": r.req_first.tolist(), "count": r.req_count.tolist(), "examined": r.req_examined.tolist(),
                "n_kvs": r.n_kvs, "n_bytes": r.n_bytes}
        if r.on_device:
            return host
        eo = r.elem_off.tolist() if pm.wire_of(mode) and r.n_kvs else None
        kvs = [kv for q in range(r.n_req) for kv in r.kvs(q)]
        return {**host, "rec": r.rec_idx.astype(np.int64).tolist(), "kvs": kvs, "arena": _dig(r.arena[: r.n_bytes]),
                "elem_off": eo}

    def device_body(self, r, mode: int):
        arr = {n: r.device_array(n, dt) for n, dt in (("rec_idx", np.uint32), ("rev", np.uint64), ("key_off", np.uint64),
                                                      ("key_len", np.uint32), ("val_off", np.uint64), ("val_len", np.uint32))}
        arena = self.eng.read_device(r.bytes_ptr, r.n_bytes, sync=False)
        kvs = []
        for k in range(r.n_kvs):
            ko_, kl, vo, vl = (int(arr[n][k]) for n in ("key_off", "key_len", "val_off", "val_len"))
            kvs.append((arena[ko_: ko_ + kl], arena[vo: vo + vl], int(arr["rev"][k])))
        eo = r.device_array("elem_off", np.uint64).tolist() if pm.wire_of(mode) and r.n_kvs else None
        return {"rec": arr["rec_idx"].astype(np.int64).tolist(), "kvs": kvs, "arena": _dig(arena), "elem_off": eo}

    def get_entry(self, g, mode: int):
        n = g.n
        st = g.status.tolist()
        out = {"status": st, "mod_rev": g.mod_rev.tolist(), "rec": [int(g.rec_idx[i]) if st[i] == 0 else None for i in range(n)]}
        if pm.wire_of(mode):
            out["elems"] = [g.element(i) for i in range(n)]
        else:
            arena = g.arena[: g.n_bytes].tobytes() if not g.on_device else self.eng.read_device(g.bytes_ptr, g.n_bytes)
            out["arena"] = _dig(arena)
            out["values"] = [arena[int(g.val_off[i]): int(g.val_off[i]) + int(g.val_len[i])] if st[i] == 0 else None
                             for i in range(n)]
        g.close()
        return out

    def page_entry(self, page, mode: int):
        if page is None:
            return None
        if page.on_device:
            rec = page.device_array("rec_idx", np.uint32)
            arena = self.eng.read_device(page.bytes_ptr, page.n_bytes, sync=False)
            eo = page.device_array("elem_off", np.uint64).tolist() if pm.wire_of(mode) else None
        else:
            rec, arena = page.rec_idx, page.arena[: page.n_bytes].tobytes()
            eo = page.elem_off.tolist() if pm.wire_of(mode) else None
        out = {"first": page.req_first.tolist(), "count": page.req_count.tolist(), "examined": page.req_examined.tolist(),
               "rec": rec.astype(np.int64).tolist(), "arena": _dig(arena), "n_bytes": page.n_bytes, "elem_off": eo}
        page.close()
        return out

    def match_entry(self, m, name: str):
        out = {"n_watchers": m.n_watchers, "start": m.start.tolist()}
        if m.on_device:
            self.h[name] = ("match", m)
        else:
            out["idx"] = m.event_idx.tolist()
            m.close()
        return out

    # -- ops
    def step(self, kind: str, a: dict):
        try:
            return getattr(self, "op_" + kind)(a)
        except KbError as e:
            return pm.err(e.code)

    def op_range_batch(self, a):
        mode = pm.MODES[a["mode"]]
        r = self.eng.range_batch(a["reqs"], mode)
        out = self.range_entry(r, mode)
        if r.on_device:
            self.h[a["h"]] = ("range", r, mode)
        else:
            r.close()
        return out

    def op_range_submit(self, a):
        self.h[a["h"]] = ("pending", self.eng.range_submit(a["reqs"], pm.MODES[a["mode"]]), pm.MODES[a["mode"]])
        return pm.OK

    def op_get_submit(self, a):
        self.h[a["h"]] = ("pending_get", self.eng.get_submit(a["reqs"], pm.GET_MODES[a["mode"]]), pm.GET_MODES[a["mode"]])
        return pm.OK

    def op_get_batch(self, a):
        mode = pm.GET_MODES[a["mode"]]
        return self.get_entry(self.eng.get_batch(a["reqs"], mode), mode)

    def op_collect(self, a):
        if a["h"] not in self.h:
            return pm.NONE
        kind, p, mode = self.h.pop(a["h"])
        if kind == "pending_get":
            return self.get_entry(p.collect(), mode)
        r = p.collect()
        out = self.range_entry(r, mode)
        if r.on_device:
            self.h[a["h"]] = ("range", r, mode)
        else:
            r.close()
        return out

    def op_pending_close(self, a):
        if a["h"] not in self.h:
            return pm.NONE
        self.h.pop(a["h"])[1].close()
        return pm.OK

    def op_range_prefetch(self, a):
        self.eng.range_prefetch(a["reqs"])
        return pm.OK

    def op_read(self, a):
        if a["h"] not in self.h:
            return pm.NONE
        x = self.h.pop(a["h"])
        if x[0] == "range":
            out = self.device_body(x[1], x[2])
        elif x[0] == "match":
            out = {"idx": x[1].device_event_idx().tolist()}
        else:  # a compaction sweep's device answer
            out = {"rec": x[1].device_array("victim_idx").astype(np.int64).tolist(),
                   "cls": x[1].device_array("victim_class").tolist()}
        x[1].close()
        return out

    def op_stream_open(self, a):
        self.h[a["h"]] = ("stream", self.eng.range_stream(a["req"], pm.MODES[a["mode"]], a["group"]), pm.MODES[a["mode"]])
        return pm.OK

    def op_stream_next(self, a):
        if a["h"] not in self.h:
            return pm.NONE
        _, s, mode = self.h[a["h"]]
        return self.page_entry(s.next(a["budget"]), mode)

    def op_stream_close(self, a):
        if a["h"] not in self.h:
            return pm.NONE
        self.h.pop(a["h"])[1].close()
        return pm.OK

    def op_partitions(self, a):
        borders, kv_first, arena_first = self.eng.range_partitions(a["start"], a["end"], a["rev"], a["part_bytes"],
                                                                   a["max_parts"])
        return {"borders": borders, "kv_first": kv_first.tolist(), "arena_first": arena_first.tolist()}

    def op_compact_sweep(self, a):
        mode = {"host": pm.KB_OUT_HOST, "device": pm.KB_OUT_DEVICE, "count": pm.KB_OUT_COUNT}[a["mode"]]
        c = self.eng.compact_sweep(a["start"], a["end"], a["rev"], a["timeout_rev"], a["support_ttl"], mode)
        out = {"n_victims": c.n_victims, "count": c.count, "examined": c.examined}
        if a["mode"] == "host":
            out.update(rec=c.victim_idx.astype(np.int64).tolist(), cls=c.victim_class.tolist())
        if a["mode"] == "device":
            self.h[a["h"]] = ("sweep", c)
        else:
            c.close()
        return out

    def op_cstream_open(self, a):
        c = self.eng.compact_stream(a["start"], a["end"], a["rev"], a["timeout_rev"], a["support_ttl"], a["group"])
        self.h[a["h"]] = ("cstream", c)
        return {"n_victims": c.n_victims, "count": c.count, "examined": c.examined}

    def op_cstream_next(self, a):
        if a["h"] not in self.h:
            return pm.NONE
        p = self.h[a["h"]][1].next(a["budget"])
        if p is None:
            return None
        return {"first": p.first, "n": p.n, "rec": p.rec_idx.astype(np.int64).tolist(), "cls": p.victim_class.tolist(),
                "keys": p.keys(), "guards": p.guards()}

    def op_cstream_close(self, a):
        if a["h"] not in self.h:
            return pm.NONE
        self.h.pop(a["h"])[1].close()
        return pm.OK

    def op_apply(self, a):
        self.eng.apply_batch(a["ops"])
        return pm.OK

    def op_expire(self, a):
        return ("dropped", self.eng.expire(a["now"]))

    def op_load(self, a):
        self.eng.load_sorted(PackedStore.from_items(a["items"]))
        return pm.OK

    def op_dump(self, a):
        self.eng.dump(self.path)
        with open(self.path, "rb") as f:
            return pm.dump_entry(f.read())

    def op_restore(self, a):
        self.eng.restore(self.path)
        return pm.OK

    def op_set_compact_revision(self, a):
        self.eng.set_compact_revision(a["rev"])
        return pm.OK

    def op_store_info(self, a):
        return ("info",) + self.eng.store_info()

    def op_watch_add(self, a):
        i = self.eng.watch_add(a["prefix"], a["min_rev"])
        self.h[a["h"]] = ("watch", i)
        return ("id", i)

    def op_watch_del(self, a):
        self.eng.watch_del(self.h.pop(a["h"])[1])
        return pm.OK

    def op_match(self, a):
        m = self.eng.watch_match(fuzz.fuzz_events(a["burst"]), pm.KB_OUT_DEVICE if a["mode"] == "device" else pm.KB_OUT_HOST)
        return self.match_entry(m, a["h"])

    def op_events_upload(self, a):
        self.h[a["h"]] = ("events", self.eng.events_upload(fuzz.fuzz_events(a["burst"])))
        return pm.OK

    def op_match_dev(self, a):
        return self.match_entry(self.eng.watch_match_dev(self.h[a["ev"]][1]), a["h"])

    def op_events_free(self, a):
        self.eng.events_free(self.h.pop(a["ev"])[1])
        return pm.OK

    def close_all(self):
        """frees the results, event slabs and pendings still held (a pending ends in collect or kb_pending_free), then
        closes the context with whatever range and compaction streams the program left open: kb_close frees those, and
        their handles' close() is a no-op afterwards"""
        for x in self.h.values():
            if x[0] == "events":
                self.eng.events_free(x[1])
            elif x[0] in ("range", "match", "sweep", "pending", "pending_get"):
                x[1].close()
        self.eng.close()
        for x in self.h.values():
            if x[0] in ("stream", "cstream"):
                x[1].close()
        self.h.clear()


def _mismatch(p: pm.Program, i: int, exp, got) -> str:
    lines = ["seed %d, KB_LANES %d, op %d: %s" % (p.seed, p.n_lanes, i, pm.describe(p.ops[i]))]
    if isinstance(exp, dict) and isinstance(got, dict):
        for k in sorted(set(exp) | set(got)):
            if exp.get(k) != got.get(k):
                lines.append("  %s: expected %s, got %s" % (k, pm.short(exp.get(k), 300), pm.short(got.get(k), 300)))
    else:
        lines.append("  expected %s\n  got      %s" % (pm.short(exp, 300), pm.short(got, 300)))
    lines.append("the 20 ops before it:")
    lines += ["  %4d %s" % (j, pm.describe(p.ops[j])[:200]) for j in range(max(0, i - 20), i)]
    lines.append("python -m tests.program_model --seed %d --lanes %d prints the whole program" % (p.seed, p.n_lanes))
    return "\n".join(lines)


@pytest.mark.parametrize("n_lanes", pm.LANES)
@pytest.mark.parametrize("seed", pm.SEEDS)
def test_program(monkeypatch, tmp_path, seed, n_lanes):
    monkeypatch.setenv("KB_LANES", str(n_lanes))  # kb_open reads it every time
    p = pm.gen_program(seed, n_lanes)
    expected, _ = pm.run_program(p)
    eng = Engine(0)
    run = Runner(eng, str(tmp_path / "program.kbd"))
    try:
        eng.load_sorted(PackedStore.from_items(p.start))
        for i, op in enumerate(p.ops):
            got = run.step(*op)
            assert got == expected[i], _mismatch(p, i, expected[i], got)
    finally:
        run.close_all()
