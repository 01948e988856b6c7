"""Deterministic plans for concurrent callers, and their expected answers (CPU only).

A plan is a base store v0, K write batches that make the versions v1 .. vK, and reads whose expected answers do not
depend on how the threads that issue them are scheduled:

* Writes are shaped like the backend's commits -- a revision-record CAS plus an object put at a fresh revision above
  every read revision of the plan, deletes as a tombstone version plus a deleted-flag revision record, and `/events/`
  puts with an expiry -- and land under WRITE_PREFIX, whose records sort after those of every invariant read.
* An invariant read reads at a revision <= the base revision inside [INV_LO, INV_HI): its answer, record indices
  included, is the same on every version.  `invariant` checks that with the C oracle instead of taking it on trust.
* A window read reads the latest state (point reads at revision 0, counts at 2^64 - 1, kb_store_info).  Its answer is
  precomputed on every version; one issued while the writer had published version a and returned when it had published
  b must equal the answer at some version in [a, b + 1], and one thread's window reads never go back in version.
* Fan-out bursts (tests/fuzz.py's seq_rotation bursts and shape_a's large burst) against one fixed watcher set.

Every expected answer is a dict of byte strings ("parts"); `digest` folds it into one key, so a thread checks an answer
with one dict lookup.  `python -m tests.concurrent_plan --seed S` prints a plan and the classes it reaches."""
from __future__ import annotations

import argparse
import hashlib
import random
import struct
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from kubebrain_b200 import synth
from kubebrain_b200._lib import KB_OUT_COUNT, KB_OUT_DEVICE, KB_OUT_HOST, KB_WIRE_ETCD_EVENTS, KB_WIRE_ETCD_KVS
from kubebrain_b200.packed import PackedStore, PackedWatchers, Slab
from oracle import binding as ko
from tests import fuzz
from tests import partition_shapes as ps

MAGIC = fuzz.MAGIC
ALL = 2**64 - 1
FZ = b"/fz/"            # fuzz_store's user keys are moved under this prefix: they sort before the synthetic store's
WRITE_PREFIX = b"/zz/"  # every write of a plan: after "/registry/" and "/fz/"
INV_LO, INV_HI = MAGIC, MAGIC + WRITE_PREFIX  # the records every invariant read may see
LONG_UK = FZ + b"long/" + b"y" * (65535 - 13 - len(FZ) - 5)  # an internal key of 65 535 bytes
MODES = {"host": KB_OUT_HOST, "device": KB_OUT_DEVICE, "kvs": KB_OUT_HOST | KB_WIRE_ETCD_KVS,
         "events": KB_OUT_DEVICE | KB_WIRE_ETCD_EVENTS, "dev_kvs": KB_OUT_DEVICE | KB_WIRE_ETCD_KVS, "count": KB_OUT_COUNT}
GET_MODES = {"host": KB_OUT_HOST, "kvs": KB_OUT_HOST | KB_WIRE_ETCD_KVS}
PAGE_BUDGET = 6000     # a range stream's byte budget: several pages per stream
GROUP = 7              # kvs per range-stream group, victims per compaction-stream group
EXPIRE_NOW = 2_000_000_000
SWEEP_REV = 60  # a compaction sweep records its revision as the compact revision: every read of a plan is at or above it


def ik(uk: bytes, rev: int) -> bytes:
    return MAGIC + uk + b"$" + struct.pack(">Q", rev)


def pad16(b: bytes) -> bytes:
    return b + b"\0" * (-len(b) % 16)


def digest(parts: Dict[str, bytes]) -> str:
    h = hashlib.sha1()
    for k in sorted(parts):
        v = parts[k]
        h.update(b"%s:%d:" % (k.encode(), len(v)))
        h.update(v)
    return h.hexdigest()


def first_difference(exp: Dict[str, bytes], got: Dict[str, bytes]) -> str:
    """the first part, and the first byte in it, where two answers differ"""
    for k in sorted(set(exp) | set(got)):
        a, b = exp.get(k, b""), got.get(k, b"")
        if a != b:
            n = min(len(a), len(b))
            i = next((j for j in range(n) if a[j] != b[j]), n)
            return "%s differs at byte %d (expected %d bytes, got %d)" % (k, i, len(a), len(b))
    return "no difference"


def _u64(x) -> bytes:
    return np.ascontiguousarray(np.asarray(x, dtype=np.uint64)).tobytes()


# ---- expected answers ------------------------------------------------------------------------------------------------
def range_parts(store: PackedStore, st: ko.OracleStore, reqs, mode: str) -> Dict[str, bytes]:
    """a range batch: rows, record indices, revisions, arena bytes (padding included) or wire elements and offsets"""
    if mode == "count":
        return {"count": _u64([ko.scan(st, [s, e], r, collect=False).count for s, e, r, _ in reqs])}
    xs = [ko.range_(st, s, e, r, lim) for s, e, r, lim in reqs]
    assert all(x.rc == 0 for x in xs)
    rec = np.concatenate([x.emit for x in xs]).astype(np.uint64) if xs else np.zeros(0, np.uint64)
    out = {"first": _u64(np.cumsum([0] + [len(x.emit) for x in xs])), "count": _u64([x.count for x in xs]),
           "examined": _u64([x.examined for x in xs]), "rec": _u64(rec),
           "rev": _u64([int.from_bytes(store.keys[int(i)][-8:], "big") for i in rec])}
    wire = MODES[mode] & (KB_WIRE_ETCD_KVS | KB_WIRE_ETCD_EVENTS)
    if wire:
        image, off = ko.wire_encode(st, rec, ko.WIRE_KVS if wire == KB_WIRE_ETCD_KVS else ko.WIRE_EVENTS)
        out.update(image=image, elem_off=_u64(off))
    else:
        out["image"] = b"".join(pad16(store.keys[int(i)]) + pad16(store.vals[int(i)]) for i in rec)
    return out


def get_parts(store: PackedStore, st: ko.OracleStore, reqs, mode: str) -> Dict[str, bytes]:
    """point reads: status, mod_rev, the record of every FOUND read and its value, or its RangeResponse element"""
    status, mod, rec, vals = [], [], [], []
    for k, rev in reqs:
        idx, m = ko.get(st, k, rev)
        status.append(0 if idx >= 0 else 2 if idx == -2 else 1)
        mod.append(m if idx != -1 else 0)
        rec.append(idx if idx >= 0 else 0)
        if idx < 0:
            vals.append(b"")
        elif mode == "kvs":
            vals.append(ko.wire_encode(st, [idx], ko.WIRE_KVS)[0])
        else:
            vals.append(store.vals[idx])
    return {"status": bytes(status), "mod_rev": _u64(mod), "rec": _u64(rec),
            "vals": b"".join(struct.pack("<I", len(v)) + v for v in vals)}


def stream_parts(store: PackedStore, st: ko.OracleStore, req, mode: str) -> Dict[str, bytes]:
    """a range stream read to the end: the pages' records, bytes and offsets concatenated, and the page sizes"""
    from tests.test_gpu_range_stream import greedy_cuts
    p = range_parts(store, st, [req], mode)
    rec = np.frombuffer(p["rec"], np.uint64)
    if "elem_off" in p:
        sizes = np.diff(np.frombuffer(p["elem_off"], np.uint64).astype(np.int64))
    else:
        sizes = np.array([len(pad16(store.keys[int(i)])) + len(pad16(store.vals[int(i)])) for i in rec], np.int64)
    cuts = greedy_cuts(sizes, GROUP, PAGE_BUDGET)
    return {"rec": p["rec"], "image": p["image"], "pages": _u64([b - a for a, b in cuts])}


def partition_parts(store: PackedStore, st: ko.OracleStore, start: bytes, end: bytes, rev: int, part_bytes: int,
                    max_parts: int) -> Dict[str, bytes]:
    borders, kv_first, arena_first = ps.partitions(store, st, start, end, rev, part_bytes, max_parts)
    return {"borders": b"".join(struct.pack("<I", len(b)) + b for b in borders), "kv_first": _u64(kv_first),
            "arena_first": _u64(arena_first)}


def sweep_parts(store: PackedStore, st: ko.OracleStore, start: bytes, end: bytes, rev: int) -> Dict[str, bytes]:
    """a compaction sweep's delete-call list: records, classes, count and examined (the compaction stream adds each
    victim's internal key and the guard of classes 3 / 4)"""
    x = ko.worker_run(st, start, end, rev, compact=True, timeout_rev=0, support_ttl=True, collect=True)
    assert x.rc == 0
    keys = [store.keys[int(i)] for i in x.victims]
    guards = [store.vals[int(i)] if c in (3, 4) else b"" for i, c in zip(x.victims, x.vclass)]
    return {"rec": _u64(x.victims), "cls": x.vclass.astype(np.uint8).tobytes(), "count": _u64([x.count]),
            "examined": _u64([x.examined]), "keys": b"".join(struct.pack("<I", len(k)) + k for k in keys),
            "guards": b"".join(struct.pack("<I", len(g)) + g for g in guards)}


def live_bytes(store: PackedStore) -> Tuple[int, int]:
    """the key-slab and value-heap bytes of a freshly laid-out snapshot; kb_store_info's can be larger by the garbage
    the writes left behind, which a layout compaction reclaims when no compaction stream defers it -- so by the schedule"""
    return sum(len(pad16(k)) for k in store.keys.tolist()), sum(len(pad16(v)) for v in store.vals.tolist())


def info_ok(plan: "Plan", v: int, got: Tuple[int, int, int]) -> bool:
    kb, vb = plan.live[v]
    return got[0] == plan.stores[v].n and got[1] >= kb and got[2] >= vb


# ---- stores and writes -----------------------------------------------------------------------------------------------
def base_items(seed: int, n_objects: int, lv: int) -> Tuple[Dict[bytes, bytes], int, synth.StoreMeta]:
    """a config-2-shaped store, fuzz_store's records under FZ, a 65 535-byte key, and pre-existing objects under
    WRITE_PREFIX for the plan's writes to update and delete"""
    store, meta = synth.gen_store(n_objects, 4, 64, lv, 40, config_id=2, tomb_frac=0.1)
    items = dict(zip(store.keys.tolist(), store.vals.tolist()))
    fz = fuzz.fuzz_store(seed, n_keys=120, max_rev=900)
    for k, v in zip(fz.keys.tolist(), fz.vals.tolist()):
        items[MAGIC + FZ + k[4:] if k.startswith(MAGIC) else k] = v
    items[ik(LONG_UK, 0)] = struct.pack(">Q", 950)
    items[ik(LONG_UK, 950)] = b"long value"
    base_rev = meta.last_rev
    for i in range(24):
        uk = WRITE_PREFIX + b"obj/%04d" % i
        items[ik(uk, 0)] = struct.pack(">Q", 500 + i)
        items[ik(uk, 500 + i)] = b"v0-%d" % i * 3
    return items, base_rev, meta


def commit_put(uk: bytes, rev: int, val: bytes, expire: int = 0) -> List[tuple]:
    return [(ik(uk, 0), struct.pack(">Q", rev), expire), (ik(uk, rev), val, expire)]


def commit_delete(uk: bytes, rev: int) -> List[tuple]:
    return [(ik(uk, 0), struct.pack(">Q", rev) + b"\0"), (ik(uk, rev), b"tombstone")]


def apply(items: Dict[bytes, bytes], ops: Sequence[tuple]) -> Dict[bytes, bytes]:
    out = dict(items)
    for op in ops:
        if op[1] is None:
            out.pop(op[0], None)
        else:
            out[op[0]] = op[1]
    return out


def write_batches(seed: int, base_rev: int, k: int, low: bool = False) -> List[List[tuple]]:
    """K commits' worth of batches at fresh revisions above base_rev (low=True: the wrong variant, whose revisions start
    at or below it and land among the invariant reads' records)"""
    rng = random.Random(seed ^ 0x77)
    rev = base_rev - 40 if low else base_rev
    out = []
    for b in range(k):
        ops = []
        for _ in range(rng.randint(2, 4)):
            rev += 1
            kind = rng.random()
            uk = (FZ + b"a" if low else WRITE_PREFIX) + b"obj/%04d" % rng.randrange(32)
            if kind < 0.25:
                ops += commit_delete(uk, rev)
            elif kind < 0.5:
                ops += commit_put(WRITE_PREFIX + b"events/ns/%04d" % rng.randrange(1000), rev, b"ev%d" % rev,
                                  EXPIRE_NOW - 5)
            else:
                ops += commit_put(uk, rev, bytes(rng.randrange(256) for _ in range(rng.choice([1, 15, 16, 17, 300]))))
        out.append(ops)
    return out


# ---- the plan --------------------------------------------------------------------------------------------------------
@dataclass
class Read:
    kind: str      # range | get | stream | partitions | sweep | cstream | count | info
    args: dict
    answers: List[str] = field(default_factory=list)  # digest on every version v0 .. vK
    exp: Optional[Dict[str, bytes]] = None             # the parts on v0 (first_difference of a wrong answer)

    @property
    def invariant(self) -> bool:
        return len(set(self.answers)) == 1


@dataclass
class Plan:
    seed: int
    base_rev: int
    items: List[Dict[bytes, bytes]]      # v0 .. vK
    batches: List[List[tuple]]           # batch k makes version k + 1
    reads: List[Read]
    meta: synth.StoreMeta
    reconcile: Tuple[bytes, bytes]       # the interval the writer lets diverge, then repairs
    stores: List[PackedStore] = field(default_factory=list)
    live: List[Tuple[int, int]] = field(default_factory=list)  # live_bytes of every version

    def store(self, v: int) -> PackedStore:
        return self.stores[v]

    @property
    def invariant_reads(self) -> List[Read]:
        return [r for r in self.reads if r.invariant]

    @property
    def window_reads(self) -> List[Read]:
        return [r for r in self.reads if not r.invariant]


def answer_of(read: Read, store: PackedStore, st: ko.OracleStore) -> Dict[str, bytes]:
    a = read.args
    if read.kind in ("range", "count"):
        return range_parts(store, st, a["reqs"], a["mode"])
    if read.kind == "get":
        return get_parts(store, st, a["reqs"], a["mode"])
    if read.kind == "stream":
        return stream_parts(store, st, a["req"], a["mode"])
    if read.kind == "partitions":
        return partition_parts(store, st, a["start"], a["end"], a["rev"], a["part_bytes"], a["max_parts"])
    if read.kind in ("sweep", "cstream"):
        return sweep_parts(store, st, a["start"], a["end"], a["rev"])
    if read.kind == "info":
        return {"n": _u64([store.n])}
    raise ValueError(read.kind)


def _reads(seed: int, items: Dict[bytes, bytes], meta: synth.StoreMeta, base_rev: int) -> List[Read]:
    rng = random.Random(seed)
    pods = MAGIC + b"/registry/pods/"
    keys = sorted(k for k in items if INV_LO <= k < INV_HI)
    revs = [meta.read_rev, base_rev, meta.first_rev + 1, 60, 900]
    out = []

    def span():
        a, b = sorted(rng.sample(keys, 2))
        return a[: rng.randint(5, len(a))], b

    for i in range(10):
        mode = ("host", "device", "kvs", "events", "dev_kvs", "count")[i % 6]
        reqs = [(*span(), rng.choice(revs), rng.choice([0, 1, 17, 300])) for _ in range(rng.randint(1, 4))]
        reqs.append((pods, pods + b"\xff", meta.read_rev, 50))
        if mode == "count":
            reqs = [(s, e, r, 0) for s, e, r, _ in reqs]
        out.append(Read("range", dict(reqs=reqs, mode=mode)))
    uks = sorted({fuzz_uk for fuzz_uk in (ko.decode(k)[0] for k in keys) if fuzz_uk is not None})
    for mode in ("host", "kvs"):
        reqs = [(rng.choice(uks), rng.choice([rng.choice(revs), rng.randint(SWEEP_REV, base_rev)])) for _ in range(12)]
        reqs.append((LONG_UK, 950))
        out.append(Read("get", dict(reqs=reqs, mode=mode)))
    out.append(Read("stream", dict(req=(MAGIC + FZ, INV_HI, 900, 0), mode="host")))
    out.append(Read("stream", dict(req=(pods, pods + b"\xff", meta.read_rev, 0), mode="kvs")))
    out.append(Read("partitions", dict(start=MAGIC + FZ, end=INV_HI, rev=base_rev, part_bytes=4096, max_parts=9)))
    out.append(Read("sweep", dict(start=INV_LO, end=INV_HI, rev=SWEEP_REV)))
    out.append(Read("cstream", dict(start=MAGIC + FZ, end=MAGIC + b"/registry/pods/", rev=SWEEP_REV)))
    # window reads: the latest state
    wk = [WRITE_PREFIX + b"obj/%04d" % i for i in range(0, 32, 3)] + [uks[0], LONG_UK]
    out.append(Read("get", dict(reqs=[(k, 0) for k in wk], mode="host")))
    out.append(Read("get", dict(reqs=[(k, 0) for k in wk[:5]], mode="kvs")))
    out.append(Read("count", dict(reqs=[(INV_LO, MAGIC + b"\xff", ALL, 0), (MAGIC + WRITE_PREFIX, MAGIC + b"/zz0", ALL, 0)],
                                  mode="count")))
    out.append(Read("info", {}))
    return out


def gen_plan(seed: int, k: int = 6, n_objects: int = 2500, lv: int = 2048, low: bool = False) -> Plan:
    items0, base_rev, meta = base_items(seed, n_objects, lv)
    batches = write_batches(seed, base_rev, k, low)
    items = [items0]
    for b in batches:
        items.append(apply(items[-1], b))
    plan = Plan(seed, base_rev, items, batches, _reads(seed, items0, meta, base_rev), meta,
                (MAGIC + WRITE_PREFIX + b"obj/", MAGIC + WRITE_PREFIX + b"obj0"))
    plan.stores = [PackedStore.from_items(list(it.items())) for it in items]
    plan.live = [live_bytes(s) for s in plan.stores]
    sts = [ko.OracleStore(s) for s in plan.stores]
    for r in plan.reads:
        parts = [answer_of(r, s, st) for s, st in zip(plan.stores, sts)]
        r.answers = [digest(p) for p in parts]
        r.exp = parts[0]
    return plan


# ---- fan-out ---------------------------------------------------------------------------------------------------------
@dataclass
class Bursts:
    events: list
    watchers: PackedWatchers
    expected: List[Tuple[np.ndarray, np.ndarray]]  # (start, idx) of every burst


def gen_bursts() -> Bursts:
    """seq_rotation's bursts (one geometry, different data) and shape_a's large burst, against one watcher set: the
    rotation's watchers followed by shape_a's"""
    seq, w1 = fuzz.seq_rotation(n_bursts=3)
    ev_a, w2 = fuzz.shape_a("random", "irregular")
    pre = w1.prefixes.tolist() + w2.prefixes.tolist()
    w = PackedWatchers(Slab.from_list(pre), np.concatenate([w1.min_rev, w2.min_rev]).astype(np.uint64))
    events = seq + [ev_a]
    return Bursts(events, w, [ko.fanout(ev, w, threads=2)[:2] for ev in events])


def classes(plan: Plan) -> Dict[str, object]:
    inv, win = plan.invariant_reads, plan.window_reads
    return {"versions": len(plan.items), "records_v0": plan.stores[0].n, "base_rev": plan.base_rev,
            "invariant": sorted({"%s/%s" % (r.kind, r.args.get("mode", "-")) for r in inv}),
            "window": sorted({"%s/%s" % (r.kind, r.args.get("mode", "-")) for r in win}),
            "ops": sorted({("del" if v is not None and v.endswith(b"\0") and len(v) == 9 else
                            "ttl" if len(op) > 2 and op[2] else "put")
                           for b in plan.batches for op in b for v in [op[1]] if op[0].endswith(b"\0" * 8)}),
            "long_key": any(len(k) == 65535 for k in plan.items[0]),
            "undecodable": sum(1 for k in plan.items[0] if ko.decode(k)[0] is None)}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    p = gen_plan(a.seed)
    for i, b in enumerate(p.batches):
        print("v%d: %s" % (i + 1, ", ".join("%s%s" % ("put " if op[1] is not None else "del ", op[0][4:48])
                                            for op in b)))
    for r in p.reads:
        print("%-9s %-10s %s  %s" % ("invariant" if r.invariant else "window", r.kind, r.args.get("mode", "-"),
                                     " ".join(x[:8] for x in r.answers)))
    print(classes(p))
