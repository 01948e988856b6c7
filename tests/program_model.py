"""Seeded programs that interleave every entry point of one context, and the model that predicts their transcript.

The caller families share context state: the lanes (lane_take / ctx_quiesce read back the rows of what is in flight
before another call reuses a lane's staging, search slab, d_sel or d_slot), the two prefetch slots (voided by
store_gen), the range streams (re-scanned when store_gen moves), the compaction streams (they pin the heap; load,
restore and dump invalidate them), the compact revision and the watcher table.  A lost store_gen bump or a lane buffer
reused one call too early shows only when several families meet on one context, so a program mixes them on purpose.

`gen_program(seed, n_lanes)` builds a starting store, watchers and 230-290 ops drawn from every entry point: 23 scripted
episodes, each aimed at one hazard, in a seeded order with a random op between some of them, then the closing ops.  The
episodes alone take that many ops, more than the 120-200 first planned.  SEEDS x LANES is the committed set that tests/test_gpu_programs.py runs.  `Model(variant).run(program)`
computes the expected transcript, one entry per op, from the C oracle alone (ko.range_, ko.get, ko.scan(compact=True),
ko.wire_encode, ko.fanout), partition_shapes.partitions, greedy_cuts / expected of test_gpu_range_stream, and
write_shapes.HeapModel / dump_image.  Each rule the model applies is one method whose docstring names the part of
include/kb_b200.h (or the code line) it restates; `variant` swaps one rule for a plausible wrong one, which is how
tests/test_programs.py shows that the programs tell every rule apart.  The model also records the hazard classes a
program reaches (`Model.classes`).

`python -m tests.program_model --seed S --lanes L` prints a program and its expected transcript."""
from __future__ import annotations

import argparse
import hashlib
import random
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Set, Tuple

import numpy as np

from kubebrain_b200._lib import (KB_ECOMPACTED, KB_ELIMIT, KB_ESTATE, KB_OUT_COUNT, KB_OUT_DEVICE, KB_OUT_HOST,
                                 KB_WIRE_ETCD_EVENTS, KB_WIRE_ETCD_KVS)
from kubebrain_b200.packed import PackedStore, PackedWatchers, Slab
from oracle import binding as ko
from tests import fuzz
from tests import partition_shapes as ps
from tests import write_shapes as ws
from tests.range_shapes import TOMB, be, ik
from tests.test_gpu_range_stream import expected as stream_expected
from tests.test_gpu_range_stream import greedy_cuts

ALL = 2**64 - 1
T0 = 1_700_000_000
MAGIC = ws.MAGIC
FULL = (b"\x00", b"\xff" * 4)
MAX_KEY = 65535
LONG_UK = b"/long/" + b"L" * (MAX_KEY - 13 - 6)  # its internal keys are exactly 65 535 bytes

MODES = {"host": KB_OUT_HOST, "device": KB_OUT_DEVICE, "count": KB_OUT_COUNT,
         "kvs": KB_OUT_HOST | KB_WIRE_ETCD_KVS, "events": KB_OUT_HOST | KB_WIRE_ETCD_EVENTS,
         "dev_kvs": KB_OUT_DEVICE | KB_WIRE_ETCD_KVS, "dev_events": KB_OUT_DEVICE | KB_WIRE_ETCD_EVENTS}
GET_MODES = {"host": KB_OUT_HOST, "device": KB_OUT_DEVICE, "kvs": KB_OUT_HOST | KB_WIRE_ETCD_KVS}
SNAPSHOT_CHANGES = ("write", "expire", "load", "restore", "dump")
SEEDS = range(6)
LANES = (1, 2, 4)
VARIANTS = ("R1", "R2", "R3", "R4_start", "R4_nozero", "R4_limit_done", "R5", "R6", "R7")

# the hazard classes every committed (seed, n_lanes) set has to reach at each lane count ("other lanes" needs two)
LANE_CLASSES = ("lane_busy:stream", "lane_busy:partitions", "lane_busy:match")
CLASSES = LANE_CLASSES + tuple("collected_after:" + k for k in SNAPSHOT_CHANGES) + (
    "prefetch_both_valid_across_write",) + tuple("stream_rescan:" + k for k in SNAPSHOT_CHANGES) + (
    "stream_rescan_beside_streams", "stream_rescan_at_key_limit",
    "cstream_deferred_then_invalidated:load", "cstream_deferred_then_invalidated:restore",
    "cstream_deferred_then_invalidated:dump", "deferred_compaction_after_last_close",
    "ecompacted_then_batch_same_lane", "watcher_churn_in_flight", "device_answer_across_layout_compaction")
MULTI_LANE_CLASSES = ("partitions_beside_other_lanes_and_streams",)


def wire_of(mode: int) -> int:
    return mode & (KB_WIRE_ETCD_KVS | KB_WIRE_ETCD_EVENTS)


def base_of(mode: int) -> int:
    return mode & 0xF


def pad16(b: bytes) -> bytes:
    return ws.pad16(b)


def key_after(k: bytes) -> Optional[bytes]:
    """kb_page.cu key_after: the least internal key greater than every key that starts with k -- k + 0x00, or, for a
    key at the 65 535-byte limit, k without its trailing 0xff bytes and with the last byte left incremented"""
    if len(k) < MAX_KEY:
        return k + b"\x00"
    k = k.rstrip(b"\xff")
    if not k:
        return None
    return k[:-1] + bytes([k[-1] + 1])


# ---- programs ---------------------------------------------------------------------------------------------------------
@dataclass
class Program:
    seed: int
    n_lanes: int
    start: List[Tuple[bytes, bytes]]
    ops: List[Tuple[str, dict]] = field(default_factory=list)


def start_items(seed: int) -> Dict[bytes, bytes]:
    """a fuzz store (tombstones, deleted-flag revision records, undecodable records, '$' inside user keys) with internal
    keys on both sides of the 16 / 32 / 48-byte chunk borders, `/events/` keys, and two keys at the 65 535-byte limit"""
    st = fuzz.fuzz_store(7000 + seed, n_keys=600 + 40 * (seed % 5))
    items = dict(zip(st.keys.tolist(), st.vals.tolist()))
    for L in (15, 16, 17, 31, 32, 33, 47, 48, 49):
        uk = (b"/c/%02d/" % L + b"k" * 64)[: L - 13]
        items[ik(uk, 0)] = be(20)
        items[ik(uk, 20)] = b"v" * L
        items[ik(uk, 3)] = b"old"
    for j in range(60):
        uk = b"/events/e%03d" % j
        items[ik(uk, 0)] = be(10 + j % 40, j % 7 == 0)
        items[ik(uk, 10 + j % 40)] = b"ev%d" % j * (j % 5)
    items[ik(LONG_UK, 0)] = be(5)
    items[ik(LONG_UK, 5)] = b"long value"
    return items


class _Gen:
    """the generator's own view of the program: enough state to aim its ops (it never predicts an answer)"""

    def __init__(self, seed: int, n_lanes: int):
        self.rng = random.Random(seed * 1009 + n_lanes)
        self.seed, self.n_lanes = seed, n_lanes
        self.items = start_items(seed)
        self.ops: List[Tuple[str, dict]] = []
        self.rev = 100
        self.ttl_t = T0
        self.n_handles = 0
        self.watchers: List[str] = []
        self.open_streams: List[str] = []
        self.open_cstreams: List[str] = []
        self.pendings: List[str] = []
        self.held: List[str] = []  # device-resident answers not read back yet
        self.device_pendings: Set[str] = set()
        self.dumped: Optional[Dict[bytes, bytes]] = None  # the generator's view of the last dump
        self._keys: Optional[List[bytes]] = None

    # -- helpers
    def h(self, p: str) -> str:
        self.n_handles += 1
        return "%s%d" % (p, self.n_handles)

    def emit(self, kind: str, **a):
        self.ops.append((kind, a))

    def keys(self) -> List[bytes]:
        if self._keys is None:
            self._keys = sorted(self.items)
        return self._keys

    def uks(self) -> List[bytes]:
        return [u for u in (ws.user_key(k) for k in self.keys()) if u is not None and len(u) < 2000]

    def next_rev(self) -> int:
        self.rev += 1
        return self.rev

    def read_rev(self) -> int:
        return self.rng.choice([ALL, ALL, 30, 59, self.rev, self.rev - 2, 105])

    def bounds(self) -> Tuple[bytes, bytes]:
        r = self.rng.random()
        if r < 0.3:
            return FULL
        if r < 0.4:
            return MAGIC, MAGIC + b"\xff" * 8
        if r < 0.5:
            return ik(b"/events/", 0), ik(b"/events0", 0)
        keys = self.keys()
        a, b = self.rng.choice(keys), self.rng.choice(keys)
        if self.rng.random() < 0.5:
            a = a[: self.rng.randint(1, max(len(a), 1))]
        if self.rng.random() < 0.5:
            b = b[: self.rng.randint(1, max(len(b), 1))] + b"\xff"
        return (a, b) if a <= b else (b, a)

    def reqs(self, n: Optional[int] = None, count: bool = False):
        out = []
        for _ in range(n or self.rng.randint(1, 3)):
            s, e = self.bounds()
            out.append((s, e, self.read_rev(), 0 if count else self.rng.choice([0, 0, 0, 1, 3, 50])))
        return out

    def mode(self) -> str:
        return self.rng.choice(list(MODES))

    def apply_local(self, ops):
        for op in ops:
            if op[1] is None:
                self.items.pop(op[0], None)
            else:
                self.items[op[0]] = op[1]
        self._keys = None

    # -- op makers
    def write(self, n: Optional[int] = None, ttl: bool = False):
        rng, ops = self.rng, []
        uks = self.uks()
        keys = self.keys()
        for _ in range(n or rng.randint(4, 30)):
            r = rng.random()
            uk = rng.choice(uks)
            if r < 0.35:
                rev = self.next_rev()
                ops += [(ik(uk, rev), bytes([rng.randrange(256)]) * rng.randint(0, 70)), (ik(uk, 0), be(rev))]
            elif r < 0.45:
                rev = self.next_rev()
                ops += [(ik(uk, rev), TOMB), (ik(uk, 0), be(rev, True))]
            elif r < 0.7:
                ops.append((rng.choice(keys), None))
            elif r < 0.8:
                v = ik(uk, rng.randint(1, 59))  # a version at or below the fuzz store's revisions: old reads see it
                ops.append((v, b"back" * rng.randint(0, 9)))
            elif r < 0.9:
                nu = uk + b"/new%d" % rng.randrange(1000)
                rev = self.next_rev()
                ops += [(ik(nu, rev), b"n" * rng.randint(1, 40)), (ik(nu, 0), be(rev))]
            else:
                ops.append((ik(uk + b"/gone", 7), None))  # absent: a no-op
        if ttl or rng.random() < 0.3:
            for j in range(rng.randint(1, 6)):
                self.ttl_t += rng.randint(0, 3)
                ops.append((ik(b"/events/ttl%04d" % rng.randrange(300), self.next_rev()), b"t" * j, self.ttl_t))
        self.apply_local(ops)
        self.emit("apply", ops=ops)

    def invalid_write(self):
        ops = [(ik(self.rng.choice(self.uks()), self.next_rev()), b"ok"), (b"k" * 65536, b"too long")]
        self.rng.shuffle(ops)
        self.emit("apply", ops=ops)

    def big_delete(self):
        """deletes a third of the records: garbage_k passes a quarter of the key tail (the layout-compaction trigger)"""
        keys = [k for k in self.keys() if len(k) < 60000]
        ops = [(k, None) for k in self.rng.sample(keys, len(keys) // 3)]
        self.apply_local(ops)
        self.emit("apply", ops=ops)

    def big_replace(self):
        """replaces the value of every object record by as many bytes: the old values become garbage past a quarter of
        the value tail (the layout-compaction trigger) while the store keeps its records"""
        recs = [k for k in self.keys() if len(k) < 60000 and ws.user_key(k) is not None and k[-8:] != bytes(8)]
        self.apply_emit([(k, b"r" * len(self.items[k])) for k in recs])

    def expire(self):
        self.emit("expire", now=self.ttl_t + self.rng.randint(-2, 3))

    def load(self):
        items = start_items(self.seed + 50 + self.rng.randrange(3))
        for k in self.rng.sample(sorted(items), len(items) // 10):
            del items[k]
        self.items = items
        self._keys = None
        self.emit("load", items=sorted(items.items()))

    def dump(self):
        self.emit("dump")
        self.dumped = dict(self.items)

    def restore(self):
        if self.dumped is None:
            self.dump()
        self.emit("restore")
        self.items = dict(self.dumped)
        self._keys = None

    def change(self, kind: str):
        {"write": self.write, "expire": self.expire_due, "load": self.load, "restore": self.restore,
         "dump": self.dump_changed}[kind]()

    def expire_due(self):
        self.write(n=2, ttl=True)
        self.emit("expire", now=self.ttl_t + 5)

    def dump_changed(self):
        self.write(n=3)  # so that the dump rewrites the layout (and moves store_gen)
        self.dump()

    def submit(self, kind: Optional[str] = None, mode: Optional[str] = None) -> str:
        h = self.h("p")
        if (kind or self.rng.choice(["range", "range", "get"])) == "get":
            self.emit("get_submit", reqs=self.gets(), mode=mode or self.rng.choice(list(GET_MODES)), h=h)
        else:
            m = mode or self.mode()
            self.emit("range_submit", reqs=self.reqs(count=m == "count"), mode=m, h=h)
            if base_of(MODES[m]) == KB_OUT_DEVICE:
                self.device_pendings.add(h)
        self.pendings.append(h)
        return h

    def collect_some(self, k: Optional[int] = None):
        self.rng.shuffle(self.pendings)
        k = len(self.pendings) if k is None else min(k, len(self.pendings))
        for _ in range(k):
            h = self.pendings.pop()
            if self.rng.random() < 0.08:
                self.emit("pending_close", h=h)
            else:
                self.emit("collect", h=h)
                if h in self.device_pendings:
                    self.held.append(h)

    def gets(self):
        out = []
        for _ in range(self.rng.randint(1, 12)):
            uk = self.rng.choice(self.uks())
            out.append((uk if self.rng.random() < 0.9 else uk + b"?", self.rng.choice([0, 0, 30, 59, self.rev])))
        return out

    def range_batch(self, reqs=None, mode: Optional[str] = None):
        m = mode or self.mode()
        h = self.h("r")
        self.emit("range_batch", reqs=reqs or self.reqs(count=m == "count"), mode=m, h=h)
        if base_of(MODES[m]) == KB_OUT_DEVICE:
            self.held.append(h)

    def stream_open(self, req=None, mode: Optional[str] = None, group: Optional[int] = None) -> str:
        h = self.h("s")
        s, e = self.bounds() if req is None else req[:2]
        rev = self.read_rev() if req is None else req[2]
        self.emit("stream_open", req=(s, e, rev, 0), mode=mode or self.rng.choice(["host", "device", "kvs", "dev_events"]),
                  group=group or self.rng.choice([1, 3, 7, 300]), h=h)
        self.open_streams.append(h)
        return h

    def stream_next(self, h: str, pages: int = 1):
        for _ in range(pages):
            self.emit("stream_next", h=h, budget=self.rng.choice([0, 100, 700, 4096, 1 << 16, ALL]))

    def stream_close(self, h: str):
        self.emit("stream_close", h=h)
        self.open_streams.remove(h)

    def cstream_open(self) -> str:
        h = self.h("c")
        s, e = self.rng.choice([FULL, FULL, self.bounds()])
        self.emit("cstream_open", start=s, end=e, rev=self.rng.choice([59, 30, self.rev]),
                  timeout_rev=self.rng.choice([0, 0, 40]), support_ttl=self.rng.random() < 0.7,
                  group=self.rng.choice([1, 4, 64, 1024]), h=h)
        self.open_cstreams.append(h)
        self.uncompact()
        return h

    def uncompact(self):
        """a sweep records its revision as the compact revision: most of the time the program clears it again, so that
        reads at old revisions keep answering"""
        if self.rng.random() < 0.85:
            self.emit("set_compact_revision", rev=None)

    def cstream_next(self, h: str, pages: int = 1):
        for _ in range(pages):
            self.emit("cstream_next", h=h, budget=self.rng.choice([0, 256, 4096, 1 << 20]))

    def cstream_close(self, h: str):
        self.emit("cstream_close", h=h)
        self.open_cstreams.remove(h)

    def partitions(self):
        s, e = self.rng.choice([FULL, FULL, self.bounds()])
        self.emit("partitions", start=s, end=e, rev=self.read_rev(),
                  part_bytes=self.rng.choice([1, 777, 4096, 1 << 16, 1 << 20]), max_parts=self.rng.choice([1, 3, 64, 4096]))

    def compact_sweep(self, rev: Optional[int] = None):
        s, e = self.rng.choice([FULL, self.bounds()])
        h = self.h("x")
        mode = self.rng.choice(["host", "device", "count"])
        self.emit("compact_sweep", start=s, end=e, rev=rev if rev is not None else self.rng.choice([59, 30, self.rev]),
                  timeout_rev=self.rng.choice([0, 40]), support_ttl=self.rng.random() < 0.7, mode=mode, h=h)
        if mode == "device":
            self.held.append(h)
        if rev is None:
            self.uncompact()

    def watch_add(self):
        h = self.h("w")
        ev = fuzz.fuzz_events(self.rng.randrange(20))
        p = fuzz.fuzz_watchers(ev, self.rng.randrange(100), n=1).prefixes[0]
        self.emit("watch_add", prefix=p, min_rev=self.rng.choice([0, 0, 20, 60]), h=h)
        self.watchers.append(h)

    def watch_del(self):
        if self.watchers:
            h = self.rng.choice(self.watchers)
            self.watchers.remove(h)
            self.emit("watch_del", h=h)

    def match(self, dev: Optional[bool] = None):
        seed = self.rng.randrange(20)
        h = self.h("m")
        if dev is None:
            dev = self.rng.random() < 0.3
        if dev:
            eh = self.h("e")
            self.emit("events_upload", burst=seed, h=eh)
            self.emit("match_dev", ev=eh, h=h)
            self.emit("events_free", ev=eh)
            self.held.append(h)
        else:
            mode = self.rng.choice(["host", "device"])
            self.emit("match", burst=seed, mode=mode, h=h)
            if mode == "device":
                self.held.append(h)

    def read_held(self, k: int = 1):
        for _ in range(min(k, len(self.held))):
            self.emit("read", h=self.held.pop(self.rng.randrange(len(self.held))))

    def random_op(self):
        r = self.rng.random()
        if r < 0.16:
            self.range_batch()
        elif r < 0.28:
            self.submit()
        elif r < 0.36:
            self.collect_some(1)
        elif r < 0.42:
            g = self.gets()
            self.emit("get_batch", reqs=g, mode=self.rng.choice(["host", "device"]))  # kb_get_batch has no wire mode
        elif r < 0.48:
            rq = self.reqs()
            self.emit("range_prefetch", reqs=rq)
            if self.rng.random() < 0.7:
                self.range_batch(rq, self.rng.choice(["host", "kvs"]))
        elif r < 0.56:
            self.write()
        elif r < 0.6:
            self.partitions()
        elif r < 0.64:
            self.compact_sweep()
        elif r < 0.68:
            self.watch_add() if self.rng.random() < 0.6 else self.watch_del()
        elif r < 0.73:
            self.match()
        elif r < 0.78 and self.open_streams:
            self.stream_next(self.rng.choice(self.open_streams))
        elif r < 0.81 and self.open_cstreams:
            self.cstream_next(self.rng.choice(self.open_cstreams))
        elif r < 0.86:
            self.emit("store_info")
        elif r < 0.9:
            self.read_held()
        elif r < 0.93:
            self.expire()
        elif r < 0.95:
            self.invalid_write()
        else:
            self.emit("set_compact_revision", rev=None)

    # -- episodes: each one builds one hazard on purpose
    def ep_lane_busy(self, what: str):
        for _ in range(self.n_lanes):  # every lane holds a batch: the current lane is busy again
            self.submit()
        if what == "stream":
            h = self.stream_open()
            self.stream_next(h, 2)
        elif what == "partitions":
            self.partitions()
        else:
            self.match(dev=False)
        self.collect_some()

    def ep_collect_after(self, kind: str):
        a = self.submit("range", self.rng.choice(["host", "device", "kvs"]))
        b = self.submit()
        self.change(kind)
        self.pendings.remove(a)
        self.pendings.append(a)
        self.collect_some()

    def ep_prefetch(self):
        r1, r2 = self.reqs(2), self.reqs(1)
        self.emit("range_prefetch", reqs=r1)
        self.emit("range_prefetch", reqs=r2)
        self.write(n=25)
        self.range_batch(r1, "host")
        self.range_batch(r2, "kvs")
        r3 = self.reqs(1)
        self.emit("range_prefetch", reqs=r3)
        self.range_batch(r3, "host")  # the hit

    def ep_stream(self, kind: str):
        s1 = self.stream_open((*FULL, ALL), group=self.rng.choice([3, 7, 300]))
        s2 = self.stream_open()
        c = self.cstream_open()
        self.stream_next(s1, self.rng.randint(1, 3))
        self.stream_next(s2)
        self.change(kind)
        for _ in range(self.rng.randint(2, 5)):
            self.stream_next(s1)
            if self.rng.random() < 0.5:
                self.stream_next(s2)
        for h in (s1, s2):
            if self.rng.random() < 0.6:
                self.stream_close(h)
        if c in self.open_cstreams and self.rng.random() < 0.7:
            self.cstream_close(c)

    def ep_long_key(self):
        """a range stream whose first page ends at a 65 535-byte key, then a write behind it: the re-scan starts at
        key_after of that key, which at the limit drops the trailing 0xff (revision 255) and increments"""
        longm = LONG_UK[:-1] + b"M"  # 65 535 bytes too, and behind every key of LONG_UK
        self.apply_emit([(ik(LONG_UK, 0), be(255)), (ik(LONG_UK, 255), b"long value 255")])
        h = self.stream_open((MAGIC + b"/long/", MAGIC + b"/long0", ALL), mode="host", group=1)
        self.emit("stream_next", h=h, budget=0)
        self.apply_emit([(ik(LONG_UK, 256), b"right behind the long key"), (ik(LONG_UK, 0), be(256)),
                         (ik(longm, 0), be(9)), (ik(longm, 9), b"after it")])
        self.stream_next(h, 3)
        self.stream_close(h)

    def apply_emit(self, ops):
        self.apply_local(ops)
        self.emit("apply", ops=ops)

    def ep_cstream(self, kind: str):
        """a compaction stream open across a write that meets the layout-compaction trigger (the stream defers it),
        then invalidated by `kind`"""
        if kind == "restore" and self.dumped is None:
            self.dump()  # so that the restore, not a dump in front of it, is what invalidates the stream
        c = self.cstream_open()
        self.cstream_next(c)
        self.big_replace()
        self.emit("store_info")
        self.cstream_next(c, 2)
        {"load": self.load, "restore": self.restore, "dump": self.dump}[kind]()
        self.cstream_next(c)
        self.cstream_close(c)
        self.write(n=4)  # the load, restore or dump rewrote the heap: this write starts from a compact layout
        self.emit("store_info")

    def ep_deferred_after_close(self):
        """the deferred layout compaction runs at the first write after the last compaction stream closed"""
        for h in list(self.open_cstreams):
            self.cstream_close(h)
        c = self.cstream_open()
        self.cstream_next(c)
        self.big_replace()
        self.emit("store_info")
        self.cstream_next(c)
        self.cstream_close(c)
        self.emit("store_info")
        self.write(n=4)
        self.emit("store_info")

    def ep_partitions_in_flight(self):
        s = self.stream_open()
        for _ in range(max(1, self.n_lanes - 1)):
            self.submit()
        self.partitions()
        self.stream_next(s)
        self.collect_some()

    def ep_ecompacted(self):
        c = self.rng.choice([40, 59, self.rev])
        self.emit("set_compact_revision", rev=c)
        for rev in (c - 1, c):
            s, e = self.bounds()
            self.range_batch([(s, e, rev, 0)], self.rng.choice(["host", "count"]))
            self.range_batch([(s, e, rev, 3)], "host")
        self.submit("range", "host")
        self.emit("stream_open", req=(*FULL, c - 1, 0), mode="host", group=7, h=self.h("s"))
        s = self.stream_open((*FULL, c), mode="kvs")
        self.emit("partitions", start=FULL[0], end=FULL[1], rev=c - 1, part_bytes=4096, max_parts=8)
        self.stream_next(s)
        self.compact_sweep(rev=c + 1)  # a sweep records its revision as the compact revision
        self.range_batch([(*FULL, c, 0)], "host")
        self.emit("set_compact_revision", rev=None)

    def ep_churn(self):
        self.submit()
        self.submit()
        self.watch_add()
        self.watch_del()
        self.watch_add()
        self.match()
        self.collect_some()

    def ep_device_across_compaction(self):
        self.range_batch(self.reqs(2), "device")
        h = self.submit("range", "dev_kvs")
        self.big_delete()
        self.collect_some()
        self.read_held(len(self.held))


def gen_program(seed: int, n_lanes: int) -> Program:
    """a deterministic program on one context; odd seeds leave a pending uncollected (the runner frees it), and a range
    stream and a compaction stream open for kb_close to free"""
    g = _Gen(seed, n_lanes)
    start = sorted(g.items.items())
    for _ in range(6):
        g.watch_add()
    eps = [lambda w=w: g.ep_lane_busy(w) for w in ("stream", "partitions", "match")]
    eps += [lambda k=k: g.ep_collect_after(k) for k in SNAPSHOT_CHANGES]
    eps += [g.ep_prefetch, g.ep_long_key, g.ep_partitions_in_flight, g.ep_ecompacted, g.ep_churn,
            g.ep_device_across_compaction]
    eps += [lambda k=k: g.ep_stream(k) for k in SNAPSHOT_CHANGES]
    eps += [lambda k=k: g.ep_cstream(k) for k in ("load", "restore", "dump")] + [g.ep_deferred_after_close]
    g.rng.shuffle(eps)
    for ep in eps:
        ep()
        if g.rng.random() < 0.3:
            g.random_op()
    while len(g.ops) < 150:
        g.random_op()
    # the end: every held device answer is read back; what is still open is closed or collected, except on odd seeds,
    # which leave one of each open
    if seed % 2:
        g.submit("range", "device")
        g.stream_open()
        g.cstream_open()
        g.pendings.pop()
        g.open_streams.pop()
        g.open_cstreams.pop()
    g.collect_some()
    for h in list(g.open_streams):
        g.stream_next(h)
        g.stream_close(h)
    for h in list(g.open_cstreams):
        g.cstream_close(h)
    g.read_held(len(g.held))
    g.emit("store_info")
    return Program(seed, n_lanes, start, g.ops)


# ---- the model --------------------------------------------------------------------------------------------------------
class Snap:
    """one snapshot as the oracle sees it"""

    def __init__(self, items: Dict[bytes, bytes]):
        self.store = PackedStore.from_items(sorted(items.items()))
        self.st = ko.OracleStore(self.store)


def _digest(b: bytes) -> str:
    return hashlib.sha256(b).hexdigest()[:16]


def err(code: int):
    return ("err", code)


OK = ("ok",)
NONE = ("none",)  # the op names a handle whose open or submit failed: nothing is called


class Model:
    """the expected transcript of a program.  `variant` names a rule replaced by a plausible wrong one (VARIANTS)."""

    def __init__(self, variant: Optional[str] = None):
        assert variant is None or variant in VARIANTS
        self.variant = variant

    # -- state
    def _reset(self, p: Program):
        self.n_lanes = p.n_lanes
        self.heap = ws.HeapModel(p.start)
        self.snap_cache: Optional[Snap] = None
        self.gen = 0
        self.out_of_order = False
        self.layout_compactions = 0
        self.deferred = False  # a layout compaction waits for the last compaction stream to close
        self.compact: Optional[int] = None
        self.cur = 0
        self.lane: List[Optional[str]] = [None] * p.n_lanes
        self.pend: Dict[str, dict] = {}
        self.prefetch: List[Optional[dict]] = [None, None]
        self.prefetch_next = 0
        self.streams: Dict[str, dict] = {}
        self.cstreams: Dict[str, dict] = {}
        self.held: Dict[str, dict] = {}
        self.watch: List[list] = []  # [prefix, min_rev, live] per id
        self.free_ids: List[int] = []
        self.wid: Dict[str, int] = {}
        self.events: Dict[str, int] = {}
        self.dump_state: Optional[Tuple[list, Optional[int]]] = None
        self.last_ecompacted_lane: Optional[int] = None
        self.classes: Set[str] = set()

    def snap(self) -> Snap:
        if self.snap_cache is None:
            self.snap_cache = Snap(self.heap.items)
        return self.snap_cache

    def _changed(self):
        self.gen += 1
        self.snap_cache = None

    def _event(self, kind: str):
        """a snapshot change (or a dump): pendings in flight remember it, for the collected_after classes"""
        for P in self.pend.values():
            P["after"].add(kind)

    def _harvest_all(self):
        """ctx_quiesce (kb_core.cu): reads back the rows of every lane"""
        self.lane = [None] * self.n_lanes

    def _take_lane(self, what: Optional[str] = None):
        """lane_take (kb_batch.cu): the current lane's batch in flight is read back before its staging is reused"""
        if self.lane[self.cur] is not None and what:
            self.classes.add("lane_busy:" + what)
        self.lane[self.cur] = None

    def _pinned(self) -> bool:
        return any(not c["invalid"] for c in self.cstreams.values())

    def _compact_fails(self, rev: int) -> bool:
        """R7. compact_race_check (kb_batch.cu): a read below the compact revision fails -- `compact_rev > rev` -- with
        KB_ECOMPACTED and changes no other state (header: kb_range_stream_open "checkCompactRace happens here")"""
        if self.compact is None:
            return False
        return self.compact >= rev if self.variant == "R7" else self.compact > rev

    # -- answers
    def range_answer(self, reqs, mode: int, snap: Snap) -> dict:
        """the oracle's answer of a range batch on `snap` in `mode` (host-visible fields, and what the arena holds)"""
        if base_of(mode) == KB_OUT_COUNT:
            return {"count": [ko.scan(snap.st, [s, e], rev, collect=False).count for s, e, rev, _ in reqs]}
        xs = [ko.range_(snap.st, *q) for q in reqs]
        emit = np.concatenate([x.emit for x in xs]).astype(np.uint64) if xs else np.zeros(0, np.uint64)
        first = np.cumsum([0] + [len(x.emit) for x in xs]).tolist()
        kvs = [kv for x in xs for kv in x.kvs(snap.store)]
        w = wire_of(mode)
        if w:
            arena, off = ko.wire_encode(snap.st, emit, ko.WIRE_KVS if w == KB_WIRE_ETCD_KVS else ko.WIRE_EVENTS)
            eo = off.tolist() if len(emit) else None
        else:
            arena = b"".join(pad16(snap.store.keys[int(i)]) + pad16(snap.store.vals[int(i)]) for i in emit)
            eo = None
        host = {"first": first, "count": [x.count for x in xs], "examined": [x.examined for x in xs],
                "n_kvs": len(emit), "n_bytes": len(arena)}
        body = {"rec": emit.tolist(), "kvs": kvs, "arena": _digest(arena), "elem_off": eo}
        if base_of(mode) == KB_OUT_DEVICE:
            return {**host, "held": body}
        return {**host, **body}

    def get_answer(self, reqs, mode: int, snap: Snap) -> dict:
        st = []
        mod, rec, vals, elems = [], [], [], []
        for k, rev in reqs:
            idx, m = ko.get(snap.st, k, rev)
            st.append(0 if idx >= 0 else (2 if idx == -2 else 1))
            mod.append(m if idx >= 0 or idx == -2 else 0)
            rec.append(idx if idx >= 0 else None)
            vals.append(snap.store.vals[idx] if idx >= 0 else None)
            elems.append(ko.wire_encode(snap.st, [idx], ko.WIRE_KVS)[0] if idx >= 0 else b"")
        out = {"status": st, "mod_rev": mod, "rec": rec}
        if wire_of(mode):
            out["elems"] = elems
        else:
            out["arena"] = _digest(b"".join(pad16(v) for v in vals if v is not None))
            out["values"] = vals
        return out

    def batch_snapshot(self, P: dict) -> Snap:
        """R1. kb_range_submit / kb_get_submit: the batch answers the snapshot it was submitted on; "any other entry
        point may be called in between (it first reads back the rows of what is in flight)" (header, kb_range_submit)"""
        return self.snap() if self.variant == "R1" else P["snap"]

    def device_body(self, H: dict) -> dict:
        """R2. KB_OUT_DEVICE: the answer stays in HBM in the result's own arena and per-kv arrays until kb_result_free,
        so it reads back unchanged after later writes, layout compactions and slab growth (header, KB_OUT_DEVICE)"""
        if self.variant == "R2" and H.get("reqs") is not None:
            return self.range_answer(H["reqs"], H["mode"], self.snap())["held"]
        return H["body"]

    def prefetched_snapshot(self, reqs) -> Snap:
        """R3. kb_range_prefetch: "identical bounds, same snapshot; anything else is ignored" -- a prefetched search
        counts only when its store_gen is the current one (kb_search.cu range_bounds_find), so a prefetch changes no
        answer.  The slot it hits is consumed."""
        ident = [(s, e) for s, e, _, _ in reqs]
        hit = None
        for sl in self.prefetch:
            if sl and sl["ident"] == ident and (sl["gen"] == self.gen or self.variant == "R3"):
                if hit is None or sl["seq"] < hit["seq"]:
                    hit = sl
        if hit is None:
            return self.snap()
        self.prefetch[self.prefetch.index(hit)] = None
        return hit["snap"] if self.variant == "R3" else self.snap()

    def stream_from(self, S: dict) -> Optional[bytes]:
        """R4. kb_range_stream_next after a snapshot change re-scans "[internal key of the last kv handed out + 0x00,
        end), at the same read revision" (header); at the 65 535-byte limit key_after increments instead (kb_page.cu)"""
        if not S["started"] or self.variant == "R4_start":
            return S["req"][0]
        if self.variant == "R4_nozero":
            return S["last_key"]
        if self.variant == "R4_limit_done" and len(S["last_key"]) == MAX_KEY:
            return None
        return key_after(S["last_key"])

    def stream_scan(self, S: dict, start: bytes):
        s, e, rev, _ = S["req"]
        snap = self.snap()
        emit, image, sizes = stream_expected(snap.store, snap.st, start, e, rev, S["mode"])
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        S["rest"] = [(int(emit[i]), image[off[i]: off[i + 1]], snap.store.keys[int(emit[i])]) for i in range(len(emit))]
        S["gen"] = self.gen

    def cstream_victims(self, C: dict) -> List[tuple]:
        """R5. kb_compact_stream_open: kb_compact_sweep's victims of the snapshot the stream was opened on, each with
        its internal key and, for classes 3 / 4, the value the sweep read; later writes keep them valid (header)"""
        if self.variant == "R5" and C["gen"] != self.gen:
            return self.sweep(C["args"], self.snap())[0]
        return C["victims"]

    def sweep(self, a: dict, snap: Snap):
        """kb_compact_sweep: ko.scan(compact=True)'s delete calls as (record, class, internal key, guard), and its run"""
        x = ko.scan(snap.st, [a["start"], a["end"]], a["rev"], compact=True, collect=False,
                    timeout_rev=a["timeout_rev"], support_ttl=a["support_ttl"])
        out = []
        for i, c in zip(x.victims.tolist(), x.vclass.tolist()):
            out.append((i, c, snap.store.keys[i], snap.store.vals[i] if c in (3, 4) else b""))
        return out, x

    def partition_fails(self, rev: int) -> bool:
        """R6. kb_range_partitions: "There is no checkCompactRace" (header); the cut follows the definition on the
        current snapshot (partition_shapes.partitions)"""
        return self.variant == "R6" and self._compact_fails(rev)

    def match_answer(self, burst: int) -> dict:
        """R8. kb_watch_match: deliveries of watcher id w = [start[w], start[w+1]) over every id handed out so far
        (cancelled ones empty), each list as ko.fanout gives it for the live watchers"""
        ev = fuzz.fuzz_events(burst)
        live = [i for i, w in enumerate(self.watch) if w[2]]
        W = len(self.watch)
        lists = {i: [] for i in range(W)}
        if live and ev.n:
            pw = PackedWatchers(Slab.from_list([self.watch[i][0] for i in live]),
                                np.array([self.watch[i][1] for i in live], np.uint64))
            start, idx, _ = ko.fanout(ev, pw)
            for j, i in enumerate(live):
                lists[i] = idx[int(start[j]): int(start[j + 1])].tolist()
        starts = [0]
        for i in range(W):
            starts.append(starts[-1] + len(lists[i]))
        return {"n_watchers": W, "start": starts, "idx": [x for i in range(W) for x in lists[i]]}

    def write_batch(self, ops) -> tuple:
        """R9. kb_apply_batch refuses a batch with a key over 65 535 bytes (KB_ELIMIT) before anything changes"""
        if any(len(op[0]) > MAX_KEY for op in ops):
            return err(KB_ELIMIT)
        pinned = self._pinned()
        self.heap.pinned = pinned
        f = self.heap.apply(ops)
        if f["n_ins"] + f["n_del"] + f["n_rep"]:
            self._changed()
            self.out_of_order = True
            if f["fired"]:
                self.out_of_order = False
                self.layout_compactions += 1
                if self.deferred:
                    self.classes.add("deferred_compaction_after_last_close")
                self.deferred = False
            if pinned and (f["displaced"] > f["threshold"] or f["garbage_k"] * ws.GARBAGE_DIV > f["ktail"] or
                           f["garbage_v"] * ws.GARBAGE_DIV > f["vtail"]):
                self.deferred = True  # the trigger holds, but an open compaction stream keeps the heap in place
                for C in self.cstreams.values():
                    C["deferred"] = C["deferred"] or not C["invalid"]
        return OK

    # -- the run
    def run(self, p: Program) -> List[tuple]:
        self._reset(p)
        return [self.step(kind, a) for kind, a in p.ops]

    def step(self, kind: str, a: dict):
        return getattr(self, "op_" + kind)(a)

    def _submit_checks(self, reqs) -> Optional[tuple]:
        self._take_lane()
        for _, _, rev, _ in reqs:
            if self._compact_fails(rev):
                self.last_ecompacted_lane = self.cur
                return err(KB_ECOMPACTED)
        if self.last_ecompacted_lane == self.cur:
            self.classes.add("ecompacted_then_batch_same_lane")
        self.last_ecompacted_lane = None
        return None

    def op_range_batch(self, a):
        mode = MODES[a["mode"]]
        e = self._submit_checks(a["reqs"])
        if e:
            return e
        snap = self.prefetched_snapshot(a["reqs"])
        ans = self.range_answer(a["reqs"], mode, snap)
        if "held" in ans:
            self.held[a["h"]] = {"body": ans.pop("held"), "reqs": a["reqs"], "mode": mode, "compactions": self.layout_compactions}
        return ans

    def op_range_submit(self, a):
        e = self._submit_checks(a["reqs"])
        if e:
            return e
        snap = self.prefetched_snapshot(a["reqs"])
        self._new_pending(a, "range", snap)
        return OK

    def _new_pending(self, a, kind, snap):
        self.pend[a["h"]] = {"kind": kind, "reqs": a["reqs"], "mode": a["mode"], "snap": snap, "after": set(),
                             "lane": self.cur}
        self.lane[self.cur] = a["h"]
        self.cur = (self.cur + 1) % self.n_lanes

    def op_get_submit(self, a):
        self._take_lane()
        self._new_pending(a, "get", self.snap())
        return OK

    def op_get_batch(self, a):
        self._take_lane()
        return self.get_answer(a["reqs"], GET_MODES[a["mode"]], self.snap())

    def op_collect(self, a):
        P = self.pend.pop(a["h"], None)
        if P is None:
            return NONE
        if self.lane[P["lane"]] == a["h"]:
            self.lane[P["lane"]] = None
        for k in P["after"]:
            self.classes.add("collected_after:" + k)
        snap = self.batch_snapshot(P)
        if P["kind"] == "get":
            return self.get_answer(P["reqs"], GET_MODES[P["mode"]], snap)
        mode = MODES[P["mode"]]
        ans = self.range_answer(P["reqs"], mode, snap)
        if "held" in ans:
            self.held[a["h"]] = {"body": ans.pop("held"), "reqs": P["reqs"], "mode": mode, "compactions": self.layout_compactions}
        return ans

    def op_pending_close(self, a):
        P = self.pend.pop(a["h"], None)
        if P is not None and self.lane[P["lane"]] == a["h"]:
            self.lane[P["lane"]] = None
        return OK if P is not None else NONE

    def op_range_prefetch(self, a):
        slot = self.prefetch_next & 1
        self.prefetch_next += 1
        self.prefetch[slot] = {"ident": [(s, e) for s, e, _, _ in a["reqs"]], "gen": self.gen, "seq": self.prefetch_next,
                               "snap": self.snap()}
        return OK

    def op_read(self, a):
        H = self.held.pop(a["h"], None)
        if H is None:
            return NONE
        if self.layout_compactions > H["compactions"] and H.get("reqs") is not None:
            self.classes.add("device_answer_across_layout_compaction")
        return self.device_body(H)

    def op_stream_open(self, a):
        s, e, rev, _ = a["req"]
        if self._compact_fails(rev):
            return err(KB_ECOMPACTED)
        self._take_lane("stream")
        S = {"req": a["req"], "mode": MODES[a["mode"]], "group": a["group"], "started": False, "last_key": None,
             "done": False}
        self.stream_scan(S, s)
        self.streams[a["h"]] = S
        return OK

    def op_stream_next(self, a):
        S = self.streams.get(a["h"])
        if S is None:
            return NONE
        if S["done"]:
            return None
        if S["gen"] != self.gen:
            if len(self.streams) > 1 and self._pinned():
                self.classes.add("stream_rescan_beside_streams")
            for k in S.get("changes", ()):
                self.classes.add("stream_rescan:" + k)
            if S["started"] and len(S["last_key"]) == MAX_KEY:
                self.classes.add("stream_rescan_at_key_limit")
            start = self.stream_from(S)
            if start is None:
                S["done"] = True
                return None
            self._take_lane("stream")
            self.stream_scan(S, start)
        S["changes"] = set()
        if not S["rest"]:
            S["done"] = True
            return None
        sizes = np.array([len(img) for _, img, _ in S["rest"]], np.int64)
        _, b = greedy_cuts(sizes, S["group"], a["budget"])[0]
        page, S["rest"] = S["rest"][:b], S["rest"][b:]
        S["started"] = True
        S["last_key"] = page[-1][2]
        arena = b"".join(img for _, img, _ in page)
        w = wire_of(S["mode"])
        eo = np.concatenate([[0], np.cumsum([len(img) for _, img, _ in page])]).tolist() if w else None
        return {"first": [0, b], "count": [b], "examined": [0], "rec": [r for r, _, _ in page], "arena": _digest(arena),
                "n_bytes": len(arena), "elem_off": eo}

    def op_stream_close(self, a):
        return OK if self.streams.pop(a["h"], None) is not None else NONE

    def op_partitions(self, a):
        if self.partition_fails(a["rev"]):
            return err(KB_ECOMPACTED)
        if self.pend and any(P["lane"] != self.cur and self.lane[P["lane"]] is not None for P in self.pend.values()) \
                and self.streams:
            self.classes.add("partitions_beside_other_lanes_and_streams")
        self._take_lane("partitions")
        snap = self.snap()
        borders, kv_first, arena_first = ps.partitions(snap.store, snap.st, a["start"], a["end"], a["rev"],
                                                       a["part_bytes"], a["max_parts"])
        return {"borders": borders, "kv_first": kv_first, "arena_first": arena_first}

    def op_compact_sweep(self, a):
        self._harvest_all()
        vic, x = self.sweep(a, self.snap())
        self.compact = a["rev"]  # scan(compact=true) stores the compact revision (kb_compact.cu sweep_locked)
        out = {"n_victims": len(vic), "count": x.count, "examined": x.examined}
        body = {"rec": [v[0] for v in vic], "cls": [v[1] for v in vic]}
        if a["mode"] == "host":
            return {**out, **body}
        if a["mode"] == "device":
            self.held[a["h"]] = {"body": body, "compactions": self.layout_compactions}
        return out

    def op_cstream_open(self, a):
        self._harvest_all()
        vic, x = self.sweep(a, self.snap())
        self.compact = a["rev"]
        self.cstreams[a["h"]] = {"victims": vic, "pos": 0, "group": a["group"], "invalid": None, "gen": self.gen,
                                 "args": a, "deferred": False}
        return {"n_victims": len(vic), "count": x.count, "examined": x.examined}

    def op_cstream_next(self, a):
        C = self.cstreams.get(a["h"])
        if C is None:
            return NONE
        if C["invalid"]:
            if C["deferred"]:
                self.classes.add("cstream_deferred_then_invalidated:" + C["invalid"])
            return err(KB_ESTATE)
        vic = self.cstream_victims(C)
        if C["pos"] >= len(vic):
            return None
        sizes = np.array([len(pad16(k)) + len(pad16(g)) for _, _, k, g in vic[C["pos"]:]], np.int64)
        _, b = greedy_cuts(sizes, C["group"], a["budget"])[0]
        page = vic[C["pos"]: C["pos"] + b]
        out = {"first": C["pos"], "n": b, "rec": [v[0] for v in page], "cls": [v[1] for v in page],
               "keys": [v[2] for v in page], "guards": [v[3] for v in page]}
        C["pos"] += b
        return out

    def op_cstream_close(self, a):
        return OK if self.cstreams.pop(a["h"], None) is not None else NONE

    def _snapshot_event(self, kind: str):
        self._event(kind)
        for S in self.streams.values():
            S.setdefault("changes", set()).add(kind)

    def op_apply(self, a):
        self._harvest_all()
        both = sum(1 for sl in self.prefetch if sl and sl["gen"] == self.gen) == 2
        gen = self.gen
        r = self.write_batch(a["ops"])
        if self.gen != gen:
            self._snapshot_event("write")
            if both:
                self.classes.add("prefetch_both_valid_across_write")
        return r

    def op_expire(self, a):
        gen = self.gen
        due = [k for t, _, k in self.heap.ttl_queue if t <= a["now"] and self.heap.ttl_of.get(k) == t]
        if due:
            self._harvest_all()
        self.heap.pinned = self._pinned()
        n, f = self.heap.expire(a["now"])
        ff = f["facts"]
        if ff and ff["n_ins"] + ff["n_del"] + ff["n_rep"]:
            self._changed()
            self.out_of_order = not ff["fired"]
            if ff["fired"]:
                self.layout_compactions += 1
                self.deferred = False
        if self.gen != gen:
            self._snapshot_event("expire")
        return ("dropped", n)

    def _install(self, items, kind: str):
        self._harvest_all()
        for C in self.cstreams.values():
            C["invalid"] = kind
        self.heap.install(items)
        self._changed()
        self.out_of_order = self.deferred = False
        self._snapshot_event(kind)

    def op_load(self, a):
        self._install(a["items"], "load")
        return OK

    def op_dump(self, a):
        self._harvest_all()
        for C in self.cstreams.values():
            C["invalid"] = "dump"
        if self.out_of_order:
            self._changed()
            self.layout_compactions += 1
            self._snapshot_event("dump")
        self.out_of_order = self.deferred = False
        self.heap.pinned = False
        self.heap.compact_layout()
        items = self.heap.sorted_items()
        self.dump_state = (items, self.compact)
        return dump_entry(ws.dump_image(items, self.compact, self.heap.max_kv))

    def op_restore(self, a):
        items, c = self.dump_state
        self._install(items, "restore")
        self.compact = c
        return OK

    def op_set_compact_revision(self, a):
        self.compact = a["rev"]
        return OK

    def op_store_info(self, a):
        return ("info",) + self.heap.info()

    def op_watch_add(self, a):
        if self.pend:
            self.classes.add("watcher_churn_in_flight")
        w = [a["prefix"], a["min_rev"], True]
        if self.free_ids:
            i = self.free_ids.pop()
            self.watch[i] = w
        else:
            self.watch.append(w)
            i = len(self.watch) - 1
        self.wid[a["h"]] = i
        return ("id", i)

    def op_watch_del(self, a):
        i = self.wid.pop(a["h"])
        if self.pend:
            self.classes.add("watcher_churn_in_flight")
        self.watch[i][2] = False
        self.free_ids.append(i)
        return OK

    def op_match(self, a):
        self._take_lane("match")
        m = self.match_answer(a["burst"])
        if a["mode"] == "device":
            self.held[a["h"]] = {"body": {"idx": m.pop("idx")}, "compactions": self.layout_compactions}
        return m

    def op_events_upload(self, a):
        self._take_lane("match")
        self.events[a["h"]] = a["burst"]
        return OK

    def op_match_dev(self, a):
        m = self.match_answer(self.events[a["ev"]])
        self.held[a["h"]] = {"body": {"idx": m.pop("idx")}, "compactions": self.layout_compactions}
        return m

    def op_events_free(self, a):
        self.events.pop(a["ev"], None)
        return OK


def dump_entry(blob: bytes) -> tuple:
    """a dump file as a transcript entry: its header fields and a digest of the whole file"""
    h = dict(zip(ws.HEADER_FIELDS, ws.DUMP_HEADER.unpack_from(blob, 0)))
    return ("dump", tuple(sorted((k, v) for k, v in h.items() if k != "magic")), _digest(blob))


def run_program(p: Program, variant: Optional[str] = None) -> Tuple[List[tuple], Set[str]]:
    m = Model(variant)
    t = m.run(p)
    return t, m.classes


# ---- printing ---------------------------------------------------------------------------------------------------------
def short(x, n: int = 96) -> str:
    if isinstance(x, bytes):
        return repr(x if len(x) <= 40 else x[:24] + b"...(%d B)" % len(x))
    if isinstance(x, dict):
        return "{" + ", ".join("%s: %s" % (k, short(v, 48)) for k, v in x.items()) + "}"
    if isinstance(x, (list, tuple)):
        if x and isinstance(x[0], tuple) and len(x[0]) == 2 and isinstance(x[0][0], bytes) and len(x) > 6:
            return "[%d items]" % len(x)
        s = ", ".join(short(v, 32) for v in list(x)[:8]) + (", ...(%d)" % len(x) if len(x) > 8 else "")
        return ("(%s)" if isinstance(x, tuple) else "[%s]") % s
    s = repr(x)
    return s if len(s) <= n else s[:n] + "..."


def describe(op: Tuple[str, dict]) -> str:
    kind, a = op
    return "%s %s" % (kind, " ".join("%s=%s" % (k, short(v, 60)) for k, v in a.items()))


def main(argv=None):
    ap = argparse.ArgumentParser(description="print a program and its expected transcript")
    ap.add_argument("--seed", type=int, required=True)
    ap.add_argument("--lanes", type=int, required=True)
    ap.add_argument("--variant", default=None, choices=VARIANTS)
    args = ap.parse_args(argv)
    p = gen_program(args.seed, args.lanes)
    t, classes = run_program(p, args.variant)
    print("seed %d, KB_LANES %d: %d records, %d ops" % (p.seed, p.n_lanes, len(p.start), len(p.ops)))
    for i, (op, e) in enumerate(zip(p.ops, t)):
        print("%4d  %s\n      -> %s" % (i, describe(op), short(e, 400)))
    print("classes: " + ", ".join(sorted(classes)))


if __name__ == "__main__":
    main()
