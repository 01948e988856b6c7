"""Host-side mirror of the hot-path half of backend.Backend (pkg/backend/backend.go:44-84):
List / Count / ListByStream / Compact (pkg/backend/range.go:124-256, compact.go:31-127) and
Watch with its ring cache (pkg/backend/watch.go:37-159, ring.go:24-118, watcherhub.go:34-100).

The write path (Create/Update/Delete), election and retry stay in the reference's Go code; this mirror only
consumes their OUTPUT formats (records, events).  Error behaviour follows the reference: the same conditions
raise, with the reference's message text.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Iterator, List, Optional, Sequence, Tuple

import numpy as np

from ._lib import Engine
from .coder import NormalCoder, prefix_end
from .packed import PackedEvents, Slab
from .scanner import COMPACT_GROUP, COMPACT_PAGE_BYTES, KeyValue, Scanner, StreamRangeResponse

HISTORY_CAPACITY = 200000  # backend.go:39
EVENT_BATCH_SIZE = 300  # backend.go:41
RESULT_CHAN_LENGTH = 100  # watch.go:30
EVENT_CREATE, EVENT_PUT, EVENT_DELETE = 0, 1, 2


@dataclass
class RangeResponse:
    revision: int
    kvs: List[KeyValue]
    more: bool = False


@dataclass
class Event:  # v2rpc.Event
    type: int
    revision: int
    kv: KeyValue


class Ring:
    """pkg/backend/ring.go:24-118 (host side: the ring only holds references; filtering runs on the GPU)"""

    def __init__(self, l: int):
        self.s = 0
        self.e = 0
        self.l = l
        self.arr: List[Optional[Event]] = [None] * l

    def add(self, event: Event):
        self.arr[self.e % self.l] = event
        if self.e == self.s + self.l:
            self.s += 1
        self.e += 1

    def size(self) -> int:
        return self.l

    def reset(self):
        self.s = self.e = 0

    def find_events(self, revision: int):
        """returns (empty, high, low, newest, oldest, events)"""
        if self.e == 0:
            return True, False, False, None, None, []
        newest, oldest = self.arr[(self.e - 1) % self.l], self.arr[self.s % self.l]
        if revision > newest.revision:
            return False, True, False, newest, oldest, []
        if revision < oldest.revision:
            return False, False, True, newest, oldest, []
        lo, hi = 0, self.e - self.s
        while lo < hi:  # sort.Search
            mid = (lo + hi) // 2
            if self.arr[(self.s + mid) % self.l].revision >= revision:
                hi = mid
            else:
                lo = mid + 1
        return False, False, False, newest, oldest, [self.arr[(self.s + i) % self.l] for i in range(lo, self.e - self.s)]


def _pack_events(events: Sequence[Event], batch: int = EVENT_BATCH_SIZE) -> PackedEvents:
    keys = Slab.from_list([e.kv.key for e in events])
    rev = np.array([e.revision for e in events], dtype=np.uint64)
    n = len(events)
    bo = np.array(list(range(0, n, batch)) + [n], dtype=np.uint64) if n else np.zeros(1, np.uint64)
    return PackedEvents(keys, rev, bo)


class Watch:
    """one Backend.Watch subscription: `out` receives the []*Event messages the reference would send on the channel"""

    def __init__(self, wid: int, prefix: bytes, revision: int):
        self.id = wid
        self.prefix = prefix
        self.revision = revision
        self.out: List[List[Event]] = []


class Backend:
    def __init__(self, engine: Engine, prefix: str = "/registry", skipped_prefixes: Sequence[str] = (),
                 watch_cache_size: int = HISTORY_CAPACITY, enable_etcd_compatibility: bool = True):
        self.engine = engine
        self.coder = NormalCoder()
        self.scanner = Scanner(engine)
        self.prefix = prefix
        self.skipped_prefixes = list(skipped_prefixes)
        self.enable_etcd_compatibility = enable_etcd_compatibility
        self.watch_cache = Ring(watch_cache_size)
        self.watches: dict = {}
        self._revision = 0

    # ---- tso (pkg/backend/tso/tso.go:47-49) ----
    def get_current_revision(self) -> int:
        return self._revision

    def set_current_revision(self, rev: int):
        self._revision = rev

    # ---- write hook ----
    def commit(self, ops: Sequence[Tuple[bytes, Optional[bytes]]]):
        """The hook a storage adaptor calls after BatchWrite.Commit succeeds (pkg/storage/interface.go:62-84; the txn
        builders of pkg/backend/txn.go:36-246 and the compaction deletes of scanner.go:538-564 all go through it):
        (internal_key, value) puts and (internal_key, None) deletes are merged into the HBM snapshot."""
        if ops:
            self.engine.apply_batch(list(ops))

    # ---- read path ----
    def get(self, key: bytes, revision: int = 0):
        """range.go:34-81 Backend.Get: returns (header revision, KeyValue | None).  A missing key, a key created after
        `revision` and a deleted key (tombstone) all answer with a nil kv."""
        cur = self.get_current_revision()
        res = self.engine.get_batch([(key, revision)])
        try:
            st, mod = int(res.status[0]), int(res.mod_rev[0])
            if st != 0:  # storage.ErrKeyNotFound (range.go:49-53)
                return cur, None
            if mod > cur:
                cur = mod
            return cur, KeyValue(key, res.value(0), mod)
        finally:
            res.close()

    def list(self, key: bytes, end: bytes, revision: int = 0, limit: int = 0) -> RangeResponse:
        """range.go:124-174"""
        if len(end) == 0:
            raise ValueError("invalid nil end field in RangeRequest")
        cur = self.get_current_revision()
        req_rev = revision or cur
        if key >= end:
            raise ValueError("invalid range end")
        lim = limit + 1 if limit > 0 else limit  # one more to learn whether there is more
        kvs = self.scanner.range(self.coder.encode_object_key(key, 0), self.coder.encode_object_key(end, 0), req_rev, lim)
        more = False
        if lim > 0 and len(kvs) > limit:
            more, kvs = True, kvs[:limit]
        return RangeResponse(cur, kvs, more)

    def count(self, key: bytes, end: bytes) -> Tuple[int, int]:
        """range.go:177-205: returns (revision, count)"""
        rev = self.get_current_revision()
        if not self.enable_etcd_compatibility:
            return rev, 0
        return rev, self.scanner.count(self.coder.encode_object_key(key, 0), self.coder.encode_object_key(end, 0), rev)

    def list_by_stream(self, start_key: bytes, end_key: bytes, rev: int = 0) -> Iterator[StreamRangeResponse]:
        """range.go:247-256 (start/end are handed to the scanner as they are, like the reference does)"""
        return self.scanner.range_stream(start_key, end_key, rev or self.get_current_revision())

    def get_partitions(self, key: bytes, end: bytes) -> List[bytes]:
        """range.go:208-244: the HBM slab is one partition, like badger (pkg/storage/badger/badger.go:52-54)"""
        return [self.coder.encode_object_key(key, 0), self.coder.encode_object_key(end, 0)]

    # ---- compaction driver ----
    def get_compact_borders(self) -> List[bytes]:
        """compact.go:107-127"""
        borders = []
        for key in [self.prefix] + self.skipped_prefixes:
            if not key.endswith("/"):
                key += "/"
            kb = key.encode()
            borders.append(self.coder.encode_object_key(kb, 0))
            borders.append(self.coder.encode_object_key(prefix_end(kb), 0))
        return sorted(borders)

    def compact(self, revision: int, timeout_revision: int = 0, support_ttl: bool = True):
        """compact.go:31-68: clamp, then one scanner.Compact per border pair; returns the victim lists"""
        cur = self.get_current_revision()
        if revision == 0 or revision > cur:
            revision = cur
        borders = self.get_compact_borders()
        out = []
        for i in range(0, len(borders), 2):
            out.append(self.scanner.compact(borders[i], borders[i + 1], revision, timeout_revision, support_ttl))
        return revision, out

    def compact_apply(self, revision: int, current: Callable[[bytes], Optional[bytes]],
                      engine_del: Optional[Callable[[List[bytes]], None]] = None, timeout_revision: int = 0,
                      support_ttl: bool = True, page_bytes: int = COMPACT_PAGE_BYTES, group: int = COMPACT_GROUP):
        """compact() with the deletes applied: for every border pair the victims arrive as pages of internal keys
        (Scanner.compact_pages), and every page's deletes are committed through commit() before the next page is asked
        for -- one batch per group of victims, as the storage adaptor does.  Classes 1, 2 and 5 (store.Del) are deleted
        as they are.  Classes 3 and 4 (store.DelCurrent, scanner.go:477-491) are deleted only if the engine still holds
        the value the sweep read: current(internal_key) is the engine's value of a key (None when absent); a different
        value is a failed CAS and the victim is skipped.  engine_del(keys), when given, deletes a group's keys from the
        engine first (engine first, mirror second).  Returns (revision, [(count, examined, deleted, skipped)] per
        border pair)."""
        cur = self.get_current_revision()
        if revision == 0 or revision > cur:
            revision = cur
        borders = self.get_compact_borders()
        out = []
        for i in range(0, len(borders), 2):
            deleted = skipped = 0
            stream = self.engine.compact_stream(borders[i], borders[i + 1], revision, timeout_revision, support_ttl, group)
            try:
                while True:
                    page = stream.next(page_bytes)
                    if page is None:
                        break
                    for g in range(0, page.n, group):
                        ops = []
                        for k in range(g, min(g + group, page.n)):
                            key = page.key(k)
                            if page.victim_class[k] in (3, 4) and current(key) != page.guard(k):
                                skipped += 1
                                continue
                            ops.append((key, None))
                        if engine_del is not None and ops:
                            engine_del([k for k, _ in ops])
                        self.commit(ops)
                        deleted += len(ops)
                out.append((stream.count, stream.examined, deleted, skipped))
            finally:
                stream.close()
        return revision, out

    # ---- watch path ----
    def watch(self, prefix: bytes, revision: int) -> Watch:
        """watch.go:37-99: subscribe, then catch up from the ring cache"""
        ring_ret = None if revision == 0 else self.watch_cache.find_events(revision)
        live_rev = revision
        catchup: List[Event] = []
        if ring_ret is not None:
            empty, high, low, newest, oldest, events = ring_ret
            if empty:
                if not revision > self.get_current_revision():
                    raise RuntimeError(" empty cache event, current revision is %d" % self.get_current_revision())
            elif high:
                pass
            elif low:
                raise RuntimeError("cache event oldest revision is %d newer than requested revision %d"
                                   % (oldest.revision, revision + 1))
            else:
                # filterByPrefix over the cached tail runs on the GPU as a one-watcher match
                catchup = self._filter_by_prefix(events, prefix)
                if catchup:
                    live_rev = newest.revision + 1
        wid = self.engine.watch_add(prefix, live_rev)
        w = Watch(wid, prefix, live_rev)
        self.watches[wid] = w
        if catchup:
            w.out.extend(self._catch_up_chunks(catchup))
        return w

    def cancel(self, w: Watch):
        self.engine.watch_del(w.id)
        self.watches.pop(w.id, None)

    def _filter_by_prefix(self, events: Sequence[Event], prefix: bytes) -> List[Event]:
        wid = self.engine.watch_add(prefix, 0)  # a temporary watcher with min_rev 0
        try:
            res = self.engine.watch_match(_pack_events(events, batch=max(len(events), 1)))
            idx = res.deliveries(wid).tolist()
            res.close()
        finally:
            self.engine.watch_del(wid)
        return [events[i] for i in idx]

    @staticmethod
    def _catch_up_chunks(events: List[Event]) -> List[List[Event]]:
        """watch.go:102-117"""
        batch = EVENT_BATCH_SIZE
        if len(events) > RESULT_CHAN_LENGTH * EVENT_BATCH_SIZE:
            batch = len(events) // (RESULT_CHAN_LENGTH - 1)
        out = []
        while True:
            if len(events) > batch:
                out.append(events[:batch])
                events = events[batch:]
            else:
                out.append(events)
                break
        return out

    def publish(self, events: Sequence[Event]):
        """what collectStorageWriteEvents + WatcherHub.Stream + processEvents do for one revision-ordered run of
        events (backend.go:208-270, watcherhub.go:78-92, watch.go:119-138): cache them, split them into <=300 event
        batches, and hand every watcher its filtered, ordered, non-empty messages"""
        events = list(events)
        for e in events:
            self.watch_cache.add(e)
            self._revision = max(self._revision, e.revision)
        if not events or not self.watches:
            return
        packed = _pack_events(events)
        res = self.engine.watch_match(packed)
        try:
            bo = packed.batch_off.astype(np.int64)
            for wid, w in self.watches.items():
                idx = res.deliveries(wid)
                if idx.size == 0:
                    continue
                b = np.searchsorted(bo, idx, side="right") - 1  # collector batch of every delivery
                cut = np.nonzero(np.diff(b))[0] + 1
                for part in np.split(idx, cut):  # one message per (watcher, batch), only when non-empty
                    w.out.append([events[int(i)] for i in part])
        finally:
            res.close()
