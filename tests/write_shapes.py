"""Write-path sequences built so that the code that changes the snapshot (kubebrain_b200/csrc/kb_store.cu) meets its
fixed boundaries on purpose (shared by the CPU and GPU tests).

A shape is a starting store and a sequence of steps (batches for kb_apply_batch, kb_expire calls, dumps, reloads).
  W1  merge / fix list: inserts at lower bound 0 and N, k inserts on one lower bound, an insert on a deleted record,
      delete runs at both ends, delete + re-put of one key in one batch, a replacement behind an insert, everything
      deleted then inserted again, 200 000 inserts into 1 000 records, every record replaced, N + n_ins around
      k_dir_merge's 256-thread blocks;
  W2  key bytes: op keys of 0 .. 65 535 bytes, near misses of a stored key in chunk 0, 31, 32, 33 and the last (the
      second pass of k_key_exists), prefixes and extensions, neighbours whose LCP is 511 .. 513 and 1 023 .. 1 025 (the
      second and third pass of summarize_record) made by an insert, a delete and a replacement, `/events/` at user-key
      offsets on both sides of a 32-lane pass, at the last offset and running into the `$` suffix;
  W3  heap: the layout-compaction trigger at its threshold and one past it (both branches of max(4096, N / 32)), garbage
      at a quarter of each tail and one chunk past it, slab growth, replacements of empty values;
  W4  TTL: many keys due in one second, expire(t) at exactly t, stale queue entries, TTL ops in one batch, an expiry
      that empties the store, TTLs dropped by kb_load_sorted and kb_restore.
`HeapModel` restates kb_apply_batch's heap accounting and predicts kb_store_info after every step; `dump_image` /
`parse_dump` restate the KBB200D1 file.  `write_classes` derives what a batch reaches from the bytes and the model alone
(never from the builders' bookkeeping), so that tests/test_write_shapes.py can assert it on any host;
`python -m tests.write_shapes` prints it."""
from __future__ import annotations

import bisect
import struct
from collections import Counter
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

MAGIC = b"\x57\xfb\x80\x8b"
EVENTS = b"/events/"

# restated from kubebrain_b200/csrc/kb_store.cu -- keep in step with it:
CHUNK = 16                # every key and value on a 16-byte boundary, zero padded
PASS_CHUNKS = 32          # k_key_exists / summarize_record: 32 chunks of two keys compared per warp pass
PASS_STARTS = 32          # summarize_record: 32 start positions of "/events/" tested per warp pass
DISPLACED_FLOOR = 4096    # apply_batch_locked: layout compaction when displaced > max(4096, N2 / 32) ...
DISPLACED_DIV = 32
GARBAGE_DIV = 4           # ... or garbage_k16 * 4 > key tail or garbage_v16 * 4 > value tail
MERGE_BLOCK = 256         # k_dir_merge: threads per block, one per old record and per insert
MAX_KEY = 65535           # klen is 16 bits
SLAB_SLACK = 64           # bytes kept zero behind each slab tail
DUMP_MAGIC = b"KBB200D1"
DUMP_HEADER = struct.Struct("<8sIIQQQQQIIQQQ")  # DumpHeader: 88 bytes
FNV_OFFSET, FNV_PRIME = 0xCBF29CE484222325, 0x100000001B3


def ik(uk: bytes, rev: int) -> bytes:
    return MAGIC + uk + b"$" + struct.pack(">Q", rev)


def chunks(n: int) -> int:
    return (n + CHUNK - 1) // CHUNK


def pad16(b: bytes) -> bytes:
    return b + b"\x00" * (-len(b) % CHUNK)


def lcp(a: bytes, b: bytes) -> int:
    m = min(len(a), len(b))
    lo, hi = 0, m
    while lo < hi:  # the longest common prefix, by bisection on slice equality
        mid = (lo + hi + 1) // 2
        if a[:mid] == b[:mid]:
            lo = mid
        else:
            hi = mid - 1
    return lo


def user_key(k: bytes) -> Optional[bytes]:
    """the user key of an internal key that decodes (coder.Decode), else None"""
    if len(k) < 13 or k[:4] != MAGIC or k[-9] != 0x24:
        return None
    return k[4:-9]


# ---- the heap model --------------------------------------------------------------------------------------------------
def _dbuf_cap(nbytes: int) -> int:
    """dbuf_ensure's allocation for a fresh buffer of `nbytes` (kb_core.cu)"""
    want = max(nbytes + nbytes // 4, 4096)
    return (want + 255) & ~255


class HeapModel:
    """kb_apply_batch's heap accounting (apply_batch_locked): chunks in use at the slab tails, garbage, records appended
    out of key order, the layout-compaction trigger and its deferral while a compaction stream is open, kb_dump's
    compaction, the TTL bookkeeping of kb_apply_batch / kb_expire.  `items` is the map the snapshot must hold."""

    def __init__(self, items: Sequence[Tuple[bytes, bytes]]):
        self.install(items)
        self.pinned = False  # an open compaction stream defers the layout compaction

    def install(self, items):
        """kb_load_sorted / kb_restore: a canonical layout, counters and TTLs afresh"""
        self.items: Dict[bytes, bytes] = dict(items)
        self.kused, self.vused = self.canonical()
        self.garbage_k = self.garbage_v = self.displaced = 0
        self.max_kv = max((chunks(len(k)) + chunks(len(v)) for k, v in self.items.items()), default=0)
        self.kcap, self.vcap = _dbuf_cap(self.kused * 16 + SLAB_SLACK), _dbuf_cap(self.vused * 16 + SLAB_SLACK)
        self.grows_k = self.grows_v = 0
        self.ttl_of: Dict[bytes, int] = {}
        self.ttl_queue: List[Tuple[int, int, bytes]] = []  # (expire, insertion order, key): a multimap's order
        self.ttl_seq = 0
        self.compactions = 0

    def canonical(self) -> Tuple[int, int]:
        return (sum(chunks(len(k)) for k in self.items), sum(chunks(len(v)) for v in self.items.values()))

    def info(self) -> Tuple[int, int, int]:
        """what kb_store_info must return"""
        return len(self.items), self.kused * 16, self.vused * 16

    def threshold(self, n2: int) -> int:
        return max(DISPLACED_FLOOR, n2 // DISPLACED_DIV)

    def compact_layout(self):
        self.kused, self.vused = self.canonical()
        self.kcap, self.vcap = _dbuf_cap(self.kused * 16 + SLAB_SLACK), _dbuf_cap(self.vused * 16 + SLAB_SLACK)
        self.garbage_k = self.garbage_v = self.displaced = 0
        self.compactions += 1

    def _reserve(self, which: str, tail16: int):
        need = tail16 * 16 + SLAB_SLACK
        cap = getattr(self, which + "cap")
        if cap < need:
            setattr(self, which + "cap", _dbuf_cap(need + need // 2))
            setattr(self, "grows_" + which, getattr(self, "grows_" + which) + 1)

    def apply(self, ops) -> Dict[str, object]:
        """one kb_apply_batch; returns the batch's facts (counts, the trigger's operands, whether it fired)"""
        last: Dict[bytes, Optional[bytes]] = {}
        for op in ops:  # last op per key wins
            last[op[0]] = op[1]
        n_ins = n_del = n_rep = 0
        gk = gv = 0
        ktail, vtail = self.kused, self.vused
        new = dict(self.items)
        for k in sorted(last):
            v = last[k]
            if v is not None:
                vtail += chunks(len(v))
                if k in self.items:
                    n_rep += 1
                    gv += chunks(len(self.items[k]))
                else:
                    n_ins += 1
                    ktail += chunks(len(k))
                self.max_kv = max(self.max_kv, chunks(len(k)) + chunks(len(v)))
                new[k] = v
            elif k in self.items:
                n_del += 1
                gk += chunks(len(k))
                gv += chunks(len(self.items[k]))
                del new[k]
        facts = dict(n_ins=n_ins, n_del=n_del, n_rep=n_rep, N=len(self.items), N2=len(new), fired=None)
        if n_ins + n_del + n_rep:  # a batch of only absent deletes changes nothing
            self._reserve("k", ktail)
            self._reserve("v", vtail)
            self.items = new
            self.kused, self.vused = ktail, vtail
            self.garbage_k += gk
            self.garbage_v += gv
            self.displaced += n_ins
            thr = self.threshold(len(new))
            facts.update(displaced=self.displaced, threshold=thr, garbage_k=self.garbage_k, garbage_v=self.garbage_v,
                         ktail=ktail, vtail=vtail, pinned=self.pinned)
            if not self.pinned:
                fired = [name for name, hit in (("displaced", self.displaced > thr),
                                                ("garbage_k", self.garbage_k * GARBAGE_DIV > ktail),
                                                ("garbage_v", self.garbage_v * GARBAGE_DIV > vtail)) if hit]
                if fired:
                    facts["fired"] = tuple(fired)
                    self.compact_layout()
        for op in ops:  # TTL bookkeeping, in op order
            k = op[0]
            if op[1] is not None and len(op) > 2 and op[2]:
                self.ttl_of[k] = op[2]
                self.ttl_seq += 1
                self.ttl_queue.append((op[2], self.ttl_seq, k))
            else:
                self.ttl_of.pop(k, None)
        return facts

    def expire(self, now: int) -> Tuple[int, Dict[str, object]]:
        """kb_expire(now): the keys whose current expiry is <= now are deleted; stale queue entries are dropped"""
        self.ttl_queue.sort()
        due, stale = [], 0
        while self.ttl_queue and self.ttl_queue[0][0] <= now:
            t, _, k = self.ttl_queue.pop(0)
            if self.ttl_of.get(k) == t:
                due.append(k)
                del self.ttl_of[k]
            else:
                stale += 1
        facts = dict(due=len(due), stale=stale, facts=None)
        if not due:
            return 0, facts
        before = len(self.items)
        facts["facts"] = self.apply([(k, None) for k in due])
        return before - len(self.items), facts

    def dump(self):
        """kb_dump compacts the layout first (and ends every compaction stream)"""
        self.pinned = False
        self.compact_layout()

    def sorted_items(self) -> List[Tuple[bytes, bytes]]:
        return sorted(self.items.items())


# ---- the dump file --------------------------------------------------------------------------------------------------
def fnv1a64_words(h: int, b: bytes) -> int:
    """kb_store.cu fnv1a64_update: 8 little-endian bytes per step, then the tail byte by byte"""
    n8 = len(b) - len(b) % 8
    for (w,) in struct.iter_unpack("<Q", b[:n8]):
        h = ((h ^ w) * FNV_PRIME) & 0xFFFFFFFFFFFFFFFF
    for c in b[n8:]:
        h = ((h ^ c) * FNV_PRIME) & 0xFFFFFFFFFFFFFFFF
    return h


def dump_image(items: Sequence[Tuple[bytes, bytes]], compact_rev: Optional[int] = None, max_kv_chunks: Optional[int] = None
               ) -> bytes:
    """the canonical KBB200D1 version-1 file of a sorted item list: header, directory (koff16 u32 x n+1 | klen u16 x n |
    voff16 u64 x n+1 | vlen u32 x n, every offset contiguous in key order), key slab, value slab, both zero padded"""
    n = len(items)
    koff, voff, ko, vo = [], [], 0, 0
    for k, v in items:
        koff.append(ko)
        voff.append(vo)
        ko += chunks(len(k))
        vo += chunks(len(v))
    koff.append(ko)
    voff.append(vo)
    parts = [struct.pack("<%dI" % (n + 1), *koff), struct.pack("<%dH" % n, *[len(k) for k, _ in items]),
             struct.pack("<%dQ" % (n + 1), *voff), struct.pack("<%dI" % n, *[len(v) for _, v in items])]
    sum_dir = FNV_OFFSET
    for p in parts:  # the directory's four arrays are summed one after the other, each from a word boundary
        sum_dir = fnv1a64_words(sum_dir, p)
    kslab = b"".join(pad16(k) for k, _ in items)
    vslab = b"".join(pad16(v) for _, v in items)
    if max_kv_chunks is None:
        max_kv_chunks = max((chunks(len(k)) + chunks(len(v)) for k, v in items), default=0)
    head = DUMP_HEADER.pack(DUMP_MAGIC, 1, DUMP_HEADER.size, n, ko, vo, int(compact_rev is not None), compact_rev or 0,
                            max_kv_chunks, 0, sum_dir, fnv1a64_words(FNV_OFFSET, kslab), fnv1a64_words(FNV_OFFSET, vslab))
    return head + b"".join(parts) + kslab + vslab


@dataclass
class Dump:
    header: Dict[str, int]
    koff16: List[int]
    klen: List[int]
    voff16: List[int]
    vlen: List[int]
    kslab: bytes
    vslab: bytes
    sums_ok: bool = field(default=False)

    def items(self) -> List[Tuple[bytes, bytes]]:
        return [(self.kslab[self.koff16[i] * 16: self.koff16[i] * 16 + self.klen[i]],
                 self.vslab[self.voff16[i] * 16: self.voff16[i] * 16 + self.vlen[i]]) for i in range(len(self.klen))]


HEADER_FIELDS = ("magic", "version", "header_bytes", "n", "key_chunks", "val_chunks", "compact_present", "compact_rev",
                 "max_kv_chunks", "pad", "sum_dir", "sum_keys", "sum_vals")


def parse_dump(blob: bytes) -> Dump:
    """a KBB200D1 file split into its fields; sums_ok says whether the three sums match the bytes"""
    h = dict(zip(HEADER_FIELDS, DUMP_HEADER.unpack_from(blob, 0)))
    n, at = h["n"], DUMP_HEADER.size
    parts = []
    for fmt, cnt in (("I", n + 1), ("H", n), ("Q", n + 1), ("I", n)):
        size = struct.calcsize("<%d%s" % (cnt, fmt))
        parts.append(blob[at: at + size])
        at += size
    koff, klen, voff, vlen = (list(struct.unpack("<%d%s" % (c, f), p)) for p, (f, c) in
                              zip(parts, (("I", n + 1), ("H", n), ("Q", n + 1), ("I", n))))
    kslab = blob[at: at + h["key_chunks"] * 16]
    at += len(kslab)
    vslab = blob[at: at + h["val_chunks"] * 16]
    sd = FNV_OFFSET
    for p in parts:
        sd = fnv1a64_words(sd, p)
    ok = (sd == h["sum_dir"] and fnv1a64_words(FNV_OFFSET, kslab) == h["sum_keys"] and
          fnv1a64_words(FNV_OFFSET, vslab) == h["sum_vals"] and at + len(vslab) == len(blob))
    return Dump(h, koff, klen, voff, vlen, kslab, vslab, ok)


# ---- shapes ---------------------------------------------------------------------------------------------------------
@dataclass
class Step:
    kind: str                       # "apply" | "expire" | "reload" (kb_load_sorted) | "restore" (kb_dump + kb_restore)
    ops: list = field(default_factory=list)
    now: int = 0
    dump: bool = False              # compare kb_dump with dump_image after this step
    stream: Optional[str] = None    # "open" / "close" a compaction stream in front of this step
    what: str = ""


@dataclass
class WShape:
    name: str
    start: List[Tuple[bytes, bytes]]
    steps: List[Step]
    revs: Tuple[int, ...] = (2**64 - 1, 6, 1)  # read revisions of the range checks
    slow: bool = False


def _mk(prefix: bytes, i: int, rev: int = 5) -> bytes:
    return ik(prefix + b"%07d" % i, rev)


def _base(n: int, prefix: bytes = b"/m/", step: int = 1000) -> List[Tuple[bytes, bytes]]:
    return [(_mk(prefix, i * step), b"v%d" % i * (i % 4)) for i in range(n)]


def _between(prefix: bytes, i: int, step: int, j: int) -> bytes:
    """a key behind record i - 1 and in front of record i of _base (lower bound i); j tells the ones of one gap apart"""
    return ik(prefix + b"%07d" % (i * step - 1) + b"/%04d" % j, 5)


def w1_merge() -> List[WShape]:
    P, S = b"/m/", 1000
    start = _base(1000, P, S)
    keys = [k for k, _ in start]
    b1 = [(ik(b"/a/0", 5), b"first"), (ik(b"/z/0", 5), b"last")]
    for gap, k in ((3, 1), (10, 2), (20, 31), (40, 32), (80, 33), (200, 257)):
        b1 += [(_between(P, gap, S, j), b"i%d" % j) for j in range(k)]
    b2 = [(keys[500], None), (_between(P, 500, S, 0), b"on deleted")]   # the insert's lower bound is deleted
    b2 += [(keys[i], None) for i in range(0, 5)] + [(ik(b"/a/1", 5), b"at 0"), (ik(b"/a/2", 5), b"at 0 too")]
    b2 += [(keys[i], None) for i in range(995, 1000)]
    b3 = [(keys[600], None), (keys[600], b"re-put"), (keys[601], b"put then"), (keys[601], None),
          (keys[700], b"replaced"), (_between(P, 700, S, 0), b"in front of a replacement")]
    steps = [Step("apply", b1, what="inserts at 0 / N, k on one bound"),
             Step("apply", b2, what="insert on a deleted record, delete runs at both ends", dump=True),
             Step("apply", b3, what="delete + re-put, replacement behind an insert")]
    m = HeapModel(start)
    for s in steps:
        m.apply(s.ops)
    cur = sorted(m.items)
    steps.append(Step("apply", [(k, b"every %d" % i) for i, k in enumerate(cur)], what="replace every record", dump=True))
    steps.append(Step("apply", [(k, None) for k in cur], what="delete every record"))
    steps.append(Step("apply", [(_mk(b"/e/", i), b"e%d" % i) for i in range(300)], what="inserts into the empty store",
                      dump=True))
    shapes = [WShape("W1 merge", start, steps)]
    for n in (255, 256, 257):
        st = _base(n, b"/t/", 10)
        sk = [k for k, _ in st]
        shapes.append(WShape("W1 N=%d" % n, st, [
            Step("apply", [(sk[n // 2], b"only a replacement")], what="n_ins 0"),
            Step("apply", [(_between(b"/t/", n - 1, 10, 0), b"one insert")], what="n_ins 1"),
            Step("apply", [(sk[0], None), (_between(b"/t/", 0, 10, 0), b"one insert at 0")], what="n_ins 1, N - 1")]))
    return shapes


def w1_big() -> WShape:
    """one batch of 200 000 inserts into a store of 1 000 (200 per gap): N + n_ins over 782 merge blocks"""
    start = _base(1000, b"/m/", 1000)
    ops = [(ik(b"/m/%07d" % (i * 5 + 1), 7), b"b%d" % i * (i % 3)) for i in range(200_000)]
    return WShape("W1 200k", start, [Step("apply", ops, what="200 000 inserts"),
                                     Step("apply", [(k, None) for k, _ in ops[::1000]], what="deletes among them")],
                  slow=True)


def _filler(n: int, seed: int) -> bytes:
    """n bytes of lower-case letters without `/events/` in them, distinct per seed early on"""
    s = (b"%05d" % seed) + bytes(97 + (i * 7 + seed) % 26 for i in range(max(n - 5, 0)))
    return s[:n]


LCP_TARGETS = (511, 512, 513, 1023, 1024, 1025)


def w2_keys() -> WShape:
    start: List[Tuple[bytes, bytes]] = []
    b1: list = []
    b2: list = []
    # op keys of every length class (raw keys below 13 bytes do not decode: they are still records)
    for L in (0, 1, 12, 13, 16, 17, 511, 512, 513, 1024, 65534, 65535):
        k = b"\x01" * min(L, 12) + (b"" if L <= 12 else (b"/len/%05d/" % L + b"q" * L)[: L - 12])
        b1.append((k, b"len %d" % L))
    # near misses of one stored key: one byte lower in chunk c (the op key is an insert whose lower bound is the
    # stored key, of the same length; k_key_exists has to see the difference in its pass c // 32)
    for c in (0, 31, 32, 33, 64):
        ns = b"/n/%02d/" % c
        base = ik(ns + _filler(1040 - 13 - len(ns), c), 5)
        assert len(base) == 1040
        at = 15 if c == 0 else (1025 if c == 64 else 16 * c + 7)
        near = base[:at] + bytes([base[at] - 1]) + base[at + 1:]
        start.append((base, b"stored %d" % c))
        b1.append((near, b"near %d" % c))
        b2.append((near, None))
    # a prefix of a stored key, and keys that extend one (by 0x00 and by a letter)
    px = ik(b"/p/" + _filler(700, 99), 5)
    start.append((px, b"px"))
    b1 += [(px[:600], b"prefix"), (px + b"\x00", b"ext nul"), (px + b"a", b"ext a")]
    # neighbours whose LCP is 511 .. 1 025: versions of one user key (L - 1 shared bytes) and near-miss user keys of one
    # length (4 + d shared bytes), each made by an insert, by deleting the record between and by a replacement
    for t in LCP_TARGETS:
        for how in ("insert", "delete", "replace"):
            ns = b"/v/%04d/%s/" % (t, how.encode())
            uk = ns + _filler(t + 1 - 13 - len(ns), t)   # internal key of t + 1 bytes: versions 5 and 6 share t
            a5, a6 = ik(uk, 5), ik(uk, 6)
            assert lcp(a5, a6) == t
            nu = ns + _filler(1100 - len(ns), t)            # near miss: the same user key but byte d = t - 4
            u1 = ik(nu, 5)
            d = t - 4
            u2 = ik(nu[:d] + bytes([nu[d] + 1]) + nu[d + 1:], 5)
            assert lcp(u1, u2) == t
            mid = ik(nu[:d] + bytes([nu[d] + 1]) + nu[d + 1: d + 40] + bytes([nu[d + 40] - 1]) + nu[d + 41:], 5)
            assert u1 < mid < u2 and lcp(mid, u2) > t
            if how == "insert":
                start += [(a5, b"a5"), (u1, b"u1")]
                b1 += [(a6, b"a6 new"), (u2, b"u2 new")]
            elif how == "delete":
                start += [(a5, b"a5"), (a5 + b"~", b"between"), (a6, b"a6"), (u1, b"u1"), (mid, b"mid"), (u2, b"u2")]
                b1 += [(a5 + b"~", None), (mid, None)]
            else:
                start += [(a5, b"a5"), (a6, b"a6"), (u1, b"u1"), (u2, b"u2")]
                b1 += [(a6, b"a6 replaced"), (u2, b"u2 replaced")]
    # `/events/` at user-key offsets 0, 31, 32, 33, 63, 64 and n - 8 (n = 100 and 1 000), and one running into `$`
    for n in (100, 1000):
        for p in (0, 31, 32, 33, 63, 64, n - 8):
            uk = b"/evt/%04d/%04d/" % (n, p)
            body = _filler(n, p + n)
            uk = (uk + body)[:p] + EVENTS + (uk + body)[p + 8:]
            uk = uk[:n]
            assert len(uk) == n and uk.find(EVENTS) == p, (n, p)
            b1.append((ik(uk, 4), b"event value %d" % p))
        uk = (b"/evt/%04d/tail" % n + _filler(n, 7))[: n - 7] + b"/events"
        b1.append((ik(uk, 4), b"not an event"))
    b3 = [(k, None) for k, _ in b1 if len(k) >= 65534] + [(px + b"\x00", None), (px, None)]
    return WShape("W2 keys", start, [Step("apply", b1, what="key bytes", dump=True),
                                     Step("apply", b2, what="near misses deleted"),
                                     Step("apply", b3, what="the longest keys and a prefix deleted", dump=True)],
                  revs=(2**64 - 1, 5, 4))


def _solve_threshold(n: int) -> int:
    """the number of inserts t into a store of n records at which displaced == max(4096, (n + t) / 32)"""
    t = DISPLACED_FLOOR
    while t != max(DISPLACED_FLOOR, (n + t) // DISPLACED_DIV):
        t = max(DISPLACED_FLOOR, (n + t) // DISPLACED_DIV)
    return t


def w3_heap() -> List[WShape]:
    shapes = []
    # the displaced trigger at its threshold and one past it, on the floor and on the N / 32 branch.  The first batch
    # also deletes 8 records and replaces 8 values by longer ones: garbage far below a quarter of either tail, but
    # enough that a compaction at the threshold would shrink both tails, so kb_store_info tells "fired" from "waited"
    for n, name in ((1000, "floor"), (140_000, "N/32")):
        start = [(ik(b"/h/%07d" % (i * 10), 5), b"h") for i in range(n)]
        dels = [(k, None) for k, _ in start[1::n // 8][:8]]
        reps = [(k, b"r" * 20) for k, _ in start[2::n // 8][:8]]
        t = _solve_threshold(n - len(dels))
        ins = [(ik(b"/h/%07d" % (i * 10 + 5), 5), b"x") for i in range(t + 1)]
        shapes.append(WShape("W3 displaced " + name, start, [
            Step("apply", ins[:t] + dels + reps, what="displaced at the threshold, some garbage"),
            Step("apply", ins[t:], what="one past it"),
            Step("apply", [(k, None) for k, _ in ins[: t // 2]], what="deletes after the compaction")],
            slow=n > 100_000))
    # garbage: 396 keys of 2 chunks + 8 of 1 chunk (800 key chunks), values empty; then the value side
    kstart = [(b"k2/%05d/" % i + b"g" * 20, b"") for i in range(396)] + [(b"k1/%02d" % i, b"") for i in range(8)]
    shapes.append(WShape("W3 garbage keys", kstart, [
        Step("apply", [(kstart[i][0], None) for i in range(100)], what="garbage_k at a quarter"),
        Step("apply", [(kstart[396][0], None)], what="one chunk past it", dump=True)]))
    vstart = [(b"v2/%05d" % i, b"w" * 32) for i in range(396)] + [(b"v1/%05d" % i, b"w") for i in range(8)]
    shapes.append(WShape("W3 garbage values", vstart, [
        Step("apply", [(vstart[i][0], b"") for i in range(0, 200, 2)], what="garbage_v at a quarter"),
        Step("apply", [(vstart[397][0], b"")], what="one chunk past it"),
        Step("apply", [(vstart[1][0], b"")], what="garbage again", dump=True)]))
    # growth: each batch doubles the store, keys and values of several chunks
    gstart = [(ik(b"/g/%07d" % (i * 1000), 5), b"g" * 40) for i in range(40)]
    steps, have = [], 40
    for r in range(5):
        steps.append(Step("apply", [(ik(b"/g/%07d" % (i * 7 + 3), 6), b"G" * (20 + r * 30)) for i in range(have * (r + 1))],
                          what="growth %d" % r))
        have *= 2
    shapes.append(WShape("W3 growth", gstart, steps, revs=(2**64 - 1, 5)))
    # replacements of empty values: nothing becomes garbage and nothing is displaced, but the layout is no longer in
    # key order -- the dump must still be canonical
    estart = [(ik(b"/z/%02d" % i, 5), b"" if i % 3 == 0 else b"z%d" % i) for i in range(10)] + [(ik(b"/z/99", 5), b"")]
    shapes.append(WShape("W3 empty values", estart, [
        Step("apply", [(estart[3][0], b"abc")], what="empty value replaced, not the last record", dump=True),
        Step("apply", [(estart[6][0], b"")], what="empty by empty, not the last record", dump=True),
        Step("apply", [(estart[-1][0], b"last")], what="empty value replaced, the last record", dump=True),
        Step("restore", what="the dump restores")]))
    # the trigger waits while a compaction stream is open, and fires on the first batch after it closed
    pstart = [(b"k2/%05d/" % i + b"g" * 20, b"") for i in range(400)]
    shapes.append(WShape("W3 pinned", pstart, [
        Step("apply", [(pstart[i][0], None) for i in range(150)], what="past a quarter, stream open", stream="open"),
        Step("apply", [(pstart[200][0], b"val")], what="stream closed", stream="close")]))
    return shapes


T0 = 1_700_000_000


def w4_ttl() -> List[WShape]:
    start = [(ik(b"/ttl/%04d" % i, 5), b"t%d" % i) for i in range(60)]
    keys = [k for k, _ in start]
    steps = [
        Step("apply", [(k, b"due", T0) for k in keys[:40]] + [(keys[40], b"a", T0 + 5), (keys[41], b"b", T0 + 10)],
             what="40 keys due in one second"),
        Step("expire", now=T0 - 1, what="one second early"),
        Step("expire", now=T0, what="exactly at t"),
        Step("apply", [(keys[40], b"a later", T0 + 20), (keys[41], b"b no ttl")], what="re-put later / without ttl"),
        Step("expire", now=T0 + 10, what="stale entries"),
        Step("apply", [(keys[42], b"c", T0 + 30), (keys[42], None), (keys[43], None), (keys[43], b"d", T0 + 30),
                       (keys[44], b"e", T0 + 30), (keys[44], b"e no ttl")], what="ttl ops inside one batch"),
        Step("expire", now=T0 + 30, what="only the del, put+ttl key"),
        Step("apply", [(keys[45], b"f", T0 + 50)], what="a ttl, then a reload"),
        Step("reload", what="kb_load_sorted drops TTLs"),
        Step("expire", now=T0 + 60),
        Step("apply", [(keys[46], b"g", T0 + 70)], what="a ttl, then a dump and restore"),
        Step("restore", what="kb_restore drops TTLs"),
        Step("expire", now=T0 + 80),
    ]
    _, m = shape_classes(WShape("", start, steps))
    steps += [Step("apply", [(k, b"end", T0 + 100) for k in sorted(m.items)], what="every key due"),
              Step("expire", now=T0 + 100, what="the expiry empties the store", dump=True),
              Step("apply", [(ik(b"/ttl/new", 9), b"after", T0 + 200)], what="writes after it")]
    return [WShape("W4 ttl", start, steps)]


def all_shapes(slow: bool = True) -> List[WShape]:
    out = w1_merge() + [w2_keys()] + w3_heap() + w4_ttl()
    if slow:
        out.insert(len(w1_merge()), w1_big())
    return [s for s in out if slow or not s.slow]


# ---- classes --------------------------------------------------------------------------------------------------------
def fixed_records(before: Dict[bytes, bytes], after: Dict[bytes, bytes]) -> List[Tuple[int, str]]:
    """records of the new store whose summary a batch must redo, from the two maps alone, with why: 'insert' (the
    record or its predecessor is new), 'delete' (its predecessor changed through deletes only), 'replace' (its value)"""
    bk = sorted(before)
    ak = sorted(after)
    prev_before = {k: (bk[i - 1] if i else None) for i, k in enumerate(bk)}
    out = []
    for i, k in enumerate(ak):
        p = ak[i - 1] if i else None
        if k not in before or (p is not None and p not in before):
            out.append((i, "insert"))
        elif prev_before[k] != p:
            out.append((i, "delete"))
        elif before[k] != after[k]:
            out.append((i, "replace"))
    return out


def write_classes(model: HeapModel, ops) -> Dict[str, object]:
    """what one batch reaches, from the bytes and the model (the model is advanced by the batch): lower-bound positions
    of the inserts, LCP passes and values of every fixed record by cause, op-key lengths, near misses and prefixes of
    the lower-bound record, `/events/` offsets of fixed records, k_dir_merge's threads, and the trigger"""
    before = dict(model.items)
    bk = sorted(before)
    N = len(bk)
    last: Dict[bytes, Optional[bytes]] = {}
    for op in ops:
        last[op[0]] = op[1]
    ins = sorted(k for k, v in last.items() if v is not None and k not in before)
    dels = {k for k, v in last.items() if v is None and k in before}
    reps = {k for k, v in last.items() if v is not None and k in before}
    lbs = Counter(bisect.bisect_left(bk, k) for k in ins)
    c: Dict[str, object] = {}
    c["lb0"] = lbs[0] > 0
    c["lbN"] = lbs[N] > 0 and N > 0
    c["per_bound"] = set(lbs.values())
    dpos = {bisect.bisect_left(bk, k) for k in dels}
    c["ins_on_deleted"] = any(p in dpos for p in lbs)
    c["del_0"] = 0 in dpos
    c["del_last"] = N - 1 in dpos and N > 0
    c["del_0_ins_0"] = 0 in dpos and lbs[0] > 0
    c["rep_behind_ins"] = any(bisect.bisect_left(bk, k) in lbs for k in reps)
    c["more_ins_than_N"] = len(ins) > N
    c["rep_all"] = N > 0 and len(reps) == N
    c["del_all"] = N > 0 and len(dels) == N
    c["ins_into_empty"] = N == 0 and len(ins) > 0
    order = {}
    for op in ops:
        order.setdefault(op[0], []).append(op[1] is None)
    c["del_then_put"] = any(a and not b for seq in order.values() for a, b in zip(seq, seq[1:]))
    c["put_then_del"] = any(not a and b for seq in order.values() for a, b in zip(seq, seq[1:]))
    c["merge_threads"] = N + len(ins)
    # op keys against the record k_key_exists compares them with (the lower bound)
    c["op_klens"] = {len(k) for k in last}
    near, pre = set(), set()
    for k in last:
        p = bisect.bisect_left(bk, k)
        if p < N and bk[p] != k:
            s = bk[p]
            d = lcp(k, s)
            if len(s) == len(k) and k[d + 1:] == s[d + 1:]:  # one byte apart: the chunk it is in
                near.add("last" if d // CHUNK == chunks(len(k)) - 1 else d // CHUNK)
            if s.startswith(k):
                pre.add("prefix")
        if p > 0 and k.startswith(bk[p - 1]) and k != bk[p - 1]:
            pre.add("extends_nul" if k[len(bk[p - 1])] == 0 else "extends")
    c["near_chunk"] = near
    c["prefix"] = pre
    # fixed records: LCP values / passes by cause, `/events/` offsets
    facts = model.apply(ops)
    after = model.items
    ak = sorted(after)
    lcps, passes, ev = set(), set(), set()
    for i, why in fixed_records(before, after):
        if i:
            v = lcp(ak[i], ak[i - 1])
            lcps.add((v, why))
            # the pass in which the lanes find the first differing chunk (the last pass when the shorter key ends)
            passes.add(min(v, min(len(ak[i]), len(ak[i - 1])) - 1) // CHUNK // PASS_CHUNKS if v else 0)
        uk = user_key(ak[i])
        if uk is not None:
            p = uk.find(EVENTS)
            if p >= 0:
                ev.add("last" if p == len(uk) - 8 else p)
            elif uk.endswith(EVENTS[:-1]):
                ev.add("into$")
    c["lcp"] = lcps
    c["lcp_pass"] = passes
    c["events_at"] = ev
    c["fired"] = facts["fired"]
    c["garbage"] = (facts.get("garbage_k", 0), facts.get("garbage_v", 0))  # after the batch, before a compaction
    if "threshold" in facts:
        c["displaced_vs_threshold"] = facts["displaced"] - facts["threshold"]
        c["big_branch"] = facts["threshold"] > DISPLACED_FLOOR
        c["gk_vs_quarter"] = facts["garbage_k"] * GARBAGE_DIV - facts["ktail"]
        c["gv_vs_quarter"] = facts["garbage_v"] * GARBAGE_DIV - facts["vtail"]
        c["pinned"] = facts["pinned"]
    return c


def shape_classes(shape: WShape) -> Tuple[List[Dict[str, object]], HeapModel]:
    """the classes of every step of a shape, and the model after it"""
    m = HeapModel(shape.start)
    out = []
    for s in shape.steps:
        if s.stream == "open":
            m.pinned = True
        elif s.stream == "close":
            m.pinned = False
        if s.kind == "apply":
            out.append(write_classes(m, s.ops))
        elif s.kind == "expire":
            queued = [t for t, _, _ in m.ttl_queue]
            dropped, f = m.expire(s.now)
            out.append(dict(expire=True, dropped=dropped, stale=f["stale"], at_now=queued.count(s.now),
                            same_second=max(Counter(queued).values(), default=0), emptied=dropped > 0 and not m.items))
        else:
            had_ttl = bool(m.ttl_of)
            m.install(m.items)
            out.append(dict(reinstall=s.kind, dropped_ttls=had_ttl))
        if s.dump:
            m.dump()
    return out, m


def merged(classes: List[Dict[str, object]]) -> Dict[str, object]:
    """the union of a shape's (or several shapes') step classes"""
    out: Dict[str, object] = {}
    for c in classes:
        for k, v in c.items():
            if isinstance(v, set):
                out.setdefault(k, set()).update(v)
            elif isinstance(v, bool):
                out[k] = out.get(k, False) or v
            else:
                out.setdefault(k, []).append(v)
    return out


if __name__ == "__main__":  # prints the classes every shape reaches
    for sh in all_shapes():
        cl, m = shape_classes(sh)
        mc = merged(cl)
        print("%-22s records %d -> %d, steps %d, compactions %d, slab growths %d/%d" % (
            sh.name, len(sh.start), len(m.items), len(sh.steps), m.compactions, m.grows_k, m.grows_v))
        for k in sorted(mc):
            v = mc[k]
            if isinstance(v, set):
                v = sorted(v, key=repr)
                if len(v) > 24:
                    v = v[:24] + ["..."]
            if v not in (False, [], None):
                print("    %-22s %s" % (k, v))
