"""The partition definition of kb_range_partitions, restated from the oracle's answer, the invariants any partitioning
must keep (checked against the oracle alone), and the stores its tests cut.

Let e_0 .. e_{n-1} be the unlimited answer of [start, end) at read_rev (ko.range_), slot[i] the raw-arena bytes
(pad16(internal key) + pad16(value) per kv) in front of e_i and T their total.
  P = min(max_parts, n, max(1, ceil(T / part_bytes))), and P = 1 when n <= 1; start >= end is one partition of no kv.
  cut k (k = 1 .. P-1) = the least i in [1, n) with slot[i] * P >= k * T; a cut with no such i, equal to the cut
  before it, or whose border is not above e_{i-1}'s internal key, is dropped.
  border of cut i = EncodeRevisionKey(userKey(e_i)): the internal key of e_i with its 8 revision bytes zeroed.
A border at or below e_{i-1} happens when e_{i-1}'s user key is e_i's + '$' + bytes that sort below e_i's revision
bytes (U and U$\\0\\0\\0\\0\\0\\0\\0: the records of U$... sort between U's revision record and U's versions).  Every
kept border is then above the one before and above start, below end, and each partition answers exactly its kvs at
read_rev.  At other read revisions the partitions answer the whole only where no user key's records straddle a border,
which, again, takes a user key that is another's + '$' + bytes (`straddles`).

The boundary shapes put k_partition_cut's (kubebrain_b200/csrc/kb_page.cu) fixed edges in place on purpose:
  Q1  key order: user keys U, U$ + 7 x 0x00 + a low byte and three nested levels of it, with and without revision
      records; cuts on either key of an interleaved pair and on both; start and end inside one object's versions, start
      between a revision record and its first version, start == revision_key(e_1), start >= end, b"" starts, ends of
      b"" and 0xff;
  Q2  search (warp_partition_point over [1, n)): n - 1 of 31 .. 34 and 1 099 (a first pivot round), every i a cut,
      slot[i] * P == k * T exactly and one kv 16 bytes longer, T == part_bytes * k and +- 1, a kv larger than several
      shares, a last kv so large that no kv reaches the late cuts;
  Q3  warps and clamps: P - 1 of 15 .. 17 and 31 .. 33 (16 warps, strided), max_parts 4096, the n clamp;
  Q4  report: cut keys of 13, 16, 17, 31 .. 33 and 65 535 bytes and of every length mod 16, P = 4096 with a 64 KiB key
      stride, small / large / small P and a longer key written between calls on one engine;
  Q5  snapshots: after a batch that deletes, tombstones or inserts in front of a cut kv, after expire, after restore.
`partition_classes` derives from the bytes and the oracle alone what each shape reaches, so that
tests/test_partition_shapes.py can assert it on any host; `python -m tests.partition_shapes` prints it."""
from __future__ import annotations

import bisect
import random
import struct
from typing import Dict, List, Optional, Sequence, Tuple

from kubebrain_b200.packed import PackedStore
from oracle import binding as ko
from tests.range_shapes import MAGIC, TOMB, be, ik

ALL = 2**64 - 1
MAX_PARTS = 4096
WARPS = 16        # k_partition_cut: one CTA of 16 warps, warp w takes cuts w + 1, w + 17, ...
PUB_HEAD = 16     # KB_PUB_HEAD: bytes in front of a report's payload


def pad16(n: int) -> int:
    return (n + 15) & ~15


def part_count(n: int, total: int, part_bytes: int, max_parts: int, start: bytes, end: bytes) -> int:
    if n <= 1 or start >= end:
        return 1
    return min(max_parts, n, max(1, -(-total // part_bytes)))


def cuts_of(sizes: Sequence[int], part_bytes: int, max_parts: int, start: bytes = b"a", end: bytes = b"b") -> List[int]:
    """the cuts (kv indices) of an answer whose kvs take sizes[i] arena bytes, before the key-order drop"""
    n = len(sizes)
    slot = [0]
    for s in sizes:
        slot.append(slot[-1] + int(s))
    total = slot[n]
    p = part_count(n, total, part_bytes, max_parts, start, end)
    scaled = [slot[i] * p for i in range(1, n)]  # non-decreasing: the cut of share k is a lower bound in it
    out: List[int] = []
    for k in range(1, p):
        i = 1 + bisect.bisect_left(scaled, k * total)
        if i >= n or (out and out[-1] == i):
            continue
        out.append(i)
    return out


def revision_key(internal_key: bytes) -> bytes:
    return internal_key[:-8] + b"\x00" * 8


def decode(internal_key: bytes) -> Optional[Tuple[bytes, int]]:
    """(user key, revision) as the coder decodes it (coder.go Decode), None when it does not"""
    if len(internal_key) < 13 or internal_key[:4] != MAGIC or internal_key[-9:-8] != b"$":
        return None
    return internal_key[4:-9], struct.unpack(">Q", internal_key[-8:])[0]


def partitions(store: PackedStore, st: ko.OracleStore, start: bytes, end: bytes, read_rev: int, part_bytes: int,
               max_parts: int) -> Tuple[List[bytes], List[int], List[int]]:
    """(borders, kv_first, arena_first) of [start, end) at read_rev"""
    if start >= end:  # the interval holds nothing
        return [start, end], [0, 0], [0, 0]
    x = ko.range_(st, start, end, read_rev, 0)
    assert x.rc == 0
    emit = [int(i) for i in x.emit]
    sizes = [pad16(len(store.keys[i])) + pad16(len(store.vals[i])) for i in emit]
    keys = [store.keys[i] for i in emit]
    cuts = [i for i in cuts_of(sizes, part_bytes, max_parts, start, end) if revision_key(keys[i]) > keys[i - 1]]
    slot = [0]
    for s in sizes:
        slot.append(slot[-1] + s)
    borders = [start] + [revision_key(keys[i]) for i in cuts] + [end]
    return borders, [0] + cuts + [len(emit)], [0] + [slot[i] for i in cuts] + [slot[-1]]


# ---- the invariants ---------------------------------------------------------------------------------------------------
def adjust_partitions_borders(parts: Sequence[Tuple[bytes, bytes]]) -> List[Tuple[bytes, bytes]]:
    """scanner.go adjustPartitionsBorders: sort the partitions by start, chain each start to the end before it, and move
    an inner end that decodes with a revision to its user key's revision key"""
    ps = sorted([list(p) for p in parts], key=lambda p: p[0])
    for i in range(len(ps)):
        if i:
            ps[i][0] = ps[i - 1][1]
        if i != len(ps) - 1:
            d = decode(ps[i][1])
            if d is not None and d[1] != 0:
                ps[i][1] = ik(d[0], 0)
    return [tuple(p) for p in ps]


def straddles(store: PackedStore, borders: Sequence[bytes]) -> List[Tuple[bytes, bytes]]:
    """(border, user key) for every inner border some user key has records on both sides of"""
    inner = sorted(borders[1:-1])
    if not inner:
        return []
    lo: Dict[bytes, bytes] = {}
    hi: Dict[bytes, bytes] = {}
    for k in store.keys.tolist():
        d = decode(k)
        if d is not None:
            lo.setdefault(d[0], k)
            hi[d[0]] = k
    out = []
    for uk, a in lo.items():
        for j in range(bisect.bisect_right(inner, a), bisect.bisect_right(inner, hi[uk])):
            out.append((inner[j], uk))  # lo < border <= hi
    return out


def check_partitions(store: PackedStore, st: ko.OracleStore, start: bytes, end: bytes, read_rev: int,
                     got: Tuple[Sequence[bytes], Sequence[int], Sequence[int]], other_revs: Sequence[int] = ()):
    """any (borders, kv_first, arena_first) of [start, end) at read_rev against the oracle alone; returns the straddles
    (the partitions then answer the whole only at read_rev)"""
    borders, kv_first, arena_first = list(got[0]), [int(x) for x in got[1]], [int(x) for x in got[2]]
    whole = ko.range_(st, start, end, read_rev, 0).emit.tolist()
    sizes = [pad16(len(store.keys[i])) + pad16(len(store.vals[i])) for i in whole]
    assert borders[0] == start and borders[-1] == end, "first and last border"
    assert len(kv_first) == len(arena_first) == len(borders), "one kv_first and arena_first per border"
    if start >= end:  # one partition, the interval itself, holding nothing
        assert len(borders) == 2 and kv_first == [0, 0] and arena_first == [0, 0], "start >= end"
        return []
    assert all(a < b for a, b in zip(borders, borders[1:])), "borders strictly increasing"
    assert kv_first[0] == 0 and kv_first[-1] == len(whole), "kv_first spans the answer"
    for p, (a, b) in enumerate(zip(borders, borders[1:])):
        assert kv_first[p] < kv_first[p + 1] or len(borders) == 2, ("partition %d holds no kv" % p)
        part = ko.range_(st, a, b, read_rev, 0).emit.tolist() if a < b else []
        assert part == whole[kv_first[p]: kv_first[p + 1]], ("partition %d answers its kvs" % p)
        assert arena_first[p + 1] - arena_first[p] == sum(sizes[kv_first[p]: kv_first[p + 1]]), \
            ("partition %d arena bytes" % p)
    for b in borders[1:-1]:
        d = decode(b)
        assert d is not None and d[1] == 0, "inner border is a revision key"
    parts = list(zip(borders, borders[1:]))
    assert adjust_partitions_borders(parts) == parts, "adjustPartitionsBorders keeps the partitions"
    split = straddles(store, borders)
    if not split:
        for r in other_revs:
            w = ko.range_(st, start, end, r, 0).emit.tolist()
            cat = []
            for a, b in parts:
                cat += ko.range_(st, a, b, r, 0).emit.tolist() if a < b else []
            assert cat == w, ("whole at revision", r)
    return split


# ---- stores -----------------------------------------------------------------------------------------------------------
READ = 1000  # read revision the shapes are built around


def uniform_store(n: int, val_len: int = 40, prefix: bytes = b"/u/") -> PackedStore:
    """n objects of one version each with equal-sized kvs: the cut of share k is ceil(k n / P)"""
    return PackedStore.from_items([(ik(prefix + b"o%07d" % j, 100 + j % 500), b"v" * val_len) for j in range(n)])


def mixed_store(seed: int = 7, n_objects: int = 3000) -> PackedStore:
    """objects with versions below and above READ, tombstoned last versions, revision-record-only keys, undecodable
    records beside every kind, user keys that prefix others, and a few kvs far larger than the rest"""
    rng = random.Random(seed)
    items = {}
    for j in range(n_objects):
        uk = b"/m/%05d" % j
        kind = rng.randrange(8)
        if kind == 7:
            uk = b"/m/%05d" % (j - 1) + rng.choice([b"", b"!", b"%", b"x", b"/sub"])  # a prefix of it exists
        revs = sorted(rng.sample(range(1, 2 * READ), rng.randint(1, 4)))
        items[ik(uk, 0)] = be(revs[-1])
        if kind == 0:  # the revision record alone
            continue
        big = rng.random() < 0.01
        for r in revs:
            items[ik(uk, r)] = b"B" * rng.randint(20_000, 60_000) if big else b"%d" % r * rng.randint(1, 40)
        if kind == 1:  # the last version is a tombstone
            items[ik(uk, revs[-1])] = TOMB
        if kind == 2:  # an undecodable record inside the key's space, next to whatever the cut lands on
            items[ik(uk, revs[0]) + b"~junk"] = b"junk"
        if kind == 3:
            items[ik(uk, 0)] = be(revs[-1], True)
    return PackedStore.from_items(sorted(items.items()))


def long_key_store(n: int = 12) -> PackedStore:
    """internal keys of exactly 65 535 bytes (the format's limit) between short ones; the short keys' values make the
    two kvs of a pair about as large, so cuts land on both"""
    items = []
    for j in range(n):
        items.append((ik(b"/l/%03d" % j, 10 + j), b"s" * 65536))
        items.append((ik(b"/l/%03d~" % j + b"k" * (65535 - 13 - 7), 20 + j), b"L" * (j * 100)))
    return PackedStore.from_items(sorted(items))


# ---- Q1: key order ----------------------------------------------------------------------------------------------------
NUL7 = b"\x00" * 7
Q1_REVS = (READ, 2, 3, 600, ALL)  # read revisions: the nested keys' low revision bytes sit around 1 .. 3


def nest(uk: bytes, low: int) -> bytes:
    """a user key whose records sort among uk's: uk + '$' + 7 x 0x00 + low, between uk@(low - 1) and uk@(low + 1)"""
    return uk + b"$" + NUL7 + bytes([low])


def q1_store(rev_records: bool = True) -> PackedStore:
    """the interleaved pair of the partitions issue (/q/c and /q/c$ + 7 x 0x00 + 0x00) and three nested levels under
    /n/k whose versions fall on both sides of the next level's records, each with or without revision records"""
    objs: Dict[bytes, List[Tuple[int, bytes]]] = {
        b"/q/a": [(100, b"a100")],
        b"/q/c": [(1000, b"c1000")],
        nest(b"/q/c", 0): [(500, b"c$500")],
        b"/q/z": [(200, b"z200")],
    }
    u = b"/n/k"
    levels = [u]
    for low in (1, 2, 3):
        levels.append(nest(levels[-1], low))
    for d, uk in enumerate(levels):  # versions below (1 .. 3), at and above the nested records
        objs[uk] = [(1, b"L%d@1" % d), (2, b"L%d@2" % d), (4, b"L%d@4" % d + b"x" * 30 * d), (600, b"L%d@600" % d),
                    (READ, TOMB if d == 2 else b"L%d@1000" % d)]
    objs[b"/n/a"] = [(5, b"a5")]
    objs[nest(b"/n/a", 9)] = [(7, b"a$7")]  # nested but entirely above its outer key's records
    objs[b"/n/z"] = [(5, b"z5"), (1500, b"z1500")]
    items = {}
    for uk, vs in objs.items():
        if rev_records:
            items[ik(uk, 0)] = be(max(r for r, _ in vs), vs[-1][1] == TOMB)
        for r, v in vs:
            items[ik(uk, r)] = v
    return PackedStore.from_items(list(items.items()))


def q1_intervals(store: PackedStore) -> List[Tuple[str, bytes, bytes]]:
    """(name, start, end): the whole prefixes and every start / end edge Q1 asks for"""
    keys = store.keys.tolist()
    c = b"/q/c"
    ck = nest(b"/n/k", 1)
    out = [("q", ik(b"/q/", 0), ik(b"/q0", 0)), ("n", ik(b"/n/", 0), ik(b"/n0", 0)),
           ("all", b"", b"\xff"), ("q_to_ff", ik(b"/q/", 0), b"\xff")]
    out += [("start_in_versions", ik(b"/n/z", 600), ik(b"/n0", 0)), ("end_in_versions", ik(b"/n/", 0), ik(ck, 3)),
            ("both_in_versions", ik(b"/n/k", 500), ik(b"/n/k", 700))]
    out += [("start_after_revrec", ik(b"/n/k", 0) + b"\x00", ik(b"/n0", 0)),
            ("start_after_revrec_q", ik(c, 0) + b"\x00", ik(b"/q0", 0))]
    # start == revision_key(e_1): e_0 is the nested key's version that sorts between /q/c's revision key and /q/c@1000
    out += [("start_is_revkey_e1", ik(c, 0), ik(b"/q0", 0))]
    out += [("start_ge_end", ik(b"/q0", 0), ik(b"/q/", 0)), ("start_eq_end", ik(c, 0), ik(c, 0)),
            ("end_empty", b"", b""), ("start_empty_end_ff", b"", b"\xff"), ("start_empty_end_mid", b"", ik(c, 0))]
    assert all(k for k in keys)
    return out


def q1_part_bytes(total: int, n: int) -> List[int]:
    """shares that put cuts on every kv (1), on about every other, and on a few"""
    return sorted({1, max(1, total // max(n // 2, 1)), max(1, total // 3), max(1, total // 5), max(1, total // 7),
                   max(1, total // 11), total + 1})


# ---- Q2: search --------------------------------------------------------------------------------------------------------
Q2_N = (32, 33, 34, 35, 1100)   # n - 1 = 31 .. 34 cut candidates, and a first pivot round over 1 099


def sized_store(val_lens: Sequence[int], prefix: bytes = b"/s/") -> PackedStore:
    """one version per object, internal keys of 23 bytes (32 padded), values of the given lengths"""
    return PackedStore.from_items([(ik(prefix + b"o%07d" % j, 10 + j % 900), b"w" * v) for j, v in enumerate(val_lens)])


def first_pivots(n: int) -> List[int]:
    """warp_partition_point's first-round pivots over [1, n) (none when n - 1 <= 32)"""
    span = n - 1
    return sorted({1 + (span - 1) * lane // 31 for lane in range(32)}) if span > 32 else []


# ---- Q4: report -------------------------------------------------------------------------------------------------------
Q4_KEY_LENS = tuple(sorted(set(range(13, 29)) | {31, 32, 33, 65535}))


def q4_store() -> PackedStore:
    """one object per internal key length of Q4_KEY_LENS (13: the empty user key), values that make every pair as large
    as the one with the 65 535-byte key, so that a cut lands on every kv"""
    items = []
    for L in Q4_KEY_LENS:
        ul = L - 13
        uk = (b"/%05d/" % L + b"k" * ul)[:ul]
        items.append((ik(uk, 7 + L % 50), b"q" * (66048 - pad16(L))))
    return PackedStore.from_items(items)


def report_bytes(parts: int, max_kv_chunks: int) -> int:
    """k_partition_cut's pinned report: head, one 32-byte entry per cut, one key stride (the largest padded pair) per
    cut; hostpub_ensure allocates 1.5 times what it is asked for"""
    return PUB_HEAD + (parts - 1) * 32 + (parts - 1) * max_kv_chunks * 16


def max_kv_chunks(store: PackedStore) -> int:
    return max((pad16(len(k)) + pad16(len(v))) // 16 for k, v in zip(store.keys.tolist(), store.vals.tolist()))


# a 65 535-byte key among uniform_store's: right behind the 820 kvs whose 80-byte pairs first outweigh its own, so that
# the cut of two shares of [/u/, /u/o0000820) lands on it
LONG_KEY = ik(b"/u/o0000819~" + b"y" * (65535 - 13 - 12), 77)


def stride_store(n: int = 4200) -> PackedStore:
    """n uniform objects and one kv with a 65 535-byte key: the report's key stride is 64 KiB + a chunk"""
    items = [(ik(b"/u/o%07d" % j, 100 + j % 500), b"v" * 40) for j in range(n)]
    items.append((LONG_KEY, b"long"))
    return PackedStore.from_items(items)


# ---- Q5: snapshots ----------------------------------------------------------------------------------------------------
def q5_store() -> PackedStore:
    """200 objects of two versions and a revision record each"""
    items = {}
    for j in range(200):
        uk = b"/r/%04d" % j
        items[ik(uk, 0)] = be(300 + j)
        items[ik(uk, 10 + j)] = b"old%d" % j * (1 + j % 7)
        items[ik(uk, 300 + j)] = b"new%d" % j * (1 + j % 11)
    return PackedStore.from_items(list(items.items()))


def apply_model(items: Dict[bytes, bytes], ops: Sequence[tuple]) -> PackedStore:
    for op in ops:
        if op[1] is None:
            items.pop(op[0], None)
        else:
            items[op[0]] = op[1]
    return PackedStore.from_items(list(items.items()))


# ---- classes ------------------------------------------------------------------------------------------------------------
def _nested(a: bytes, b: bytes) -> bool:
    """is user key b user key a + '$' + bytes"""
    return len(b) > len(a) and b[: len(a) + 1] == a + b"$"


def order_classes(store: PackedStore, st: ko.OracleStore, start: bytes, end: bytes, read_rev: int,
                  part_bytes_list: Sequence[int], max_parts: int = MAX_PARTS) -> Dict[str, object]:
    """what one interval's cuts reach in key order: cuts dropped because their border is not above the kv in front,
    cuts on the outer / inner key of a nested pair in the answer and both in one call, where start sits"""
    emit = ko.range_(st, start, end, read_rev, 0).emit.tolist()
    keys = [store.keys[i] for i in emit]
    uks = [decode(k)[0] for k in keys]
    sizes = [pad16(len(store.keys[i])) + pad16(len(store.vals[i])) for i in emit]
    outer = {a for a in uks for b in uks if _nested(a, b)}
    inner = {b for a in uks for b in uks if _nested(a, b)}
    c: Dict[str, object] = dict(n=len(emit), order_drop=False, on_outer=False, on_inner=False, both=False, depth=0,
                                straddle=False, start_ge_end=start >= end, start_empty=start == b"",
                                end=("empty" if end == b"" else "ff" if end == b"\xff" else "key"))
    depth = {u: 0 for u in uks}
    for u in sorted(uks, key=len):
        for a in uks:
            if _nested(a, u):
                depth[u] = max(depth[u], depth[a] + 1)
    c["depth"] = max(depth.values(), default=0)
    for pb in part_bytes_list:
        raw = cuts_of(sizes, pb, max_parts, start, end)
        kept = [i for i in raw if revision_key(keys[i]) > keys[i - 1]]
        c["order_drop"] |= len(kept) < len(raw)
        hit_o = any(uks[i] in outer for i in raw)
        hit_i = any(uks[i] in inner for i in raw)
        c["on_outer"] |= hit_o
        c["on_inner"] |= hit_i
        c["both"] |= hit_o and hit_i
        borders = [start] + [revision_key(keys[i]) for i in kept] + [end]
        c["straddle"] |= bool(straddles(store, borders))
    # where start sits against the records of one user key
    lb = st.lower_bound(start)
    below = decode(store.keys[lb - 1]) if lb > 0 else None
    above = decode(store.keys[lb]) if lb < store.n else None
    c["start_in_versions"] = bool(below and above and below[0] == above[0] and below[1] > 0)
    c["start_after_revrec"] = bool(below and above and below[0] == above[0] and below[1] == 0)
    c["start_is_revkey_e1"] = len(keys) > 1 and start == revision_key(keys[1])
    lb = st.lower_bound(end)
    below = decode(store.keys[lb - 1]) if 0 < lb <= store.n else None
    above = decode(store.keys[lb]) if lb < store.n else None
    c["end_in_versions"] = bool(below and above and below[0] == above[0] and below[1] > 0)
    return c


def search_classes(sizes: Sequence[int], part_bytes: int, max_parts: int) -> Dict[str, object]:
    """what one call reaches in the cut search: cuts at i = 1 and n - 1, on a first-round pivot and one past it, exact
    equality slot[i] * P == k * T, cuts no kv reaches, repeated cuts, P against T / part_bytes"""
    n = len(sizes)
    slot = [0]
    for s in sizes:
        slot.append(slot[-1] + s)
    T = slot[n]
    P = part_count(n, T, part_bytes, max_parts, b"a", b"b")
    raw = []
    for k in range(1, P):
        i = next((i for i in range(1, n) if slot[i] * P >= k * T), n)
        raw.append((k, i))
    piv = set(first_pivots(n))
    cuts = {i for _, i in raw}
    return dict(n=n, P=P, at1=1 in cuts, at_last=(n - 1) in cuts, on_pivot=bool(cuts & piv),
                past_pivot=bool(cuts & {p + 1 for p in piv}), exact=any(i < n and slot[i] * P == k * T for k, i in raw),
                unreached=any(i == n for _, i in raw), repeated=len({i for _, i in raw if i < n}) < len(
                    [i for _, i in raw if i < n]), t_vs_share=(T - part_bytes * (P if T % part_bytes == 0 else P - 1)))


def partition_classes() -> Dict[str, Dict[str, object]]:
    out: Dict[str, Dict[str, object]] = {}
    for rr in (True, False):
        store = q1_store(rr)
        st = ko.OracleStore(store)
        for name, s, e in q1_intervals(store):
            for rev in (READ, ALL):
                emit = ko.range_(st, s, e, rev, 0).emit.tolist()
                total = sum(pad16(len(store.keys[i])) + pad16(len(store.vals[i])) for i in emit)
                out["Q1 %s%s rev=%d" % (name, "" if rr else " no-revrec", rev if rev != ALL else -1)] = order_classes(
                    store, st, s, e, rev, q1_part_bytes(total, len(emit)))
    for n in Q2_N:
        sizes = [80] * n
        out["Q2 n=%d every" % n] = search_classes(sizes, 1, MAX_PARTS)
        out["Q2 n=%d exact" % n] = search_classes(sizes, 80 * n // 2, MAX_PARTS)
    sizes = [80] * 34
    sizes[17] += 16
    out["Q2 n=34 bumped"] = search_classes(sizes, sum(sizes) // 2, MAX_PARTS)
    for d in (-1, 0, 1):
        out["Q2 T=7pb%+d" % d] = search_classes([80] * 35, 80 * 35 // 7 + d, MAX_PARTS)
    big = [80] * 100
    big[40] = 80 * 100 * 3
    out["Q2 big"] = search_classes(big, sum(big) // 20, MAX_PARTS)
    last = [80] * 100 + [80 * 100 * 5]
    out["Q2 last huge"] = search_classes(last, sum(last) // 20, MAX_PARTS)
    for p in (16, 17, 18, 32, 33, 34):
        out["Q3 P=%d" % p] = dict(P=p, cuts=p - 1, last_warp=(p - 2) % WARPS, rounds=-(-(p - 1) // WARPS))
    st = q4_store()
    out["Q4 key lengths"] = dict(lens=sorted({len(k) for k in st.keys.tolist()}),
                                 mod16=sorted({len(k) % 16 for k in st.keys.tolist()}))
    out["Q4 stride"] = dict(max_kv_chunks=max_kv_chunks(stride_store()),
                            report=report_bytes(MAX_PARTS, max_kv_chunks(stride_store())))
    return out


if __name__ == "__main__":  # prints the classes every shape reaches
    for name, c in partition_classes().items():
        print(name)
        for k in sorted(c):
            v = c[k]
            if isinstance(v, (set, list)):
                v = sorted(v, key=repr)
            if v not in (False, [], None):
                print("    %-18s %s" % (k, v))
