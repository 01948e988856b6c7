"""The partition definition of kb_range_partitions, restated from the oracle's answer, and the stores its tests cut.

Let e_0 .. e_{n-1} be the unlimited answer of [start, end) at read_rev (ko.range_), slot[i] the raw-arena bytes
(pad16(internal key) + pad16(value) per kv) in front of e_i and T their total.
  P = min(max_parts, n, max(1, ceil(T / part_bytes))), and P = 1 when n <= 1 or start >= end.
  cut k (k = 1 .. P-1) = the least i in [1, n) with slot[i] * P >= k * T; a cut with no such i, or equal to the cut
  before it, is dropped.
  border of cut i = EncodeRevisionKey(userKey(e_i)): the internal key of e_i with its 8 revision bytes zeroed."""
from __future__ import annotations

import bisect
import random
from typing import List, Sequence, Tuple

from kubebrain_b200.packed import PackedStore
from oracle import binding as ko
from tests.range_shapes import TOMB, be, ik

ALL = 2**64 - 1
MAX_PARTS = 4096


def pad16(n: int) -> int:
    return (n + 15) & ~15


def part_count(n: int, total: int, part_bytes: int, max_parts: int, start: bytes, end: bytes) -> int:
    if n <= 1 or start >= end:
        return 1
    return min(max_parts, n, max(1, -(-total // part_bytes)))


def cuts_of(sizes: Sequence[int], part_bytes: int, max_parts: int, start: bytes = b"a", end: bytes = b"b") -> List[int]:
    """the kept cuts (kv indices) of an answer whose kvs take sizes[i] arena bytes"""
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


def partitions(store: PackedStore, st: ko.OracleStore, start: bytes, end: bytes, read_rev: int, part_bytes: int,
               max_parts: int) -> Tuple[List[bytes], List[int], List[int]]:
    """(borders, kv_first, arena_first) of [start, end) at read_rev"""
    x = ko.range_(st, start, end, read_rev, 0)
    assert x.rc == 0
    emit = [int(i) for i in x.emit]
    sizes = [pad16(len(store.keys[i])) + pad16(len(store.vals[i])) for i in emit]
    cuts = cuts_of(sizes, part_bytes, max_parts, start, end)
    slot = [0]
    for s in sizes:
        slot.append(slot[-1] + s)
    borders = [start] + [revision_key(store.keys[emit[i]]) for i in cuts] + [end]
    return borders, [0] + cuts + [len(emit)], [0] + [slot[i] for i in cuts] + [slot[-1]]


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
