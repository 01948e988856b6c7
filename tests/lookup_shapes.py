"""Stores, bounds and point reads built so that the bound search, the point-read kernels and the page cut
(kubebrain_b200/csrc/kb_search.cu: k_search / key_less; kb_batch.cu: k_get_resolve / k_get_finalize / get_submit_locked's
arena bound; kb_page.cu: k_page_cut) meet their fixed boundaries on purpose, and answers past 4 GiB (shared by the CPU and GPU tests).
  S1  pivots: store sizes around 32, 33, 33^2 and 33^3 records and one of 10^6, bounds equal to every record (or to every
      first- and second-round pivot and its neighbours), just below it and just above it, below the first and above the
      last record;
  S2  compare chunks: a bound whose first difference with a record falls on both sides of key_less's three prefetched
      chunks and of every later chunk seam, bounds that are proper prefixes of records and the reverse (ending at 16, 32,
      48, 64; continuing in 0x00 bytes or not), a bound of 65 535 bytes;
  P1  resolve: same-length neighbours of a read that differ only in the first, second or third 512-byte pass of
      k_get_resolve, a neighbour whose user key is the read key + '$' ..., reads below the first and above the last
      record, below an object's first version, at revisions whose top byte is '$', a bound + 0x00 that is a stored key,
      values one byte away from `tombstone` in each word the kernel compares;
  P2  finalize and arena: batches on both sides of k_get_finalize's 256-read chunks with FOUND reads only at chunk edges,
      empty values, wire elements whose body length crosses a varint length, one record read many times whose element
      is larger than its slab bytes;
  C   page cut: streams of 33, 34, 65 and 1 057 kvs (range and compaction), a budget of exactly the bytes of every cut;
  X   answers past 4 GiB: one range batch, one point-read batch and one range stream whose arena offsets cross 2^32.
`lookup_classes` derives from the store bytes and the oracle alone (never from the builders' bookkeeping) what each shape
reaches, so that tests/test_lookup_shapes.py can assert it on any host; `python -m tests.lookup_shapes` prints it."""
from __future__ import annotations

import bisect
import random
import struct
from typing import Dict, List, Sequence, Tuple

import numpy as np

from kubebrain_b200.packed import PackedStore, Slab
from tests import pyref

MAGIC = b"\x57\xfb\x80\x8b"
TOMB = b"tombstone"
ALL = 2**64 - 1
MASK64 = 2**64 - 1

# restated from kubebrain_b200/csrc/kb_search.cu (k_search, key_less), kb_internal.cuh (warp_prefix_eq), kb_batch.cu
# and kb_page.cu -- keep in step with them:
LANES = 32             # k_search / k_get_resolve / k_page_cut: one warp per bound, read or page
PIVOTS = 33            # k_search: pivot of lane l at lo + span * (l + 1) / 33; a span <= 32 is the final round
PREFETCH = 3           # key_less / KB_BOUND_READAHEAD16: chunks 0 .. 2 loaded together, the loop starts at chunk 3
CHUNK = 16             # keys and values on 16-byte boundaries, zero padded
RESOLVE_PASS = 512     # k_get_resolve (warp_prefix_eq): 32 lanes x 16 bytes of magic + key + '$' compared per pass
FINALIZE_CHUNK = 256   # k_get_finalize: reads per block-scan step, with a carry between steps
CUT_CANDIDATES = 32    # k_page_cut: cut candidates tested per pivot round; <= 32 left is the final round
WIRE_SLACK = 48        # get_submit_locked / range_submit_locked: wire tags and varints per element, at most
X_LINE = 2**32         # the line every X answer crosses


def ik(uk: bytes, rev: int) -> bytes:
    return MAGIC + uk + b"$" + struct.pack(">Q", rev)


def pad16(n: int) -> int:
    return (n + CHUNK - 1) & ~(CHUNK - 1)


def _letters(n: int, seed: int) -> bytes:
    """n bytes in 'b' .. 'y' (one up or down stays a letter), different per seed"""
    return bytes(98 + (i * 7 + seed * 13 + (i * i) % 5) % 24 for i in range(n))


def first_diff(a: bytes, b: bytes) -> int:
    """the first position where a and b differ; min(len) when one is a prefix of the other"""
    m = min(len(a), len(b))
    for i in range(m):
        if a[i] != b[i]:
            return i
    return m


def store_of(items) -> PackedStore:
    return PackedStore.from_items(list(dict(items).items()))


# ---- S1: pivots -----------------------------------------------------------------------------------------------------
S1_SIZES = (1, 2, 31, 32, 33, 34, 65, 66, 1088, 1089, 1090, 35936, 35937, 35938)
S1_BIG = 1_000_000
S1_ALL_BELOW = 2000     # stores up to this size get bounds at every record


def s1_key(i: int) -> bytes:
    return ik(b"/registry/s1/%08d" % (2 * i), 5)


def s1_store(n: int) -> PackedStore:
    keys = [s1_key(i) for i in range(n)]
    return PackedStore(Slab.from_list(keys), Slab.from_list([b""] * n))


def round_pivots(lo: int, hi: int) -> List[int]:
    span = hi - lo
    return [lo + span * (lane + 1) // PIVOTS for lane in range(LANES)] if span > LANES else []


def search_pivots(n: int) -> Tuple[List[int], List[int]]:
    """the first- and second-round pivots of k_search on n records (the same for every bound)"""
    r1 = round_pivots(0, n)
    r2: List[int] = []
    if r1:
        edges = [(0, r1[0])] + [(r1[k] + 1, r1[k + 1]) for k in range(len(r1) - 1)] + [(r1[-1] + 1, n)]
        for lo, hi in edges:
            r2 += round_pivots(lo, hi)
    return r1, r2


def s1_bounds(keys: Sequence[bytes], seed: int = 1) -> List[bytes]:
    """bounds equal to, just below (a proper prefix) and just above (+ 0x00) the chosen records, and beyond both ends"""
    n = len(keys)
    if n <= S1_ALL_BELOW:
        pick = set(range(n))
    else:
        r1, r2 = search_pivots(n)
        pick = {j for p in r1 + r2 for j in (p - 1, p, p + 1) if 0 <= j < n}
        pick |= set(random.Random(seed).sample(range(n), 400)) | {0, n - 1}
    out = [b"", b"\x00", MAGIC]
    for i in sorted(pick):
        k = keys[i]
        out += [k, k[:-1], k + b"\x00"]
    if n:
        out += [keys[-1] + b"\xff", b"\xff"]
    return out


def search_trace(keys: Sequence[bytes], b: bytes) -> Tuple[int, List[int]]:
    """k_search on a sorted key list, restated: (lower bound, span of every round)"""
    lo, hi, spans = 0, len(keys), []
    while hi > lo:
        span = hi - lo
        spans.append(span)
        if span <= LANES:
            lo += sum(1 for lane in range(span) if keys[lo + lane] < b)
            break
        piv = round_pivots(lo, hi)
        k = sum(1 for p in piv if keys[p] < b)
        nlo = piv[k - 1] + 1 if k > 0 else lo
        nhi = piv[k] if k < LANES else hi
        lo, hi = nlo, nhi
    return lo, spans


# ---- S2: compare chunks ---------------------------------------------------------------------------------------------
DIFF_AT = (0, 15, 16, 31, 32, 47, 48, 63, 64, 1000)
PREFIX_AT = (16, 32, 48, 64)
S2_LEN = 1100


def s2_shape() -> Tuple[PackedStore, List[bytes]]:
    keys: List[bytes] = []
    bounds: List[bytes] = []
    fam = iter(range(0x30, 0x7f))
    for d in DIFF_AT:  # a record, the same bytes one higher at d, and bounds one up / one down at d
        r = bytes([next(fam)]) + _letters(S2_LEN - 1, d)
        up = r[:d] + bytes([r[d] + 2]) + r[d + 1:]
        keys += [r, up]
        bounds += [r[:d] + bytes([r[d] + 1]) + r[d + 1:], r[:d] + bytes([r[d] - 1]) + r[d + 1:]]
        bounds += [r[:d] + bytes([r[d] + 1]), up[: d + 1] + b"\x00" * 40]  # shorter / longer after the difference
    for m in PREFIX_AT:
        for tail in (b"", b"\x00"):
            # the bound a proper prefix of a record (the record goes on in letters or in 0x00 bytes)
            x = bytes([next(fam)]) + _letters(m - 1, m)
            keys.append(x + (tail * 40 if tail else _letters(40, 3)))
            bounds.append(x)
            # the record a proper prefix of the bound (the bound goes on in letters or in 0x00 bytes)
            y = bytes([next(fam)]) + _letters(m - 1, m + 1)
            keys.append(y)
            bounds.append(y + (tail * 40 if tail else _letters(40, 4)))
    long_base = keys[0]
    bounds += [long_base + _letters(65535 - len(long_base), 9),                      # above the record: a prefix of it
               long_base[:500] + bytes([long_base[500] - 1]) + _letters(65535 - 501, 10)]  # below it, at byte 500
    keys = sorted(set(keys))
    bounds += list(keys)  # and every record itself
    return PackedStore(Slab.from_list(keys), Slab.from_list([b"s2"] * len(keys))), bounds


def search_classes(keys: Sequence[bytes], bounds: Sequence[bytes]) -> Dict[str, object]:
    """what a set of bounds reaches in k_search / key_less, from the keys alone: the first difference (or the prefix
    relation) with the two records around the lower bound, the final round's span and the lane the answer ends on"""
    n = len(keys)
    r1, r2 = search_pivots(n)
    piv = set(r1) | set(r2)
    c: Dict[str, object] = dict(n=n, diff_at=set(), prefix=set(), final_span=set(), at_pivot=set(), rounds=set(),
                                equal=False, last_lane=False, below_all=False, above_all=False, max_bound=0)
    for b in bounds:
        lb = bisect.bisect_left(keys, b)
        got, spans = search_trace(keys, b)
        assert got == lb
        c["rounds"].add(len(spans))
        if spans:
            c["final_span"].add(spans[-1])
        c["below_all"] |= lb == 0 and n > 0
        c["above_all"] |= lb == n and n > 0
        c["max_bound"] = max(c["max_bound"], len(b))
        for j in (lb - 1, lb):
            if 0 <= j < n:
                k = keys[j]
                if k == b:
                    c["equal"] = True
                    if j in piv:
                        c["at_pivot"].add("r1" if j in r1 else "r2")
                    continue
                d = first_diff(k, b)
                if d < min(len(k), len(b)):
                    c["diff_at"].add(d)
                else:  # the shorter ends at d: which one, and whether the longer goes on in 0x00 bytes
                    longer = k if len(k) > len(b) else b
                    who = "bound_prefix" if len(b) < len(k) else "record_prefix"
                    c["prefix"].add((who, d, "nul" if longer[d] == 0 else "byte"))
        # the answer taken by the final round's last lane: lower bound at the end of a full final window
        if spans and spans[-1] == LANES and lb > 0:
            c["last_lane"] = True
    return c


# ---- P1: resolve ------------------------------------------------------------------------------------------------------
PRE_TARGETS = (511, 512, 513, 1023, 1024, 1025)   # pre = magic + key + '$' = len(key) + 5
NEAR_CHUNKS = (0, 31, 32, 33, "last")
R24 = 0x2400000000000500                          # a revision whose top byte is '$'
TOMB_OFFSETS = (0, 3, 4, 7, 8)


def _near_pos(pre: int, c) -> int:
    """the internal-key byte a neighbour changes to differ from the read only in chunk c (a user-key byte)"""
    return pre - 2 if c == "last" else (15 if c == 0 else 16 * c + 7)


def p1_shape() -> Tuple[PackedStore, List[Tuple[bytes, int]]]:
    items: Dict[bytes, bytes] = {}
    reads: List[Tuple[bytes, int]] = []
    for pre in PRE_TARGETS:
        ul = pre - 5
        for c in NEAR_CHUNKS:
            p = _near_pos(pre, c)
            if p > pre - 2:
                continue
            head = b"%04d%-2s" % (pre, str(c)[:2].encode())
            k = head + _letters(ul - len(head), pre + p)       # the read key: no records of its own
            u = p - 4                                          # the byte in the user key
            nb = k[:u] + bytes([k[u] - 1]) + k[u + 1:]         # same length, just below it
            items[ik(nb, 5)] = b"near %d %s" % (pre, str(c).encode())
            reads += [(k, 0), (k, 5), (k, 6)]
        # an object with keys of this length that is found
        m = b"%04dFF" % pre + _letters(ul - 6, pre)
        items[ik(m, 0)] = struct.pack(">Q", 20)
        items[ik(m, 10)] = b"v10"
        items[ik(m, 20)] = b"v20 " + _letters(30, pre)
        reads += [(m, r) for r in (0, 1, 9, 10, 11, 19, 20, 21, ALL)]
    # the lower neighbour's user key is the read key + '$' ...: it passes the compare of pre bytes, fails kl == pre + 8
    for j, ext in enumerate((b"$\x00\x00", b"$abc", b"$" + b"\x00" * 7, b"$" + b"z" * 7)):
        k = b"/p1/dollar/%d" % j
        items[ik(k + ext, 5)] = b"ext"
        reads += [(k, 0), (k, 5), (k, ALL)]
    items[ik(b"/p1/dollar/9", 3)] = b"shadowed"                   # with an older version of its own below the extension
    items[ik(b"/p1/dollar/9$\x00", 5)] = b"ext"
    reads += [(b"/p1/dollar/9", 0), (b"/p1/dollar/9", 3), (b"/p1/dollar/9", 4)]
    # below the first and above the last record
    reads += [(b"", 0), (b"!", 5), (b"\xff\xff", 0), (b"\xff", ALL)]
    # below an object's first version: the candidate is its revision record (rev 0), or another key
    items[ik(b"/p1/early/a", 0)] = struct.pack(">Q", 40)
    items[ik(b"/p1/early/a", 30)] = b"a30"
    items[ik(b"/p1/early/a", 40)] = b"a40"
    items[ik(b"/p1/early/b", 30)] = b"b30"
    for k in (b"/p1/early/a", b"/p1/early/b"):
        reads += [(k, r) for r in (0, 1, 29, 30, 31, 39, 40, 41, ALL, ALL - 1)]
    # revisions whose top byte is '$'
    for r in (R24 - 7, R24 + 9, 0x24FFFFFFFFFFFFF0):
        items[ik(b"/p1/top24", r)] = b"t%x" % r
    reads += [(b"/p1/top24", r) for r in (R24 - 8, R24 - 7, R24 - 6, R24, R24 + 9, R24 + 10, 0x24FFFFFFFFFFFFEF,
                                          0x24FFFFFFFFFFFFF0, 0x24FFFFFFFFFFFFF1, 0x2500000000000000, 0)]
    # the bound + 0x00 is a stored key: key + '$' at revision (R << 8) mod 2^64
    items[ik(b"/p1/shift", 7)] = b"v7"
    items[ik(b"/p1/shift$", (R24 << 8) & MASK64)] = b"shifted"
    reads += [(b"/p1/shift", r) for r in (R24 - 1, R24, R24 + 1, 0)] + [(b"/p1/shift$", 0)]
    # tombstones and values one byte away from one, in each of the three words the kernel compares
    vals = [TOMB, TOMB[:-1], TOMB + b"\x00", TOMB + b"e"]
    vals += [TOMB[:o] + bytes([TOMB[o] + 1]) + TOMB[o + 1:] for o in TOMB_OFFSETS]
    vals += [TOMB[:o] + bytes([TOMB[o] - 1]) + TOMB[o + 1:] for o in TOMB_OFFSETS]
    for j, v in enumerate(vals):
        k = b"/p1/tomb/%02d" % j
        items[ik(k, 8)] = v
        items[ik(k, 4)] = b"before"
        reads += [(k, 0), (k, 8), (k, 4)]
    return store_of(items), reads


def get_classes(keys: Sequence[bytes], vals: Sequence[bytes], reads) -> Dict[str, object]:
    """what point reads reach in k_get_resolve, from the keys and the reference alone: the lower bound of every read's
    bound, its candidate (the record below), whether the candidate has the right length, the chunk and pass of the
    first difference of a same-length candidate, the reference's answer"""
    n = len(keys)
    c: Dict[str, object] = dict(pre=set(), near=set(), passes=set(), ext_dollar=False, idx0=False, idx_n=False,
                                rev_record=False, top24=False, bound_is_key=False, tomb=set(), status=set(), found_pre=set())
    for uk, rev in reads:
        r = rev or ALL
        bound = ik(uk, r) + b"\x00"
        pre = len(uk) + 5
        idx = bisect.bisect_left(keys, bound)
        c["idx0"] |= idx == 0
        c["idx_n"] |= idx == n
        c["top24"] |= (r >> 56) == 0x24
        c["bound_is_key"] |= idx < n and keys[idx] == bound
        got, mod = pyref.get(keys, vals, uk, rev)
        status = "found" if got >= 0 else "tombstone" if got == -2 else "not_found"
        c["status"].add(status)
        if idx == 0:
            continue
        cand = keys[idx - 1]
        if len(cand) == pre + 8:
            d = first_diff(cand[:pre], bound[:pre])
            if d < pre:
                ch = d // CHUNK
                c["near"].add((pre, "last" if ch == (pre - 2) // CHUNK else ch))
                c["passes"].add(d // RESOLVE_PASS)
            elif cand[pre:] == b"\x00" * 8:
                c["rev_record"] = True
            if status == "found":
                c["found_pre"].add(pre)
        elif cand[:pre] == bound[:pre]:
            c["ext_dollar"] = True  # its user key is the read key + '$' ...
        c["pre"].add(pre)
        if len(cand) == pre + 8 and cand[:pre] == bound[:pre]:  # the candidate answers: what its value is
            v = vals[idx - 1]
            if v == TOMB:
                c["tomb"].add("equal")
            elif len(v) == 9 and sum(x != y for x, y in zip(v, TOMB)) == 1:
                c["tomb"].add(first_diff(v, TOMB))
            elif v.startswith(TOMB[:8]):
                c["tomb"].add("len%d" % len(v))
    return c


# ---- P2: finalize and arena -----------------------------------------------------------------------------------------
P2_SIZES = (1, 255, 256, 257, 511, 512, 513, 65535, 65536, 65537)
P2_PATTERNS = ("none", "all", "edge255", "edge0", "last", "alternate")
BODY_TARGETS = (127, 128, 16383, 16384)


def varint_len(v: int) -> int:
    n = 1
    while v >= 0x80:
        v >>= 7
        n += 1
    return n


def kv_body(ul: int, vl: int, rev: int) -> int:
    """mvccpb.KeyValue's body bytes (kb_wire.cuh wire_sizes)"""
    return ((1 + varint_len(ul) + ul) if ul else 0) + ((1 + varint_len(rev)) if rev else 0) + \
        ((1 + varint_len(vl) + vl) if vl else 0)


def kvs_elem(ul: int, vl: int, rev: int) -> int:
    b = kv_body(ul, vl, rev)
    return 1 + varint_len(b) + b


def _value_for_body(ul: int, rev: int, target: int) -> int:
    for vl in range(1, 20000):
        if kv_body(ul, vl, rev) == target:
            return vl
    raise AssertionError((ul, rev, target))


def p2_store() -> Tuple[PackedStore, List[bytes], List[bytes]]:
    """objects with values of 0 .. 199 bytes (every fifth empty) and values whose wire body is 127, 128, 16 383 and
    16 384 bytes; returns the store, user keys that are found and user keys that are not"""
    items: Dict[bytes, bytes] = {}
    found = []
    for i in range(300):
        uk = b"/p2/%05d" % i
        items[ik(uk, 0)] = struct.pack(">Q", 10 + i)
        items[ik(uk, 10 + i)] = b"" if i % 5 == 0 else bytes([i % 251]) * ((i * 37) % 200)
        found.append(uk)
    for t in BODY_TARGETS:
        for rev in (1, 300, 2**40):
            uk = b"/p2/w/%05d/%d" % (t, rev)
            vl = _value_for_body(len(uk), rev, t)
            items[ik(uk, rev)] = bytes([t % 251]) * vl
            found.append(uk)
    missing = [b"/p2/%05d/none" % i for i in range(300)]
    return store_of(items), found, missing


def p2_reads(n: int, pattern: str, found: Sequence[bytes], missing: Sequence[bytes]) -> List[Tuple[bytes, int]]:
    hit = {"none": lambda i: False, "all": lambda i: True, "edge255": lambda i: i % FINALIZE_CHUNK == FINALIZE_CHUNK - 1,
           "edge0": lambda i: i % FINALIZE_CHUNK == 0, "last": lambda i: i == n - 1,
           "alternate": lambda i: i % 2 == 1}[pattern]
    return [((found[(i * 7) % len(found)] if hit(i) else missing[i % len(missing)]), 0) for i in range(n)]


P2_ONE_REV = 2**63 + 5


def p2_one_store() -> PackedStore:
    """one record: a 3-byte user key (a 16-byte internal key), a 16-byte value, a revision >= 2^63 -- its wire element
    (36 bytes) is larger than its slab bytes (32)"""
    return store_of({ik(b"abc", P2_ONE_REV): b"0123456789abcdef"})


def get_arena_bound(reads: Sequence[Tuple[bytes, int]], max_kv_chunks: int, slab_bytes: int, wire: bool) -> int:
    """get_submit_locked's arena bound: n times the largest pair, capped at `most` copies of both slabs, + 48 n (wire)"""
    n = len(reads)
    ub = n * max_kv_chunks * CHUNK
    if ub > slab_bytes:
        most = max(np.unique([k for k, _ in reads], return_counts=True)[1]) if n else 0
        ub = min(ub, int(most) * slab_bytes)
    return ub + (n * WIRE_SLACK if wire else 0)


def finalize_classes(status_found: Sequence[bool]) -> Dict[str, object]:
    """where the FOUND reads of a batch sit against k_get_finalize's 256-read chunks"""
    n = len(status_found)
    f = [i for i, x in enumerate(status_found) if x]
    return dict(n=n, chunks=(n + FINALIZE_CHUNK - 1) // FINALIZE_CHUNK, found=len(f),
                at=set(i % FINALIZE_CHUNK for i in f) if len(set(i % FINALIZE_CHUNK for i in f)) <= 2 else "spread",
                carry=any(i >= FINALIZE_CHUNK for i in f))


# ---- C: page cut ------------------------------------------------------------------------------------------------------
C_SIZES = (33, 34, 65, 1057)
C_GROUPS = (1, 7)


def c_range_store(n: int) -> PackedStore:
    """n objects of one version each, pairs of different sizes (every cut is at a different byte count)"""
    return store_of({ik(b"/c/%05d" % i + b"k" * (i % 23), 5): bytes([i % 251]) * ((i * 29) % 97) for i in range(n)})


def c_compact_store(n: int) -> PackedStore:
    """n objects of two versions each: a sweep at revision 9 deletes the n older ones"""
    items = {}
    for i in range(n):
        uk = b"/c/%05d" % i + b"q" * (i % 37)
        items[ik(uk, 5)] = b"old"
        items[ik(uk, 7)] = b"new %d" % i
    return store_of(items)


def cut_candidates(n: int, group: int) -> int:
    return (n + group - 1) // group


def cut_classes(sizes: Sequence[int], group: int) -> Dict[str, object]:
    """the first page's cut search: candidate cuts, pivot rounds, and which candidates are first-round pivots"""
    g = cut_candidates(len(sizes), group)
    # candidates k = 1 .. g (the page ends at min(k group, n)); the first round's pivots are 1 + (g - 1) lane / 31
    piv = sorted({1 + (g - 1) * lane // (CUT_CANDIDATES - 1) for lane in range(CUT_CANDIDATES)}) if g > CUT_CANDIDATES else []
    return dict(candidates=g, pivot_round=g > CUT_CANDIDATES, pivots=piv,
                distinct=len(set(np.cumsum(sizes).tolist())) == len(sizes))


# ---- X: answers past 4 GiB ------------------------------------------------------------------------------------------
X_N = 4100
X_KEY = b"abc"                  # internal key of 16 bytes
X_VAL_EXACT = 2**20 - 16        # pair of exactly 2^20: the kv of request 4 096 starts at 2^32
X_VAL_STRADDLE = 2**20          # pair of 2^20 + 16: kv 4 095 straddles 2^32
X_REV = 77
X_PAGE = 256 << 20


def x_store(val_len: int, n_objects: int = 1) -> PackedStore:
    """n objects with 3-byte user keys and values of val_len bytes; each value starts with its object's number and ends
    in 0xa5, so that a shifted or truncated copy shows"""
    keys = [ik(struct.pack(">I", i)[1:] if n_objects > 1 else X_KEY, X_REV) for i in range(n_objects)]
    data = np.zeros(n_objects * val_len, np.uint8)
    starts = np.arange(n_objects, dtype=np.int64) * val_len
    for b in range(4):
        data[starts + b] = (np.arange(n_objects) >> (8 * b)) & 0xFF
    data[starts + val_len - 1] = 0xA5
    data[starts + 4] = 0x5A
    return PackedStore(Slab.from_list(keys), Slab(data, (np.arange(n_objects + 1, dtype=np.uint64) * val_len)))


def x_pair(key: bytes, val: bytes) -> np.ndarray:
    """a kv's bytes in the raw arena: [internal key, zero padded][value, zero padded]"""
    out = np.zeros(pad16(len(key)) + pad16(len(val)), np.uint8)
    out[: len(key)] = np.frombuffer(key, np.uint8)
    out[pad16(len(key)): pad16(len(key)) + len(val)] = np.frombuffer(val, np.uint8)
    return out


def x_layout(unit: int, n: int = X_N) -> Dict[str, object]:
    """where 2^32 falls in an answer of n entries of `unit` bytes each"""
    k = X_LINE // unit
    return dict(total=n * unit, past=n * unit > X_LINE, starts_at_line=X_LINE % unit == 0 and k < n,
                straddles=X_LINE % unit != 0 and k < n, entry_at_line=k)


def lookup_classes() -> Dict[str, Dict[str, object]]:
    """every shape's classes (the X and the large S1 stores by their sizes alone)"""
    out: Dict[str, Dict[str, object]] = {}
    for n in S1_SIZES:
        st = s1_store(n)
        keys = st.keys.tolist()
        out["S1 n=%d" % n] = search_classes(keys, s1_bounds(keys))
    st, bounds = s2_shape()
    out["S2"] = search_classes(st.keys.tolist(), bounds)
    st, reads = p1_shape()
    out["P1"] = get_classes(st.keys.tolist(), st.vals.tolist(), reads)
    st, found, missing = p2_store()
    keys, vals = st.keys.tolist(), st.vals.tolist()
    for n in P2_SIZES:
        for pat in P2_PATTERNS:
            reads = p2_reads(n, pat, found, missing)
            out["P2 n=%d %s" % (n, pat)] = finalize_classes([pyref.get(keys, vals, k, r)[0] >= 0 for k, r in reads])
    for n in C_SIZES:
        st = c_range_store(n)
        sizes = [pad16(len(st.keys[i])) + pad16(len(st.vals[i])) for i in range(n)]
        for g in C_GROUPS:
            out["C n=%d group=%d" % (n, g)] = cut_classes(sizes, g)
    out["X1 exact"] = x_layout(pad16(len(ik(X_KEY, X_REV))) + pad16(X_VAL_EXACT))
    out["X1 straddle"] = x_layout(pad16(len(ik(X_KEY, X_REV))) + pad16(X_VAL_STRADDLE))
    out["X1 wire"] = x_layout(kvs_elem(len(X_KEY), X_VAL_EXACT, X_REV))
    out["X2 raw"] = x_layout(pad16(X_VAL_EXACT))
    out["X3 stream"] = x_layout(pad16(len(ik(X_KEY, X_REV))) + pad16(X_VAL_EXACT))
    return out


if __name__ == "__main__":  # prints the classes every shape reaches
    for name, c in lookup_classes().items():
        print(name)
        for k in sorted(c):
            v = c[k]
            if isinstance(v, (set, list)):
                v = sorted(v, key=repr)
                if len(v) > 24:
                    v = v[:24] + ["..."]
            if v not in (False, [], None):
                print("    %-14s %s" % (k, v))
