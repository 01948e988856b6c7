"""Reconciliation cases built so that kb_reconcile (kubebrain_b200/csrc/kb_reconcile.cu) meets its boundaries on purpose
(shared by the CPU and GPU tests).

A shape is what the snapshot holds (`mirror`), what the engine holds (`engine`), the interval, and either one call over
the interval or a chunked walk of it the way the storage adaptor's Verify walks the engine (chunk ends at the interval's
end on EOF, else at the last key + 0x00).
  edges   diffs at the first and last record of the interval, a key equal to `start`, a key equal to `end` that must be
          neither read nor touched, divergent records just outside both borders;
  values  differences at byte 0, 15, 16, 17 and the last byte of a 4096-byte value, lengths one apart with equal padded
          chunks, empty versus "\\0", `tombstone` values, 8- versus 9-byte revision-record values;
  keys    diff keys of 1, 15, 16, 17 and 65535 bytes, keys one apart in their last byte, a key that is a prefix of the next;
  sizes   n and hi - lo at 0, 1, 31/32/33, 127/128/129, 1023/1024/1025 and 10^5: all missing, all extra, identical, one
          diff in 10^5;
  walks   chunks of 1, 2, 7 and 4096, with chunk ends on divergent keys;
  interplay  an open compaction stream, an open range stream, a range batch in flight, TTL keys changed and unchanged.
`diff` is the plain merge model; `walk` restates the chunking; `reconcile_classes` derives what a shape reaches from the
bytes alone, so that tests/test_reconcile_shapes.py can assert it on any host.  `python -m tests.reconcile_shapes`
prints it."""
from __future__ import annotations

import struct
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

from tests.write_shapes import CHUNK, T0, ik, pad16

MISSING, EXTRA, CHANGED = 1, 2, 3
NO_SRC = 2**64 - 1
SIZES = (0, 1, 31, 32, 33, 127, 128, 129, 1023, 1024, 1025)
BIG = 100_000

Items = List[Tuple[bytes, bytes]]


def diff(mirror: Dict[bytes, bytes], inp: Items, start: bytes, end: bytes) -> List[Tuple[int, bytes, int]]:
    """the diff of one call: (kind, key, src_idx) in key order -- inp is the engine's records of [start, end)"""
    mine = {k: v for k, v in mirror.items() if start <= k < end} if start < end else {}
    out = []
    given = {k: i for i, (k, _) in enumerate(inp)}
    for k in sorted(set(mine) | set(given)):
        if k not in mine:
            out.append((MISSING, k, given[k]))
        elif k not in given:
            out.append((EXTRA, k, NO_SRC))
        elif inp[given[k]][1] != mine[k]:
            out.append((CHANGED, k, given[k]))
    return out


def ops_of(d, inp: Items):
    """the batch a real call commits: puts of the engine's value (no TTL) and deletes, in key order"""
    return [(k, None) if kind == EXTRA else (k, inp[src][1]) for kind, k, src in d]


def interval_items(items: Dict[bytes, bytes], start: bytes, end: bytes) -> Items:
    return sorted((k, v) for k, v in items.items() if start <= k < end)


def walk(engine: Dict[bytes, bytes], start: bytes, end: bytes, chunk: int) -> List[Tuple[bytes, bytes, Items]]:
    """the chunks of a Verify walk: (chunk start, chunk end, the engine's records of the chunk)"""
    out = []
    cur = start
    all_items = interval_items(engine, start, end)
    i = 0
    while True:
        got = all_items[i: i + chunk]
        i += len(got)
        if len(got) < chunk:  # EOF: the chunk ends at the interval's end
            out.append((cur, end, got))
            return out
        nxt = got[-1][0] + b"\x00"
        out.append((cur, nxt, got))
        cur = nxt


@dataclass
class RShape:
    name: str
    mirror: Items
    engine: Items
    start: bytes
    end: bytes
    chunks: Tuple[int, ...] = ()         # () = one call over [start, end); else a walk per chunk size
    ttl: Dict[bytes, int] = field(default_factory=dict)  # mirror keys put again with this expiry after the load
    interplay: str = ""                  # "compact_stream" | "range_stream" | "range_batch" | "ttl"
    tags: Tuple[str, ...] = ()           # what the shape is built to reach (checked against reconcile_classes)
    slow: bool = False


def _k(ns: bytes, i: int, rev: int = 5) -> bytes:
    return ik(ns + b"%07d" % i, rev)


def _items(ns: bytes, idx, val=lambda i: b"v%d" % i) -> Items:
    return [(_k(ns, i), val(i)) for i in idx]


# ---- edges ----------------------------------------------------------------------------------------------------------
def edges() -> List[RShape]:
    base = _items(b"/e/", range(20))
    s, e = base[3][0], base[15][0]  # a key equal to start (record 3) and one equal to end (record 15)
    eng = dict(base)
    eng[base[3][0]] = b"first changed"          # the first record of the interval, which is `start`
    eng[base[14][0]] = b"last changed"          # its last record
    eng[base[15][0]] = b"end: not read"         # key == end: outside, divergent, must stay
    eng[base[2][0]] = b"just below start"       # divergent records just outside both borders
    del eng[base[16][0]]
    mirror = dict(base)
    mirror[_k(b"/e/", 9) + b"x"] = b"extra in the middle"
    shapes = [RShape("edges", sorted(mirror.items()), sorted(eng.items()), s, e,
                     tags=("diff_first", "diff_last", "key_eq_start", "key_eq_end", "outside_divergent"))]
    # the first and last records of the interval missing / extra (not changed)
    m2 = dict(base)
    del m2[base[3][0]]
    e2 = dict(base)
    del e2[base[14][0]]
    shapes.append(RShape("edges missing first, extra last", sorted(m2.items()), sorted(e2.items()), s, e,
                         tags=("diff_first", "diff_last", "key_eq_start")))
    return shapes


# ---- values ---------------------------------------------------------------------------------------------------------
def values() -> RShape:
    mirror, eng = [], []
    big = bytes((i * 31 + 7) % 251 for i in range(4096))
    for j, at in enumerate((0, 15, 16, 17, 4095)):
        k = _k(b"/val/byte/", j)
        mirror.append((k, big))
        eng.append((k, big[:at] + bytes([big[at] ^ 0x5A]) + big[at + 1:]))
    pairs = [(b"abc", b"abc\x00"), (b"x" * 16, b"x" * 15), (b"x" * 31, b"x" * 31 + b"\x00"), (b"", b"\x00"),
             (b"tombstone", b"tombstonf"), (b"tombstone", b"tombstone"), (b"live", b"tombstone"),
             (struct.pack(">Q", 7), struct.pack(">Q", 7) + b"\x01"), (struct.pack(">Q", 8), struct.pack(">Q", 9)),
             (b"same", b"same"), (big, big)]
    for j, (a, b) in enumerate(pairs):
        k = ik(b"/val/pair/%02d" % j, 0 if len(a) in (8, 9) or len(b) in (8, 9) else 5)
        mirror.append((k, a))
        eng.append((k, b))
    return RShape("values", sorted(mirror), sorted(eng), b"", b"\xff" * 4,
                  tags=("byte_0", "byte_15", "byte_16", "byte_17", "byte_last", "len_pm1_equal_pad", "empty_vs_nul",
                        "tombstone", "rev8_vs_9"))


# ---- keys -----------------------------------------------------------------------------------------------------------
def keys() -> RShape:
    mirror, eng = [], []
    for L in (1, 15, 16, 17, 65535):
        k = (b"\x01" + b"/k/%05d/" % L + b"q" * L)[:L]
        (mirror if L % 2 else eng).append((k, b"len %d" % L))  # odd lengths only in the snapshot, even only given
    a = _k(b"/kl/", 1)
    b = a[:-1] + bytes([a[-1] + 1])                 # one apart in the last byte
    mirror += [(a, b"a"), (b, b"b")]
    eng += [(a, b"a"), (b, b"b changed")]
    p = ik(b"/kp/prefix", 5)
    mirror += [(p, b"p")]
    eng += [(p, b"p"), (p + b"/longer", b"extends the one before")]
    return RShape("keys", sorted(mirror), sorted(eng), b"", b"\xff" * 4,
                  tags=("klen_1", "klen_15", "klen_16", "klen_17", "klen_65535", "last_byte_only", "prefix_of_next"))


# ---- sizes ----------------------------------------------------------------------------------------------------------
def sizes() -> List[RShape]:
    out = []
    outside = _items(b"/out/", range(3))  # records outside the interval, in both
    S, E = ik(b"/s/", 0), ik(b"/s0", 0)
    for n in SIZES:
        recs = _items(b"/s/", range(n))
        out.append(RShape("all missing %d" % n, outside, outside + recs, S, E, tags=("n_%d" % n,) + ("all_missing",) * (n > 0)))
        out.append(RShape("all extra %d" % n, outside + recs, outside, S, E, tags=("span_%d" % n,) + ("all_extra",) * (n > 0)))
        out.append(RShape("identical %d" % n, outside + recs, outside + recs, S, E,
                          tags=("n_%d" % n, "span_%d" % n, "identical")))
    recs = _items(b"/s/", range(BIG), lambda i: b"b%d" % (i % 97))
    one = list(recs)
    one[BIG // 2] = (one[BIG // 2][0], b"the one diff")
    out += [RShape("all missing 1e5", [], recs, S, E, tags=("n_1e5", "all_missing"), slow=True),
            RShape("all extra 1e5", recs, [], S, E, tags=("span_1e5", "all_extra"), slow=True),
            RShape("one diff in 1e5", recs, one, S, E, tags=("n_1e5", "span_1e5", "one_in_1e5"), slow=True)]
    return out


# ---- walks ----------------------------------------------------------------------------------------------------------
def walks() -> List[RShape]:
    base = _items(b"/w/", range(60))
    eng = dict(base)
    mirror = dict(base)
    for i in (0, 6, 13, 20, 27, 34, 41, 48, 55):   # every 7th record of the engine differs: chunk 7 ends on them
        eng[base[i][0]] = b"changed %d" % i
    for i in (1, 9, 30):
        del mirror[base[i][0]]
    for i in (17, 44):
        mirror[base[i][0] + b"~"] = b"only in the snapshot"
    s, e = ik(b"/w/", 0), ik(b"/w0", 0)
    shapes = [RShape("walk 1 2 7 4096", sorted(mirror.items()), sorted(eng.items()), s, e, chunks=(1, 2, 7, 4096),
                     tags=("chunk_1", "chunk_2", "chunk_7", "chunk_4096", "chunk_end_on_diff"))]
    big = _items(b"/w/", range(10_000), lambda i: b"w%d" % (i % 13))
    be = dict(big)
    for i in range(4095, 10_000, 4096):
        be[big[i][0]] = b"diverged at a chunk end"
    shapes.append(RShape("walk 4096 over 10 000", big, sorted(be.items()), s, e, chunks=(4096,),
                         tags=("chunk_4096", "chunk_end_on_diff")))
    return shapes


# ---- interplay ------------------------------------------------------------------------------------------------------
def interplay() -> List[RShape]:
    # three versions per user key and revision records, so that a compaction sweep has victims of several classes
    mirror = []
    for u in range(300):
        uk = b"/i/%05d" % u
        mirror += [(ik(uk, r), b"val %d %d" % (u, r)) for r in (3, 4, 5)]
        mirror.append((ik(uk, 0), struct.pack(">Q", 5) + (b"\x01" if u % 10 == 0 else b"")))
    mirror.sort()
    eng = dict(mirror)
    for j, (k, _) in enumerate(mirror[::37]):
        eng[k] = b"engine %d" % j
    for k, _ in mirror[5::91]:
        del eng[k]
    eng[ik(b"/i/00042x", 4)] = b"missing from the snapshot"
    e = sorted(eng.items())
    ttl = {k: T0 + 10 for k, _ in mirror[::19]}      # some of these change (they lose the TTL), most do not
    S, E = b"", b"\xff" * 4
    out = [RShape("interplay compact stream", mirror, e, S, E, interplay="compact_stream", tags=("compact_stream",)),
           RShape("interplay range stream", mirror, e, S, E, interplay="range_stream", tags=("range_stream",)),
           RShape("interplay range stream, empty diff", mirror, mirror, S, E, interplay="range_stream",
                  tags=("range_stream", "identical")),
           RShape("interplay range batch", mirror, e, S, E, interplay="range_batch", tags=("range_batch",)),
           RShape("interplay ttl", mirror, e, S, E, ttl=ttl, interplay="ttl", tags=("ttl_changed", "ttl_unchanged"))]
    return out


def all_shapes(slow: bool = True) -> List[RShape]:
    out = edges() + [values(), keys()] + sizes() + walks() + interplay()
    return [s for s in out if slow or not s.slow]


# ---- rejections -----------------------------------------------------------------------------------------------------
def rejections() -> List[Tuple[str, str, bytes, bytes, Items]]:
    """(name, expected code name, start, end, items) of calls kb_reconcile refuses; NULL arrays are built by the test"""
    a, b, c = _k(b"/r/", 1), _k(b"/r/", 2), _k(b"/r/", 3)
    S, E = ik(b"/r/", 0), ik(b"/r0", 0)
    return [
        ("unsorted", "KB_EUNSORTED", S, E, [(b, b"x"), (a, b"x")]),
        ("duplicate", "KB_EUNSORTED", S, E, [(a, b"x"), (a, b"y")]),
        ("key below start", "KB_EINVAL", a + b"\x00", E, [(a, b"x"), (b, b"x")]),
        ("key equal to end", "KB_EINVAL", S, c, [(a, b"x"), (c, b"x")]),
        ("start == end with records", "KB_EINVAL", a, a, [(a, b"x")]),
        ("start > end with records", "KB_EINVAL", E, S, [(a, b"x")]),
        ("65 536-byte key", "KB_ELIMIT", b"", b"\xff" * 4, [(b"\x01" * 65536, b"x")]),
        ("65 536-byte start", "KB_ELIMIT", b"\x01" * 65536, b"\xff" * 4, []),
    ]


# ---- classes --------------------------------------------------------------------------------------------------------
def _size_class(prefix: str, n: int) -> Optional[str]:
    if n in SIZES:
        return "%s_%d" % (prefix, n)
    return "%s_1e5" % prefix if n >= BIG else None


def reconcile_classes(shape: RShape) -> set:
    """what a shape reaches, from the bytes and the model alone"""
    c = set()
    mirror, engine = dict(shape.mirror), dict(shape.engine)
    calls = []  # (start, end, inp) of every call
    if shape.chunks:
        for ch in shape.chunks:
            c.add("chunk_%d" % ch)
            cur = dict(mirror)
            for s, e, inp in walk(engine, shape.start, shape.end, ch):
                d = diff(cur, inp, s, e)
                if inp and e == inp[-1][0] + b"\x00" and any(k == inp[-1][0] for _, k, _ in d):
                    c.add("chunk_end_on_diff")
                for k, v in ops_of(d, inp):
                    cur.pop(k) if v is None else cur.__setitem__(k, v)
                calls.append((s, e, inp, d))
            assert interval_items(cur, shape.start, shape.end) == interval_items(engine, shape.start, shape.end)
    else:
        inp = interval_items(engine, shape.start, shape.end)
        calls.append((shape.start, shape.end, inp, diff(mirror, inp, shape.start, shape.end)))
    s, e = shape.start, shape.end
    both = sorted(set(mirror) | set(engine))
    if s in both:
        c.add("key_eq_start")
    if e in both:
        c.add("key_eq_end")
    if any(not (s <= k < e) and mirror.get(k) != engine.get(k) for k in both):
        c.add("outside_divergent")
    inside = [k for k in both if s <= k < e]
    for _, _, inp, d in calls[:1] if not shape.chunks else []:
        dk = {k for _, k, _ in d}
        if inside and inside[0] in dk:
            c.add("diff_first")
        if inside and inside[-1] in dk:
            c.add("diff_last")
    span = len([k for k in mirror if s <= k < e])
    n = len([k for k in engine if s <= k < e])
    for name in (_size_class("n", n), _size_class("span", span)):
        if name and not shape.chunks:
            c.add(name)
    d_all = [x for call in calls for x in call[3]]
    if not shape.chunks:
        if n and all(kind == MISSING for kind, _, _ in d_all) and len(d_all) == n:
            c.add("all_missing")
        if span and all(kind == EXTRA for kind, _, _ in d_all) and len(d_all) == span:
            c.add("all_extra")
        if not d_all:
            c.add("identical")
        if len(d_all) == 1 and n >= BIG:
            c.add("one_in_1e5")
    for kind, k, _ in d_all:
        if len(k) in (1, 15, 16, 17, 65535):
            c.add("klen_%d" % len(k))
        if kind != CHANGED:
            continue
        a, b = mirror[k], engine[k]
        if len(a) == len(b):
            at = next(i for i in range(len(a)) if a[i] != b[i])
            if len(a) == 4096:
                c.add("byte_last" if at == len(a) - 1 else "byte_%d" % at)
        elif abs(len(a) - len(b)) == 1 and pad16(a) == pad16(b):
            c.add("len_pm1_equal_pad")
        if {a, b} == {b"", b"\x00"}:
            c.add("empty_vs_nul")
        if b"tombstone" in (a, b):
            c.add("tombstone")
        if {len(a), len(b)} == {8, 9}:
            c.add("rev8_vs_9")
    dks = {k for _, k, _ in d_all}
    for x, y in zip(both, both[1:]):  # neighbours, one of them a diff
        if x not in dks and y not in dks:
            continue
        if len(x) == len(y) and x[:-1] == y[:-1]:
            c.add("last_byte_only")
        if y.startswith(x):
            c.add("prefix_of_next")
    if shape.interplay and shape.interplay != "ttl":
        c.add(shape.interplay)
    if shape.ttl:
        if any(k in dks for k in shape.ttl):
            c.add("ttl_changed")
        if any(k not in dks for k in shape.ttl):
            c.add("ttl_unchanged")
    return c


if __name__ == "__main__":
    for sh in all_shapes():
        print("%-36s mirror %6d engine %6d  %s" % (sh.name, len(sh.mirror), len(sh.engine),
                                                   " ".join(sorted(reconcile_classes(sh)))))
