"""Stores and sweeps built so that the compaction sweep and the compaction stream's capture (kubebrain_b200/csrc:
kb_decode.cuh k_decode_lcp's sweep flags, kb_scan.cu k_emit<true> / k_tile_scan / k_place_victims, k_victim_capture /
k_victim_jobs) meet their fixed boundaries on purpose (shared by the CPU and GPU tests).
  K1  classes and their order within one record's turn: superseded only, tombstone only, superseded + tombstone, a
      deleted-flag revision record, the `tombstone`-valued revision record below, at and above the revision its first
      8 bytes spell, TTL revision records and objects; bounds inside one object's versions, between a revision record
      and its first version, start == end; a store with no victim and one where every record is one;
  K2  slots and tiles: tiles whose records all make 0, 1 or 2 delete calls at their turn and tiles whose count changes
      exactly at the seam, one object of N tombstone versions (2N - 1 calls for N records), a store where every record
      makes 2 calls (exactly the victim buffer's 2N), one sweep of 1.1 M records across k_tile_scan's chunk of 1 024
      tiles, started 0, 1, 255, 256 and 1 023 records in;
  K3  revision and TTL comparisons at -1, equal and +1 of revisions 1, 2, 1 000, 2^63 - 1 .. 2^63 + 1, 2^64 - 2 and
      2^64 - 1 (sweep revision 0 included): the Q5 test, 7- to 10-byte revision-record values, the TTL timeout for
      objects and revision records, the timeout above the sweep revision, expired runs in front of live versions and
      expired runs that end on a tile seam;
  K4  capture and pages: streams of 1 to 70 000 victims (up to 69 capture tiles), keys of 13 .. 65 535 bytes and guards
      of 8 .. 2^20 bytes at every pad16 edge;
  K5  past 4 GiB: 4 100 class-4 victims of exactly 2^20 bytes each (victim 4 096 starts at 2^32) and of 2^20 + 16
      (victim 4 095's guard straddles it).
`compact_classes` derives from the store bytes and the oracle alone (never from the builders' bookkeeping) what each
shape reaches, so that tests/test_compact_shapes.py can assert it on any host; `python -m tests.compact_shapes` prints
it."""
from __future__ import annotations

import struct
from typing import Dict, List, Sequence, Tuple

import numpy as np

from kubebrain_b200.packed import PackedStore, Slab
from tests import pyref

MAGIC = b"\x57\xfb\x80\x8b"
TOMB = b"tombstone"
ALL = 2**64 - 1
T_TOMB = int.from_bytes(TOMB[:8], "big")  # 0x746f6d6273746f6e: the revision a `tombstone` revision record spells

# restated from kubebrain_b200/csrc -- keep in step with it:
TILE = 1024            # k_decode_lcp / k_emit / k_place_victims: records per tile
SCAN_CHUNK = 1024      # k_tile_scan: tiles per CTA; a sweep crosses a chunk above TILE * SCAN_CHUNK records
CAPTURE_TILE = 1024    # k_victim_capture: victims per tile
LOOKBACK = 32          # k_victim_capture: tile states warp 0 reads per look-back step
CHUNK = 16             # keys and guards on 16-byte boundaries in a page's arena
LINE = 2**32


def ik(uk: bytes, rev: int) -> bytes:
    return MAGIC + uk + b"$" + struct.pack(">Q", rev)


def be(rev: int) -> bytes:
    return struct.pack(">Q", rev)


def pad16(n: int) -> int:
    return (n + CHUNK - 1) & ~(CHUNK - 1)


def store_of(items) -> PackedStore:
    return PackedStore.from_items(list(dict(items).items()))


def concat(*stores: PackedStore) -> PackedStore:
    """stores whose key ranges follow each other, as one store"""
    def cat(slabs: Sequence[Slab]) -> Slab:
        offs, base = [np.zeros(1, np.uint64)], np.uint64(0)
        for s in slabs:
            offs.append(s.off[1:] + base)
            base = base + s.off[-1]
        return Slab(np.concatenate([s.data for s in slabs]), np.concatenate(offs))
    for a, b in zip(stores, stores[1:]):
        assert a.keys[a.n - 1] < b.keys[0]
    return PackedStore(cat([s.keys for s in stores]), cat([s.vals for s in stores]))


def _ranges(starts: np.ndarray, lens: np.ndarray) -> np.ndarray:
    """the byte indices of the concatenated ranges [starts[i], starts[i] + lens[i])"""
    lens = lens.astype(np.int64)
    tot = int(lens.sum())
    if tot == 0:
        return np.zeros(0, np.int64)
    base = np.repeat(starts.astype(np.int64) - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens)
    return base + np.arange(tot, dtype=np.int64)


V_FILL, V_REV, V_TOMB = 0, 1, 2   # value kinds of vec_store


def vec_store(head: bytes, obj: np.ndarray, rev: np.ndarray, vlen: np.ndarray, vkind: np.ndarray,
              vrev: np.ndarray = None, extra: np.ndarray = None) -> PackedStore:
    """records built without a Python loop: key i = magic + head + obj[i] in 8 decimal digits + 'k' x extra[i] + '$' +
    rev[i]; value i = vlen[i] bytes of (i % 251) + 1, or the same with its first 8 bytes the revision vrev[i] (V_REV),
    or `tombstone` (V_TOMB).  obj ascending with the records of one object in ascending rev make the keys ascending."""
    n = len(obj)
    obj = obj.astype(np.int64)
    rev = rev.astype(np.uint64)
    extra = np.zeros(n, np.int64) if extra is None else extra.astype(np.int64)
    h = MAGIC + head
    klen = len(h) + 8 + extra + 9
    koff = np.zeros(n + 1, np.uint64)
    np.cumsum(klen, out=koff[1:])
    k0 = koff[:-1].astype(np.int64)
    kd = np.empty(int(koff[-1]), np.uint8)
    for j, c in enumerate(h):
        kd[k0 + j] = c
    for j in range(8):
        kd[k0 + len(h) + j] = (obj // 10 ** (7 - j)) % 10 + 48
    if extra.any():
        kd[_ranges(k0 + len(h) + 8, extra)] = ord("k")
    tail = k0 + klen - 9
    kd[tail] = ord("$")
    for j in range(8):
        kd[tail + 1 + j] = ((rev >> np.uint64(56 - 8 * j)) & np.uint64(0xFF)).astype(np.uint8)
    vlen = vlen.astype(np.int64)
    voff = np.zeros(n + 1, np.uint64)
    np.cumsum(vlen, out=voff[1:])
    v0 = voff[:-1].astype(np.int64)
    vd = np.repeat((np.arange(n) % 251 + 1).astype(np.uint8), vlen)
    r = np.nonzero(vkind == V_REV)[0]
    if len(r):
        assert (vlen[r] >= 8).all()
        vr = vrev[r].astype(np.uint64)
        for j in range(8):
            vd[v0[r] + j] = ((vr >> np.uint64(56 - 8 * j)) & np.uint64(0xFF)).astype(np.uint8)
    t = np.nonzero(vkind == V_TOMB)[0]
    if len(t):
        assert (vlen[t] == 9).all()
        for j, c in enumerate(TOMB):
            vd[v0[t] + j] = c
    return PackedStore(Slab(kd, koff), Slab(vd, voff))


# ---- K1: classes and their order within a record -----------------------------------------------------------------
K1_REV = 100
K1_TIMEOUT = 50
K1_TOMB_REVS = (T_TOMB - 1, T_TOMB, T_TOMB + 1)


def k1_store() -> PackedStore:
    v = b"value"
    items = {
        ik(b"/k1/a-sup", 10): v, ik(b"/k1/a-sup", 20): v,                       # 10 superseded at 20's turn
        ik(b"/k1/b-tomb", 10): TOMB,                                             # tombstone only
        ik(b"/k1/c-suptomb", 10): v, ik(b"/k1/c-suptomb", 20): TOMB,             # 20's turn: [1 (10)] [2 (20)]
        ik(b"/k1/d-revdel", 0): be(30) + b"\x01", ik(b"/k1/d-revdel", 10): v, ik(b"/k1/d-revdel", 30): TOMB,
        ik(b"/k1/e-tombrev", 0): TOMB, ik(b"/k1/e-tombrev", 10): v,              # 2, then 3 or the Q5 skip
        ik(b"/k1/e-tombrev2", 0): TOMB,
        ik(b"/k1/f/events/rr", 0): be(40), ik(b"/k1/f/events/rr", 40): v,        # TTL revision record
        ik(b"/k1/g/events/obj", 30): v, ik(b"/k1/g/events/obj", 60): v,          # TTL object, then a live one
        ik(b"/k1/h-live", 0): be(70), ik(b"/k1/h-live", 70): v,
    }
    for r in range(10, 60, 10):                                                  # bounds inside its versions
        items[ik(b"/k1/i-many", r)] = v if r != 40 else TOMB
    return store_of(items)


def k1_sweeps() -> List[Tuple[bytes, bytes, int, int, bool]]:
    """(start, end, rev, timeout_rev, support_ttl)"""
    s, e = MAGIC, b"\xff"
    out = [(s, e, K1_REV, 0, True), (s, e, K1_REV, K1_TIMEOUT, False), (s, e, K1_REV, K1_TIMEOUT, True)]
    out += [(s, e, r, 0, True) for r in K1_TOMB_REVS]
    out += [(ik(b"/k1/i-many", 15), ik(b"/k1/i-many", 45), K1_REV, 0, True),     # inside one object's versions
            (ik(b"/k1/d-revdel", 1), e, K1_REV, 0, True),                        # after a revision record
            (ik(b"/k1/d-revdel", 0), ik(b"/k1/d-revdel", 1), K1_REV, 0, True),   # the revision record alone
            (ik(b"/k1/a-sup", 20), ik(b"/k1/a-sup", 20), K1_REV, 0, True)]       # start == end
    return out


def k1_none_store() -> PackedStore:
    """nothing is a victim: an 8-byte revision record and one live version per object"""
    items = {}
    for i in range(300):
        uk = b"/k1/none/%04d" % i
        items[ik(uk, 0)] = be(5 + i)
        items[ik(uk, 5 + i)] = b"v%d" % i
    return store_of(items)


def k1_every_store() -> PackedStore:
    """every record is a victim: a deleted-flag revision record, a superseded version and a tombstone per object"""
    items = {}
    for i in range(300):
        uk = b"/k1/every/%04d" % i
        items[ik(uk, 0)] = be(7 + i) + b"\x01"
        items[ik(uk, 5 + i)] = b"v%d" % i
        items[ik(uk, 7 + i)] = TOMB
    return store_of(items)


# ---- K2: slots and tiles ---------------------------------------------------------------------------------------------
# object types: the delete calls each of its records makes at its turn in a plain sweep at revision ALL
OBJ_RECORDS = {"Z": (0,), "O": (1,), "W": (2,), "S": (0, 1), "D": (1, 2)}
K2_SEGMENTS = "ZOWZWOZ"       # tiles of one type each: every change 0->1->2->0->2->1->0 falls on a seam
K2_STARTS = (0, 1, 255, 256, 1023)
K2_CHAIN_N = (1, 2, 1024, 1025, 300_000)
K2_FULL_N = (1024, 1025)
K2_BIG_N = 1_100_000
K2_BIG_PATTERN = "SOWDZSW"    # 10 records, dense calls everywhere


def typed_store(head: bytes, types: Sequence[str]) -> PackedStore:
    """one object per type: Z a live version, O a tombstone, W a `tombstone` revision record, S two live versions,
    D two tombstone versions"""
    codes = np.frombuffer("".join(types).encode(), np.uint8)
    nrec = np.where((codes == ord("S")) | (codes == ord("D")), 2, 1)
    obj = np.repeat(np.arange(len(codes)), nrec)
    first = np.concatenate([[0], np.cumsum(nrec)[:-1]])
    second = np.zeros(len(obj), bool)
    second[first[nrec == 2] + 1] = True
    c = codes[obj]
    rev = np.where(c == ord("W"), 0, np.where(second, 2, 1)).astype(np.uint64)
    tomb = (c == ord("O")) | (c == ord("W")) | (c == ord("D"))
    vlen = np.where(tomb, 9, 6)
    return vec_store(head, obj, rev, vlen, np.where(tomb, V_TOMB, V_FILL))


def k2_tiles_store() -> PackedStore:
    """tiles of 1 024 records of one type each, a D tile (1, 2, 1, 2 ..), a tile that is one chain of tombstone versions,
    and an S object across a seam"""
    types = []
    for t in K2_SEGMENTS:
        types += [t] * TILE
    types += ["D"] * (TILE // 2)
    types += ["Z"] * (TILE - 1) + ["S"] + ["O"] * (TILE - 1)
    a = typed_store(b"/k2/t/", types)
    b = chain_store(TILE, head=b"/k2/u/")
    c = typed_store(b"/k2/v/", ["W"] * TILE)
    return concat(a, b, c)


def chain_store(n: int, head: bytes = b"/k2/c/") -> PackedStore:
    """one object of n tombstone versions: each is superseded by the next and is itself a tombstone -- 2n - 1 calls"""
    return vec_store(head, np.zeros(n, np.int64), np.arange(1, n + 1, dtype=np.uint64), np.full(n, 9),
                     np.full(n, V_TOMB))


def full_store(n: int) -> PackedStore:
    """n `tombstone` revision records: 2 calls each at a sweep revision >= T_TOMB, exactly 2n"""
    return typed_store(b"/k2/w/", ["W"] * n)


def big_store(n: int = K2_BIG_N) -> PackedStore:
    reps = -(-n // 10)
    st = typed_store(b"/k2/b/", list(K2_BIG_PATTERN) * reps)
    assert st.n == 10 * reps
    return st


# ---- K3: revision and TTL comparisons --------------------------------------------------------------------------------
K3_ANCHORS = (1, 2, 1000, 2**63 - 1, 2**63, 2**63 + 1, 2**64 - 2, 2**64 - 1)
K3_TTL_END = MAGIC + b"/z"   # the 7-byte `/events/` revision records live behind it (the oracle errors on them in TTL
                             # sweeps, as Go would panic)
K3_SEAM_RUNS = (1023, 1024, 1025, 2049)


def near(a: int) -> List[int]:
    return [r for r in (a - 1, a, a + 1) if 0 <= r <= ALL]


def k3_store() -> PackedStore:
    items: Dict[bytes, bytes] = {}
    for a in K3_ANCHORS:
        h = b"/k3/%016x/" % a
        for d, r in enumerate(near(a)):
            items[ik(h + b"q5/%d" % d, 0)] = be(r) + b"\x00"              # Q5 against the sweep revision
            items[ik(h + b"q5/%d" % d, 1)] = b"q5 version"
            items[ik(h + b"events/rr8/%d" % d, 0)] = be(r)                # TTL revision records, VL8 without VL9
            items[ik(h + b"events/rr9/%d" % d, 0)] = be(r) + b"\x02"      # VL8 and VL9: TTL and Q5
            items[ik(h + b"events/rr10/%d" % d, 0)] = be(r) + b"\x02\x03"
        for r in near(a):                                                 # TTL objects; expired in front of live
            if r:
                items[ik(h + b"events/obj", r)] = b"o%x" % r
        for ln in (7, 8, 9, 10):                                          # value lengths around VL8 / VL9
            items[ik(h + b"vl/%02d" % ln, 0)] = (be(a) + b"\x04\x05")[:ln]
        if a:
            items[ik(h + b"live", a)] = b"live"
    items[ik(b"/k3/tombrev", 0)] = TOMB
    items[ik(b"/k3/tombrev", 3)] = b"after"
    for j, ln in enumerate((0, 3, 7)):                                    # `/events/` with short revision-record values
        items[ik(b"/z/events/short/%d" % j, 0)] = be(5)[:ln]
        items[ik(b"/z/events/short/%d" % j, 5)] = b"s"
    return store_of(items)


def k3_sweeps() -> List[Tuple[bytes, bytes, int, int, bool]]:
    out = []
    for a in K3_ANCHORS:
        for r in near(a):
            out += [(MAGIC, b"\xff", r, 0, True), (MAGIC, b"\xff", r, 0, False)]
            for t in near(a):
                if t:
                    out += [(MAGIC, K3_TTL_END, r, t, False), (MAGIC, b"\xff", r, t, True)]
    for r in (T_TOMB - 1, T_TOMB, T_TOMB + 1):
        out.append((MAGIC, b"\xff", r, 0, True))
    return sorted(set(out))


def k3_seam_store() -> PackedStore:
    """expired `/events/` runs of K3_SEAM_RUNS versions, each followed by two live versions; run j starts right after a
    tile seam when the sweep starts at the store's first record (a lone live object in front of each run pads to it)"""
    items: Dict[bytes, bytes] = {}
    pos = 0
    for j, run in enumerate(K3_SEAM_RUNS):
        pad = (-pos - run - 1) % TILE   # so that the run's last record is the last of a tile
        for i in range(pad + 1):
            items[ik(b"/k3s/%d/a/%05d" % (j, i), 7)] = b"pad"
        uk = b"/k3s/%d/events/run" % j
        for r in range(1, run + 1):
            items[ik(uk, r)] = b"e"
        items[ik(uk, 5000)] = b"live"
        items[ik(uk, 5001)] = b"live2"
        pos += pad + 1 + run + 2
    return store_of(items)


K3_SEAM_TIMEOUT = 4000


# ---- K4: capture and pages -------------------------------------------------------------------------------------------
K4_COUNTS = (1, 1023, 1024, 1025, 32768, 32769, 33793, 70000)
K4_KEY_LENS = (13, 16, 17, 31, 32, 33, 65535)
K4_GUARD_LENS = (8, 9, 15, 16, 17, 2**20)
K4_GROUPS = (1, 7, 1024)
K4_REV, K4_TIMEOUT = 100, 50


def k4_count_store(n: int = max(K4_COUNTS)) -> PackedStore:
    """n objects of two versions each (the older one is a victim), keys of 25 .. 65 bytes (every pad16 edge)"""
    obj = np.repeat(np.arange(n), 2)
    rev = np.tile(np.array([1, 2], np.uint64), n)
    extra = (obj * 7) % 41
    return vec_store(b"/k4/", obj, rev, np.full(2 * n, 6), np.full(2 * n, V_FILL), extra=extra)


def k4_count_end(store: PackedStore, v: int) -> bytes:
    """the end bound of a sweep whose victims are the first v objects' older versions"""
    return store.keys[2 * v] if 2 * v < store.n else b"\xff"


def k4_entry_store() -> PackedStore:
    """victims with keys of every K4_KEY_LENS (class 1), guards of every K4_GUARD_LENS (class 4; 9 also class 3), and a
    65 535-byte key with a 2^20-byte guard"""
    items: Dict[bytes, bytes] = {}
    for kl in K4_KEY_LENS:
        uk = b"" if kl == 13 else (b"/k4e/%05d/" % kl + b"x" * kl)[: kl - 13]
        items[ik(uk, 1)] = b"old"
        items[ik(uk, 2)] = b"new"
    for gl in K4_GUARD_LENS:
        uk = b"/k4g/events/%07d" % gl
        items[ik(uk, 0)] = (be(10) + bytes(range(1, 256)) * (gl // 255 + 1))[:gl]
        items[ik(uk, 10)] = b"v"
    for gl in (9,):
        items[ik(b"/k4g/revdel/%d" % gl, 0)] = be(20) + b"\x01"
        items[ik(b"/k4g/revdel/%d" % gl, 20)] = b"v"
    big = b"/k4h/events/" + b"y" * (65535 - 13 - 12)
    items[ik(big, 0)] = be(30) + b"\x07" * (2**20 - 8)
    items[ik(big, 30)] = TOMB
    return store_of(items)


def k4_entry_sweeps() -> List[Tuple[bytes, bytes, int, int, bool]]:
    return [(MAGIC, b"\xff", K4_REV, 0, True), (MAGIC, b"\xff", K4_REV, K4_TIMEOUT, False)]


# ---- K5: past 4 GiB --------------------------------------------------------------------------------------------------
K5_N = 4100
K5_KEY = 25                     # ik(b"/events/%04d", 0)
K5_GUARD_EXACT = 2**20 - 32     # entry of exactly 2^20: victim 4 096 starts at 2^32
K5_GUARD_STRADDLE = 2**20 - 16  # entry of 2^20 + 16: victim 4 095's guard straddles 2^32
K5_VREV, K5_TIMEOUT, K5_REV = 5, 10, 100
K5_PAGE = 256 << 20


def k5_key(i: int) -> bytes:
    return ik(b"/events/%04d" % i, 0)


def k5_store(glen: int, n: int = K5_N) -> PackedStore:
    """n `/events/` revision records with glen-byte values: the revision K5_VREV, then the record's number in 4 bytes,
    0x5a, zeros, and 0xa5 last, so that a shifted or truncated copy shows"""
    keys = Slab.from_list([k5_key(i) for i in range(n)])
    data = np.zeros(n * glen, np.uint8)
    starts = np.arange(n, dtype=np.int64) * glen
    for j, c in enumerate(be(K5_VREV)):
        data[starts + j] = c
    for b in range(4):
        data[starts + 8 + b] = (np.arange(n) >> (8 * b)) & 0xFF
    data[starts + 12] = 0x5A
    data[starts + glen - 1] = 0xA5
    return PackedStore(keys, Slab(data, np.arange(n + 1, dtype=np.uint64) * np.uint64(glen)))


def k5_guard(i: int, glen: int) -> np.ndarray:
    g = np.zeros(glen, np.uint8)
    g[:8] = np.frombuffer(be(K5_VREV), np.uint8)
    g[8:12] = np.frombuffer(struct.pack("<I", i), np.uint8)
    g[12] = 0x5A
    g[glen - 1] = 0xA5
    return g


def k5_layout(glen: int, n: int = K5_N) -> Dict[str, object]:
    unit = pad16(K5_KEY) + pad16(glen)
    k = LINE // unit
    starts_at = LINE % unit == 0
    guard_straddles = not starts_at and k * unit + pad16(K5_KEY) < LINE
    return dict(unit=unit, total=n * unit, past=n * unit > LINE, starts_at_line=starts_at and k < n,
                guard_straddles=guard_straddles and k < n, entry_at_line=k)


# ---- classes -----------------------------------------------------------------------------------------------------------
def _facts(store: PackedStore):
    """per record: decodes, revision, user key contains `/events/`"""
    ok, rev, ev = [], [], []
    for k in store.keys.tolist():
        try:
            uk, r = pyref.decode(k)
            ok.append(True), rev.append(r), ev.append(b"/events/" in uk)
        except pyref.DecodeError:
            ok.append(False), rev.append(0), ev.append(False)
    return np.array(ok, bool), np.array(rev, np.uint64), np.array(ev, bool)


def turn_calls(store: PackedStore, facts, lo: int, hi: int, x, rev: int, timeout_rev: int, support_ttl: bool):
    """the record at whose turn each of the oracle's delete calls x is made, and its class, over [lo, hi): a superseded
    victim is called at the turn of the next record that takes part (decodes, is not expired, revision <= rev); every
    other class at its own"""
    ok, rv, ev = facts
    vals = store.vals
    ttl = not support_ttl and timeout_rev != 0
    part = ok[lo:hi] & (rv[lo:hi] <= np.uint64(rev))
    if ttl:
        for i in np.nonzero(ev[lo:hi] & ok[lo:hi])[0]:
            j = lo + int(i)
            if rv[j] == 0:
                v = vals[j]
                if len(v) >= 8 and int.from_bytes(v[:8], "big") <= timeout_rev:
                    part[i] = False
            elif int(rv[j]) <= timeout_rev:
                part[i] = False
    takes = np.nonzero(part)[0] + lo
    vic, cls = x.victims.astype(np.int64), x.vclass.astype(np.int64)
    sup = cls == 1
    turn = vic.copy()
    if sup.any():
        turn[sup] = takes[np.searchsorted(takes, vic[sup], side="right")]
    return turn, cls


def sweep_classes(store: PackedStore, facts, st, s: bytes, e: bytes, rev: int, timeout_rev: int, support_ttl: bool,
                  ko) -> Dict[str, object]:
    x = ko.worker_run(st, s, e, rev, compact=True, timeout_rev=timeout_rev, support_ttl=support_ttl, collect=True)
    assert x.rc == 0, (s[:20], e[:20], rev, timeout_rev, support_ttl)
    lo, hi = st.lower_bound(s), max(st.lower_bound(e), st.lower_bound(s))
    n = hi - lo
    turn, cls = turn_calls(store, facts, lo, hi, x, rev, timeout_rev, support_ttl)
    per = np.bincount(turn - lo, minlength=n) if n else np.zeros(0, np.int64)
    combos = set()
    if len(turn):
        cut = np.nonzero(np.diff(turn))[0] + 1
        for g in np.split(cls, cut):
            combos.add(tuple(int(c) for c in g))
    c: Dict[str, object] = dict(n=n, victims=len(x.victims), classes=set(int(v) for v in np.unique(cls)),
                                combos=combos, max_per_record=int(per.max()) if n else 0, start=lo)
    ntiles = -(-n // TILE)
    if n:
        tiles = np.zeros(ntiles * TILE, np.int64) - 1
        tiles[:n] = per
        tiles = tiles.reshape(ntiles, TILE)
        uniform = [int(t[0]) if (t[t >= 0] == t[0]).all() else None for t in tiles]
        c["uniform_tiles"] = set(u for u in uniform if u is not None)
        c["seam_changes"] = set((a, b) for a, b in zip(uniform, uniform[1:]) if a is not None and b is not None and a != b)
        c["chunks"] = -(-ntiles // SCAN_CHUNK)
        if ntiles > SCAN_CHUNK:
            c["calls_around_chunk_seam"] = (int(per[(SCAN_CHUNK - 1) * TILE: SCAN_CHUNK * TILE].sum()),
                                            int(per[SCAN_CHUNK * TILE: (SCAN_CHUNK + 1) * TILE].sum()))
    return c


def k3_comparisons(store: PackedStore, facts, sweeps, ko) -> Dict[str, object]:
    """which comparisons of k_decode_lcp each K3 sweep puts at -1 / 0 / +1: Q5 (9-byte revision-record value against the
    sweep revision), TTL objects and TTL revision records (against the timeout), with the oracle's class for each"""
    ok, rv, ev = facts
    keys, vals = store.keys.tolist(), store.vals.tolist()
    st = ko.OracleStore(store)
    c: Dict[str, object] = dict(q5=set(), ttl_obj=set(), ttl_rev=set(), vl=set(), timeout_above_rev=False,
                                ttl_off_with_timeout=False, no_ttl_zero_timeout=False, sweep_revs=set(),
                                expired_before_live=False, short_events_plain=False, tombrev=set())
    for s, e, rev, trev, sttl in sweeps:
        x = ko.worker_run(st, s, e, rev, compact=True, timeout_rev=trev, support_ttl=sttl, collect=True)
        assert x.rc == 0
        got = {}
        for i, cl in zip(x.victims.tolist(), x.vclass.tolist()):
            got.setdefault(int(i), []).append(int(cl))
        ttl = not sttl and trev != 0
        c["sweep_revs"].add(rev)
        c["timeout_above_rev"] |= ttl and trev > rev
        c["ttl_off_with_timeout"] |= sttl and trev != 0
        c["no_ttl_zero_timeout"] |= not sttl and trev == 0
        lo, hi = st.lower_bound(s), st.lower_bound(e)
        for i in range(lo, hi):
            if not ok[i]:
                continue
            k, v = keys[i], vals[i]
            mine = tuple(got.get(i, []))
            if rv[i] == 0 and len(v) == 9 and not (ttl and ev[i]):
                d = int.from_bytes(v[:8], "big") - rev
                if abs(d) <= 1:
                    c["q5"].add((d, 3 in mine))
                if v == TOMB:
                    c["tombrev"].add((d if abs(d) <= 1 else "far", mine))
            if rv[i] == 0:
                c["vl"].add((len(v), bool(ev[i]), ttl))
                c["short_events_plain"] |= bool(ev[i]) and len(v) < 8 and not ttl
            if ttl and ev[i]:
                if rv[i] == 0 and len(v) >= 8:
                    d = int.from_bytes(v[:8], "big") - trev
                    if abs(d) <= 1:
                        c["ttl_rev"].add((d, 4 in mine))
                elif rv[i] != 0:
                    d = int(rv[i]) - trev
                    if abs(d) <= 1:
                        c["ttl_obj"].add((d, 5 in mine))
                    if d > 0 and int(rv[i]) <= rev and i > lo and rv[i - 1] != 0 and 5 in got.get(i - 1, []) \
                            and keys[i - 1][:-8] == k[:-8]:
                        c["expired_before_live"] = True
    return c


def seam_classes(store: PackedStore, facts, ko) -> Dict[str, object]:
    """where the expired runs of k3_seam_store end against the tiles of a TTL sweep from its first record"""
    x = ko.worker_run(ko.OracleStore(store), MAGIC, b"\xff", ALL - 1, compact=True, timeout_rev=K3_SEAM_TIMEOUT,
                      support_ttl=False, collect=True)
    assert x.rc == 0
    ok, rv, ev = facts
    v5 = set(int(i) for i, c in zip(x.victims, x.vclass) if c == 5)
    ends = set()
    for i in v5:
        if i + 1 < store.n and i + 1 not in v5 and ev[i + 1] and rv[i + 1] > K3_SEAM_TIMEOUT:
            ends.add(i % TILE)
    return dict(run_end_in_tile=ends, expired=len(v5), superseded_after=int((x.vclass == 1).sum()))


def capture_classes(sizes: Sequence[int]) -> Dict[str, object]:
    """a stream's victims against k_victim_capture's tiles"""
    n = len(sizes)
    return dict(n=n, tiles=-(-n // CAPTURE_TILE), lookback_steps=-(-(-(-n // CAPTURE_TILE) - 1) // LOOKBACK) if n else 0,
                total=int(np.sum(np.asarray(sizes, np.int64))) if n else 0)


def entry_classes(store: PackedStore, x) -> Dict[str, object]:
    keys = [len(store.keys[int(i)]) for i in x.victims]
    guards = [len(store.vals[int(i)]) for i, c in zip(x.victims, x.vclass) if c in (3, 4)]
    return dict(key_lens=set(keys), guard_lens=set(guards), classes=set(int(c) for c in x.vclass))


def compact_classes(big: bool = True) -> Dict[str, Dict[str, object]]:
    """every shape's classes (K5 by its layout alone; without `big`, the 1.1 M and 300 000 stores are left out)"""
    from oracle import binding as ko

    out: Dict[str, Dict[str, object]] = {}

    def sweeps(name, store, sw):
        f = _facts(store)
        st = ko.OracleStore(store)
        for s, e, rev, trev, sttl in sw:
            out["%s %s..%s rev=%x t=%x ttl=%d" % (name, s[4:40], e[4:40], rev, trev, sttl)] = \
                sweep_classes(store, f, st, s, e, rev, trev, sttl, ko)

    sweeps("K1", k1_store(), k1_sweeps())
    sweeps("K1 none", k1_none_store(), [(MAGIC, b"\xff", ALL, 0, True)])
    sweeps("K1 every", k1_every_store(), [(MAGIC, b"\xff", ALL, 0, True)])
    t = k2_tiles_store()
    sweeps("K2 tiles", t, [(t.keys[j], b"\xff", ALL, 0, True) for j in K2_STARTS])
    for n in K2_CHAIN_N if big else K2_CHAIN_N[:-1]:
        sweeps("K2 chain %d" % n, chain_store(n), [(MAGIC, b"\xff", ALL, 0, True)])
    for n in K2_FULL_N:
        sweeps("K2 full %d" % n, full_store(n), [(MAGIC, b"\xff", ALL, 0, True)])
    if big:
        b = big_store()
        sweeps("K2 big", b, [(b.keys[j], b"\xff", ALL, 0, True) for j in K2_STARTS])
    k3 = k3_store()
    out["K3"] = k3_comparisons(k3, _facts(k3), k3_sweeps(), ko)
    s3 = k3_seam_store()
    out["K3 seam"] = seam_classes(s3, _facts(s3), ko)
    c4 = k4_count_store()
    st4 = ko.OracleStore(c4)
    for v in K4_COUNTS:
        x = ko.worker_run(st4, MAGIC, k4_count_end(c4, v), ALL, compact=True, collect=True)
        sizes = [pad16(len(c4.keys[int(i)])) for i in x.victims]
        out["K4 count %d" % v] = dict(capture_classes(sizes), key_pad=set(len(c4.keys[int(i)]) % 16 for i in x.victims[:64]))
    e4 = k4_entry_store()
    st = ko.OracleStore(e4)
    for s, e, rev, trev, sttl in k4_entry_sweeps():
        x = ko.worker_run(st, s, e, rev, compact=True, timeout_rev=trev, support_ttl=sttl, collect=True)
        out["K4 entries t=%d" % trev] = entry_classes(e4, x)
    out["K5 exact"] = k5_layout(K5_GUARD_EXACT)
    out["K5 straddle"] = k5_layout(K5_GUARD_STRADDLE)
    return out


if __name__ == "__main__":  # prints the classes every shape reaches
    for name, c in compact_classes().items():
        print(name)
        for k in sorted(c):
            v = c[k]
            if isinstance(v, (set, list)):
                v = sorted(v, key=repr)
                if len(v) > 24:
                    v = v[:24] + ["..."]
            if v not in (False, [], None):
                print("    %-24s %s" % (k, v))
