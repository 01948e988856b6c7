"""Range-scan stores and request batches built so that the scan kernels' fixed boundaries fall on purpose (shared by the
CPU and GPU tests).

The range path (kubebrain_b200/csrc/kb_scan.cu, kb_copy.cu, kb_decode.cuh, kb_wire.cuh) branches on boundaries a fuzz store is too
small to reach and a regular synthetic too uniform to reach:
  R1  tile seams: runs of records that are not PREVOK (they cannot become the loop's `prev`) ending exactly at a tile
      seam, of lengths on both sides of k_emit's 256-record carry window and over more than 32 tiles (one look-back
      step), followed by the same key, a key only the running LCP minimum tells apart, a tombstone or a revision record;
  R2  limit probe windows: sparse visibility, so that a limited request settles in probe round 0, 1 or 2, or is reached
      only by a window's trailing emission;
  R3  pair sizes: emitted pairs on both sides of k_gather's 160-chunk round, the largest key, empty and 1 MiB values,
      requests of 1, 31, 32, 33, 64 and 65 kvs, and wire elements on both sides of k_wire_copy's ring room.
`range_classes` derives from the store bytes and the oracle alone (never from the builders' bookkeeping) what a batch
reaches, so that tests/test_range_shapes.py can assert it on any host; `python -m tests.range_shapes` prints it."""
from __future__ import annotations

import random
import struct
from collections import Counter
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from kubebrain_b200.packed import PackedStore
from oracle import binding as ko

MAGIC = b"\x57\xfb\x80\x8b"
TOMB = b"tombstone"

# restated from csrc/ -- keep in step with it:
TILE = 1024           # KB_TILE: records per tile, counted from each request's first record
CARRY = 256           # k_emit: meta words in front of a tile looked at before the decoupled look-back
LOOKBACK = 32         # k_emit: tile states per look-back step
SCAN_CHUNK = 1024     # k_tile_scan: tiles per CTA
WINDOW_MIN = 8192     # KB_LIMIT_WINDOW_MIN; the first window is max(8192, 8 limit) rounded up to a tile, then x8
GATHER_ROUND = 160    # k_gather: 32 lanes x GATHER_U chunks per round
GATHER_BLOCK = 32     # k_gather: jobs per block
LCP_INF = 0xFFFF      # KB_LCP_INF

READ = 1000           # read revision of every R1 / R2 request, and the sweep revision on R1
TTL = 500             # timeout revision of the TTL sweeps on R1


def ik(uk: bytes, rev: int) -> bytes:
    return MAGIC + uk + b"$" + struct.pack(">Q", rev)


def be(rev: int, deleted: bool = False) -> bytes:
    """a revision-record value: 8 bytes, or 9 with the deleted flag"""
    return struct.pack(">Q", rev) + (b"\x01" if deleted else b"")


def _val(rng: random.Random) -> bytes:
    return bytes(rng.randrange(256) for _ in range(rng.choice([0, 1, 7, 16, 17, 40])))


# ---- R1: tile seams ----------------------------------------------------------------------------------------------
RUN_LENS = (0, 1, 31, 32, 255, 256, 257, 1023, 1024, 1025)
KINDS = ("versions", "objects", "undecodable", "revdel", "expired")
FOLLOWS = {  # what can stand at the seam after each kind of run (a key's versions ascend: some pairs cannot be built)
    "versions": ("diff", "tomb", "revrec"),
    "objects": ("diff", "tomb", "revrec"),
    "undecodable": ("diff", "same", "trap", "tomb", "revrec"),
    "revdel": ("diff", "trap", "tomb", "revrec"),
    "expired": ("diff", "trap", "tomb", "revrec"),
}
STARTS = (0, 1, 255, 256, 1023)


@dataclass
class Shape:
    store: PackedStore
    starts: Dict[str, bytes]  # named request start keys
    end: bytes                # one past every record


def r1_store(seed: int = 1, lens: Sequence[int] = RUN_LENS, long_tiles: int = 40) -> Shape:
    """Cases laid out one after the other, each `filler | carried | run of L | seam record ...` with the run ending on a
    seam of a request that starts at record 0.  Kinds of run (none of their records is PREVOK):
      versions     versions of the carried record's object above the read revision (one user key throughout)
      objects      one version each of L objects above the read revision (the key changes inside the run)
      undecodable  keys that do not decode (the split byte is not '$'), inside the carried object's key space
      revdel       sweep only: revision records with the deleted flag above the sweep revision (the Q5 `continue`)
      expired      TTL sweep only: `/events/` objects at or below the timeout revision
    Seam records: diff (another object), same (the carried object's next version), trap (the run's last record shares
    all but the revision with the seam record, the carried record does not: only the running LCP minimum over the run
    says "other key"), tomb (a tombstone), revrec (a revision record).  Every kind also gets one run of `long_tiles`
    tiles, and the first record of the long `versions` run is the named start "reach_back"."""
    rng = random.Random(seed)
    items: List[Tuple[bytes, bytes]] = []
    starts: Dict[str, bytes] = {}
    cases = [(k, L, f) for k in KINDS for L in lens for f in FOLLOWS[k]]
    rng.shuffle(cases)
    cases += [(k, long_tiles * TILE, "diff") for k in KINDS]
    for c, (kind, L, follow) in enumerate(cases):
        ns = b"/c%05d/" % c + (b"events/" if kind == "expired" else b"")
        a, b = ns + b"k/a0000000", ns + b"k/z0000000"  # equal lengths: the same-key test compares the LCP
        fill = (-(len(items) + 1 + L)) % TILE
        items += [(ik(ns + b"f%05d" % j, 900), _val(rng)) for j in range(fill)]
        items.append((ik(a, 900), _val(rng)))  # the carried record
        if kind == "versions" and L >= TILE * long_tiles:
            starts["reach_back"] = ik(a, READ + 1)
        run: List[Tuple[bytes, bytes]] = []
        trap = follow == "trap" and L > 0
        for j in range(L - trap):
            if kind == "versions":
                run.append((ik(a, READ + 1 + j), _val(rng)))
            elif kind == "objects":
                run.append((ik(ns + b"k/b%07d" % j, READ + 1), _val(rng)))
            elif kind == "undecodable":
                run.append((ik(a, 900) + b"~%08d" % j, b"junk"))
            elif kind == "revdel":
                run.append((ik(ns + b"k/b%07d" % j, 0), be(READ + 100, True)))
            else:
                run.append((ik(ns + b"k/b%07d" % j, TTL - 100), _val(rng)))
        if trap:
            run.append({"undecodable": (ik(b, 949) + b"~00000000", b"junk"),
                        "revdel": (ik(b, 0), be(READ + 100, True)),
                        "expired": (ik(b, 0), be(TTL - 100))}[kind])
        items += run
        if follow == "same":
            items += [(ik(a, 950), _val(rng)), (ik(a, 960), _val(rng))]
        else:
            if follow == "revrec":
                items.append((ik(b, 0), be(950)))
            items.append((ik(b, 950), TOMB if follow == "tomb" else _val(rng)))
        items.append((ik(ns + b"zz", 970), _val(rng)))
    keys = [k for k, _ in items]
    assert all(x < y for x, y in zip(keys, keys[1:])), "r1_store: records out of order"
    store = PackedStore.from_items(items)
    for s in STARTS:
        starts["s%d" % s] = store.keys[s]
    return Shape(store, starts, b"\xff")


def r1_requests(shape: Shape, rev: int = READ) -> List[Tuple[bytes, bytes, int, int]]:
    """every named start to the end, with runs of empty requests at the start, in the middle and at the end of the
    batch (requests without records share their successor's first tile)"""
    e = shape.end
    k0 = shape.store.keys[0]
    empty = [(k0, k0, rev, 0), (e, e, rev, 0), (k0 + b"\x00", k0 + b"\x00", rev, 0)]
    full = [(s, e, rev, 0) for s in shape.starts.values()]
    return empty + full[:3] + empty + full[3:] + empty


# ---- R2: limit probe windows ---------------------------------------------------------------------------------------
# region: name, records per object (one visible version, then versions above the read revision), objects
R2_REGIONS = (("dense", 1, 9000), ("p1000", 1000, 30), ("p1023", 1023, 12), ("p2000", 2000, 8),
              ("p10000", 10000, 4), ("p40000", 40000, 3))


def r2_store() -> PackedStore:
    items = []
    for i, (name, per, n) in enumerate(R2_REGIONS):
        for j in range(n):
            uk = b"/r2/%d%s/o%05d" % (i, name.encode(), j)
            items.append((ik(uk, 500 + j % 400), b"v%d" % j))
            items += [(ik(uk, READ + 1 + v), b"x") for v in range(per - 1)]
    return PackedStore.from_items(items)


def _region(store: PackedStore, name: str, n_records: Optional[int] = None) -> Tuple[bytes, bytes]:
    i = [r[0] for r in R2_REGIONS].index(name)
    p = b"/r2/%d%s/" % (i, name.encode())
    st = ko.OracleStore(store)
    lo = st.lower_bound(MAGIC + p)
    if n_records is None:
        return MAGIC + p, MAGIC + p[:-1] + b"0"
    return MAGIC + p, store.keys[lo + n_records]


def r2_requests(store: PackedStore) -> Dict[str, Tuple[bytes, bytes, int, int]]:
    rq = {}
    s, e = _region(store, "dense", WINDOW_MIN)
    rq["w0"] = (s, e, READ, 5)             # interval of exactly the first window: not probed
    s, e = _region(store, "dense", WINDOW_MIN + 1)
    rq["w0+1"] = (s, e, READ, 5)           # one record more: probed
    s, e = _region(store, "p1000")
    rq["round0"] = (s, e, READ, 5)
    rq["unlimited"] = (s, e, READ, 0)
    s, e = _region(store, "p1023")
    rq["tile_end"] = (s, e, READ, 1)       # the first emission happens on record 1023, the last of tile 0
    s, e = _region(store, "p2000")
    rq["trailing0"] = (s, e, READ, 5)      # 4 emissions inside window 0, the 5th only as its trailing emission
    s, e = _region(store, "p10000")
    rq["round1"] = (s, e, READ, 2)
    rq["never"] = (s, e, READ, 1000)       # 4 objects
    s, e = _region(store, "p40000")
    rq["round2"] = (s, e, READ, 2)         # window 1 ends after the 2nd visible version: trailing, then round 2
    s, e = _region(store, "p1000", 20000)
    for d, name in ((-1, "total-1"), (0, "total"), (1, "total+1")):
        rq[name] = (s, e, READ, 20 + d)    # 20 objects: 19 emissions inside the loop, the 20th at the end
    return rq


R2_BATCHES = {
    "single": ("round0",),
    "round0": ("w0+1", "round0", "tile_end"),
    "limited": ("w0", "w0+1", "round0", "tile_end", "trailing0", "round1", "round2", "never", "total-1", "total",
                "total+1"),
    "mixed": ("w0+1", "round0", "tile_end", "unlimited"),
}


# ---- R3: pair sizes ------------------------------------------------------------------------------------------------
R3_CHUNKS = (1, 2, 159, 160, 161, 319, 320, 321)
R3_KVS = (1, 31, 32, 33, 64, 65)


def _pair(c: int, j: int) -> Tuple[int, int]:
    """(user key length, value length) of a pair of c >= 2 padded chunks; j turns the value's length inside its last
    chunk (so the wire elements start on every alignment)"""
    ul = 19 if c == 2 or j % 2 else 35  # internal keys of 32 and 48 bytes: two and three chunks
    nv = c - (ul + 13 + 15) // 16
    return ul, ((nv - 1) * 16 + 1 + (j * 7) % 16) if nv else 0


def r3_store(seed: int = 3) -> PackedStore:
    """groups /r3/g<N>/ of N objects (N in R3_KVS) with pairs cycling through R3_CHUNKS but 1; in front of them 33
    one-chunk pairs (keys of at most 16 bytes, empty values) and the 13-byte key of the empty user key; /r3/big/: a
    65 535-byte key (the largest klen) in two versions that share 65 534 bytes, a second key of that length that differs
    in its last user-key byte, and a 1 MiB value"""
    rng = random.Random(seed)
    items = [(ik(b"", 1), b"")] + [(ik(b"#%02d" % j, 2), b"") for j in range(32)]
    for N in R3_KVS:
        for j in range(N):
            c = R3_CHUNKS[1 + (j + N) % (len(R3_CHUNKS) - 1)]
            ul, vl = _pair(c, j)
            uk = (b"/r3/g%02d/%04d" % (N, j)).ljust(ul, b"u")
            items.append((ik(uk, 100 + j), bytes(rng.randrange(256) for _ in range(vl))))
    big = b"/r3/big/"
    huge = big + b"h" * (65535 - 13 - len(big))
    items += [(ik(huge, 5), b"older"), (ik(huge, 6), b""), (ik(huge[:-1] + b"i", 7), b"second"),
              (ik(big + b"m", 9), bytes(rng.randrange(256) for _ in range((1 << 20) + 3)))]
    return PackedStore.from_items(items)


def r3_requests(store: PackedStore) -> List[Tuple[bytes, bytes, int, int]]:
    """the short keys ('#' sorts in front of '$' and '/'), one request per group, then the big group"""
    out = [(MAGIC, MAGIC + b"/r3/", 2**63, 0)]
    for N in R3_KVS:
        out.append((MAGIC + b"/r3/g%02d/" % N, MAGIC + b"/r3/g%02d0" % N, 2**63, 0))
    out.append((MAGIC + b"/r3/big/", MAGIC + b"/r3/big0", 2**63, 0))
    return out


def wire_store(kind: str, seed: int = 4) -> PackedStore:
    """the wire copy's three ring geometries: largest pair below 32 chunks (room 32: everything fits), 100 chunks
    (room 100: elements of exactly 100 wire chunks), and above 160 (room 160: elements of 160 and 161 chunks, the
    second copied straight from the slab).  Value lengths step through all 16 remainders."""
    rng = random.Random(seed)
    top = {"small": 31, "mid": 100, "large": 400}[kind]
    items = []
    for j in range(70):
        wc = [top, top - 1, 2 + j % 20, min(top, 161), min(top, 160), min(top, 159)][j % 6]
        # 15-byte user keys: 4 + 15 and 13 + 15 bytes take the same two chunks, so an element's wire chunk count
        # (magic + user key, value) equals its pair's
        nv = wc - 2
        vl = nv * 16 - (j % 16) if nv else 0
        items.append((ik(b"/w/%s/%07d" % (kind.encode()[:3], j) + b"q", 10 + j),
                      bytes(rng.randrange(256) for _ in range(vl))))
    return PackedStore.from_items(items)


# ---- classes --------------------------------------------------------------------------------------------------------
def _chunks(n: int) -> int:
    return (n + 15) // 16


def _lcp(a: bytes, b: bytes) -> int:
    lo, hi = 0, min(len(a), len(b))
    while lo < hi:  # the longest common prefix, by bisection on slice equality
        m = (lo + hi + 1) // 2
        if a[:m] == b[:m]:
            lo = m
        else:
            hi = m - 1
    return lo


def record_facts(store: PackedStore) -> Dict[str, np.ndarray]:
    """per record, from the bytes: decodes, revision, revision record, tombstone value, value lengths 8 / 9, `/events/`
    in the user key, the revision a revision-record value carries"""
    keys, vals = store.keys.tolist(), store.vals.tolist()
    n = len(keys)
    f = {k: np.zeros(n, bool) for k in ("dec", "rev0", "tomb", "vl8", "vl9", "events")}
    f["rev"] = np.zeros(n, np.uint64)
    f["vrev"] = np.zeros(n, np.uint64)
    f["lcp"] = np.array([LCP_INF] + [_lcp(a, b) for a, b in zip(keys, keys[1:])], np.int64)[:n]  # with record i - 1
    f["klen"] = np.diff(store.keys.off.astype(np.int64))
    for i, (k, v) in enumerate(zip(keys, vals)):
        if len(k) < 13 or k[:4] != MAGIC or k[-9] != 0x24:
            continue
        f["dec"][i] = True
        r = int.from_bytes(k[-8:], "big")
        f["rev"][i] = r
        f["rev0"][i] = r == 0
        f["tomb"][i] = v == TOMB
        f["vl8"][i] = len(v) >= 8
        f["vl9"][i] = len(v) == 9
        f["events"][i] = b"/events/" in k[4:-9]
        if len(v) >= 8:
            f["vrev"][i] = int.from_bytes(v[:8], "big")
    return f


def prevok(f: Dict[str, np.ndarray], read_rev: int, compact: bool = False, timeout_rev: int = 0,
           support_ttl: bool = True) -> np.ndarray:
    """the records worker.run would make its `prev` (scanner.go:430-495): decodable, not TTL-expired, visible, and not
    a deleted-flag revision record above the sweep revision"""
    rev, vrev = f["rev"], f["vrev"]
    exp = np.zeros(len(rev), bool)
    if compact and not support_ttl and timeout_rev:
        exp = f["events"] & np.where(f["rev0"], f["vl8"] & (vrev <= np.uint64(timeout_rev)), rev <= np.uint64(timeout_rev))
    ok = f["dec"] & ~exp & (rev <= np.uint64(read_rev))
    if compact:
        ok &= ~(f["rev0"] & f["vl9"] & (vrev > np.uint64(read_rev)))
    return ok


def _seam_follow(f, ok: np.ndarray, p: int, s: int) -> str:
    """what stands at seam record s after the carried record p (-1: none), by k_emit's same-key rule"""
    if not ok[s]:
        return "run"  # the run goes on across the seam
    if f["rev0"][s]:
        return "revrec"
    if f["tomb"][s]:
        return "tomb"
    if p < 0:
        return "diff"
    kl, lcp = int(f["klen"][s]), f["lcp"]
    if int(f["klen"][p]) == kl and int(lcp[p + 1 : s + 1].min()) >= kl - 9:
        return "same"
    if s - 1 > p and int(f["klen"][p]) == kl and int(lcp[s]) >= kl - 9:
        return "trap"  # the record in front of the seam alone would say "same key"
    return "diff"


def seam_classes(store: PackedStore, reqs, compact: bool = False, timeout_rev: int = 0, support_ttl: bool = True,
                 f=None) -> Dict[str, object]:
    """for every seam of every request: the length of the non-PREVOK run in front of it (-1: it reaches back to the
    request's first record) and, for the runs of RUN_LENS and those reaching back, what stands at the seam; the tiles
    of the batch and the tile every request starts on"""
    f = f or record_facts(store)
    st = ko.OracleStore(store)
    runs, follows, pairs = Counter(), Counter(), Counter()
    ntiles, tile0 = 0, []
    oks = {}
    for s, e, rev, _ in reqs:
        lo, hi = st.lower_bound(s), max(st.lower_bound(e), st.lower_bound(s))
        tile0.append(ntiles)
        ntiles += (hi - lo + TILE - 1) // TILE
        if rev not in oks:
            oks[rev] = prevok(f, rev, compact, timeout_rev, support_ttl)
        ok_all = oks[rev]
        ok = ok_all[lo:hi]
        last = np.maximum.accumulate(np.where(ok, np.arange(hi - lo), -1)) if hi > lo else ok
        for t in range(TILE, hi - lo, TILE):
            p = int(last[t - 1])
            L = t - 1 - p if p >= 0 else -1
            runs[L] += 1
            if L in RUN_LENS or L == -1:
                fo = _seam_follow(f, ok_all, lo + p if p >= 0 else -1, lo + t)
                follows[fo] += 1
                pairs[(L, fo)] += 1
    return dict(runs=runs, follows=follows, pairs=pairs, tiles=ntiles, tile0=tile0)


def probe_round(st: ko.OracleStore, store: PackedStore, req) -> Tuple[Optional[int], List[bool]]:
    """the probe round a limited request settles in (None: not probed), restated with the oracle's loop on the window
    bounds; and per round whether the window's trailing emission alone would have reached the limit"""
    s, e, rev, lim = req
    lo, hi = st.lower_bound(s), st.lower_bound(e)
    if lim <= 0:
        return None, []
    w = -(-max(WINDOW_MIN, 8 * lim) // TILE) * TILE
    if hi - lo <= w:
        return None, []
    trailing = []
    for rnd in range(16):
        whole = lo + w >= hi
        end = e if whole else store.keys[lo + w]
        r = ko.worker_run(st, s, end, rev, lim)
        full = ko.worker_run(st, s, end, rev, 0)
        trailing.append(not r.limit_stop and len(full.emit) >= lim)
        if r.limit_stop or whole:
            return rnd, trailing
        w *= 8
    raise AssertionError("probe did not settle")


def range_classes(store: PackedStore, reqs, wire: bool = False) -> Dict[str, object]:
    """what a batch reaches, from the store bytes and the oracle: seams (seam_classes), probe rounds and whether the
    batch reuses its probe pass as the final pass, emitted pairs' chunk counts, kvs per request, wire fit against the
    ring room and element start alignments"""
    st = ko.OracleStore(store)
    rounds, trailing = [], 0
    for q in reqs:
        r, t = probe_round(st, store, q)
        rounds.append(r)
        trailing += any(t)
    # the probe pass is the final pass when every request of a plain-mode batch was probed and settled in round 0
    reuse = not wire and len(reqs) > 0 and all(r == 0 for r in rounds)
    emits = [ko.range_(st, s, e, rev, lim).emit for s, e, rev, lim in reqs]
    allk = np.concatenate(emits).astype(np.int64) if emits else np.zeros(0, np.int64)
    kl = np.diff(store.keys.off.astype(np.int64))
    vl = np.diff(store.vals.off.astype(np.int64))
    kvc = (kl + 15) // 16 + (vl + 15) // 16
    max_kv = int(kvc.max()) if store.n else 0
    room = min(max(max_kv, 32), 160)
    wc = (4 + (kl - 13) + 15) // 16 + (vl + 15) // 16
    ew = wc[allk]
    _, off = ko.wire_encode(st, allk.astype(np.uint64), ko.WIRE_KVS)
    return dict(
        rounds=rounds, reuse=reuse, trailing=trailing,
        chunks=Counter(kvc[allk].tolist()), max_klen=int(kl[allk].max()) if len(allk) else 0,
        min_klen=int(kl[allk].min()) if len(allk) else 0,
        max_vlen=int(vl[allk].max()) if len(allk) else 0, min_vlen=int(vl[allk].min()) if len(allk) else 0,
        kvs=[len(x) for x in emits], kvs_mod32=sorted({len(x) % GATHER_BLOCK for x in emits}),
        max_kv_chunks=max_kv, room=room,
        wire=dict(fit=int((ew <= room).sum()), at_room=int((ew == room).sum()), room_plus_1=int((ew == room + 1).sum()),
                  nofit=int((ew > room).sum())),
        align=sorted({int(x) % 16 for x in off[:-1]}))


if __name__ == "__main__":  # prints the classes every shape reaches
    sh = r1_store()
    reqs = r1_requests(sh)
    f = record_facts(sh.store)
    print("R1 records", sh.store.n)
    for name, kw in (("range", {}), ("sweep", dict(compact=True)),
                     ("ttl sweep", dict(compact=True, timeout_rev=TTL, support_ttl=False))):
        c = seam_classes(sh.store, reqs, f=f, **kw)
        print("R1", name, "tiles", c["tiles"], "runs", sorted((k, v) for k, v in c["runs"].items() if k in RUN_LENS
                                                               or k < 0 or k >= TILE * 31), "follows", dict(c["follows"]))
    s2 = r2_store()
    rq = r2_requests(s2)
    for b, names in R2_BATCHES.items():
        c = range_classes(s2, [rq[n] for n in names])
        print("R2", b, dict(zip(names, c["rounds"])), "reuse", c["reuse"], "trailing", c["trailing"])
    s3 = r3_store()
    print("R3", range_classes(s3, r3_requests(s3)))
    for kind in ("small", "mid", "large"):
        ws = wire_store(kind)
        print("wire", kind, range_classes(ws, [(MAGIC, b"\xff", 2**63, 0)]))
