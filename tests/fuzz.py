"""Adversarial random inputs for the parity tests (shared by CPU and GPU tests)."""
from __future__ import annotations

import random
import struct
from collections import Counter
from dataclasses import dataclass
from typing import Dict, List, Sequence, Tuple

import numpy as np

from kubebrain_b200.packed import PackedEvents, PackedStore, PackedWatchers, Slab

MAGIC = b"\x57\xfb\x80\x8b"
TOMB = b"tombstone"


def fuzz_store(seed: int, n_keys: int = 60, max_rev: int = 60) -> PackedStore:
    """records with: shared prefixes, '$' and bytes below '$' inside user keys, user keys that are prefixes of each
    other, empty user key, missing revision records, 8/9/odd-length revision-record values, tombstones, 9-byte values
    that are not tombstones, undecodable keys (bad magic / bad split byte / shorter than 13 bytes)."""
    rng = random.Random(seed)
    alphabet = [b"a", b"b", b"/", b"$", b"#", b"\x00", b"\xff", b"events", b"/events/", b"zz"]
    user_keys = set()
    while len(user_keys) < n_keys:
        parts = rng.randint(0, 6)
        uk = b"".join(rng.choice(alphabet) for _ in range(parts))
        if rng.random() < 0.3 and user_keys:
            uk = rng.choice(sorted(user_keys)) + rng.choice(alphabet)  # extensions of existing keys
        if rng.random() < 0.1:
            uk = uk + b"x" * rng.randint(20, 300)  # long keys (several 16-byte chunks, > staging stride)
        user_keys.add(uk)
    items = {}
    for uk in sorted(user_keys):  # sorted: set order depends on the per-process hash seed
        revs = sorted(rng.sample(range(1, max_rev), rng.randint(0, 5)))
        if rng.random() < 0.85:
            r = rng.random()
            latest = revs[-1] if revs else rng.randint(1, max_rev)
            if r < 0.5:
                val = struct.pack(">Q", latest)
            elif r < 0.8:
                val = struct.pack(">Q", rng.choice([latest, rng.randint(1, max_rev)])) + b"\x00"
            elif r < 0.9:
                val = TOMB  # a 9-byte revision-record value that happens to be the tombstone literal
            else:
                val = bytes(rng.randrange(256) for _ in range(rng.choice([0, 3, 8, 9, 12])))
            if len(val) < 8 and b"/events/" in uk:
                val = struct.pack(">Q", latest)  # Go would panic on value[:8] in compactIfExpired
            items[MAGIC + uk + b"$" + b"\x00" * 8] = val
        for i, rev in enumerate(revs):
            r = rng.random()
            if r < 0.2:
                val = TOMB
            elif r < 0.3:
                val = bytes(rng.randrange(256) for _ in range(9))
            elif r < 0.35:
                val = b""
            else:
                val = bytes(rng.randrange(256) for _ in range(rng.randint(1, 40)))
            items[MAGIC + uk + b"$" + struct.pack(">Q", rev)] = val
    # undecodable records
    for _ in range(rng.randint(0, 6)):
        kind = rng.randint(0, 3)
        uk = rng.choice(sorted(user_keys))
        if kind == 0:
            k = b"\x57\xfb\x80\x8c" + uk + b"$" + struct.pack(">Q", rng.randint(0, max_rev))
        elif kind == 1:
            k = MAGIC + uk + b"%" + struct.pack(">Q", rng.randint(0, max_rev))
        elif kind == 2:
            k = MAGIC + bytes(rng.randrange(256) for _ in range(rng.randint(1, 8)))
        else:
            k = bytes(rng.randrange(256) for _ in range(rng.randint(1, 30)))
        items.setdefault(k, b"junk")
    return PackedStore.from_items(list(items.items()))


def fuzz_bounds(store: PackedStore, seed: int, n: int = 8) -> List[Tuple[bytes, bytes]]:
    rng = random.Random(seed)
    keys = store.keys.tolist()
    out = [(b"\x00", b"\xff" * 4), (MAGIC, MAGIC + b"\xff" * 8)]
    for _ in range(n):
        a, b = rng.choice(keys), rng.choice(keys)
        if rng.random() < 0.5:
            a = a[: rng.randint(1, max(len(a), 1))]
        if rng.random() < 0.5:
            b = b[: rng.randint(1, max(len(b), 1))] + b"\xff"
        if a > b:
            a, b = b, a
        out.append((a, b))
    out.append((keys[0], keys[0]))  # empty
    out.append((keys[-1], keys[-1] + b"\x00"))  # last record only
    return out


def fuzz_events(seed: int, n: int = 200, monotone: bool = True) -> PackedEvents:
    rng = random.Random(seed)
    alphabet = [b"a", b"b", b"/", b"/ns-1/", b"/ns-22/", b"pods", b"x" * 20]
    keys, revs = [], []
    rev = rng.randint(1, 50)
    for _ in range(n):
        keys.append(b"".join(rng.choice(alphabet) for _ in range(rng.randint(0, 6))))
        if monotone:
            rev += rng.randint(0, 2)
            revs.append(rev)
        else:
            revs.append(rng.randint(1, 100))
    cuts = sorted(set([0, n] + [rng.randint(0, n) for _ in range(rng.randint(0, 8))]))
    return PackedEvents(Slab.from_list(keys), np.array(revs, dtype=np.uint64), np.array(cuts, dtype=np.uint64))


def fuzz_watchers(ev: PackedEvents, seed: int, n: int = 40) -> PackedWatchers:
    rng = random.Random(seed)
    keys = ev.keys.tolist() or [b""]
    pref, mr = [], []
    maxrev = int(ev.rev.max()) if ev.n else 10
    for _ in range(n):
        r = rng.random()
        k = rng.choice(keys)
        if r < 0.1:
            p = b""
        elif r < 0.7:
            p = k[: rng.randint(0, len(k))]
        elif r < 0.8:
            p = k + b"more"  # longer than any key it could match
        elif r < 0.9 and pref:
            p = rng.choice(pref)  # duplicate prefix (several watchers in one group)
        else:
            p = bytes(rng.randrange(256) for _ in range(rng.randint(1, 5)))
        pref.append(p)
        mr.append(rng.choice([0, 0, rng.randint(0, maxrev + 2)]))
    return PackedWatchers(Slab.from_list(pref), np.array(mr, dtype=np.uint64))


# ---- watch fan-out bursts with exact group sizes -------------------------------------------------------------------
# The fan-out (kubebrain_b200/csrc/kb_watch.cu) picks its path per prefix group from the group's match count, and per
# burst from the shape of the revisions.  The generator below builds bursts that reach each path on purpose; the
# helper after it restates the thresholds and reports which paths a burst reaches, so that the tests can assert it.

REV_MODES = ("consecutive", "runs", "random", "stepback")
CUT_MODES = ("one", "b300", "irregular")
MR_ALL = ("0", "first", "mid", "last", "above", "strip")
PLACES = ("cluster", "border", "spread", "ends")

# restated from kb_watch.cu -- keep in step with it:
FAN_THREADS = 384          # FAN_THREADS: a large group's bitmap is expanded in jobs of this many 32-event words
WINDOW = 256 * 32          # BM_WORDS x 32: events per shared-memory window of the medium groups' sort (d_sort_medium)
HALF_WARP, WARP = 16, 32   # d_watcher_count: <= 16 matches -> half-warp rank sort; <= 32 -> one warp (d_watcher_big)


def fanout_thresholds(E: int) -> Dict[str, int]:
    """match_locked: groups above big_t get a global bitmap (d_expand_large); one bitmap word per 32 events"""
    big_t = max(1024, E // 64)
    bm_words = (E + 31) // 32
    return {"big_t": big_t, "bm_words": bm_words, "chunks_per_group": (bm_words + FAN_THREADS - 1) // FAN_THREADS}


def group_class(n: int, big_t: int) -> str:
    if n == 0:
        return "none"
    if n <= HALF_WARP:
        return "half"
    if n <= WARP:
        return "warp"
    return "medium" if n <= big_t else "large"


def medium_windows(m: np.ndarray) -> int:
    """windows d_sort_medium walks for a group with ascending matches m: from (min & ~31) in steps of WINDOW to max"""
    return 0 if len(m) == 0 else (int(m[-1]) - (int(m[0]) & ~31)) // WINDOW + 1


@dataclass
class Group:
    """`n` events get the key `prefix + b"#<event index>"`; every entry of `min_revs` is one watcher of `prefix` (see
    `_min_rev`).  The group's match count is `n` plus the events of the groups nested inside it.  `place`:
      cluster  n consecutive events inside one WINDOW-aligned window
      border   the first event, the rest centred one WINDOW after it: across the medium sort's window border
      spread   evenly over the burst
      ends     event 0 and event E-1, the rest spread"""
    prefix: bytes
    n: int = 0
    place: str = "spread"
    min_revs: Tuple[str, ...] = ("0",)


def tag(i: int, length: int = 8) -> bytes:
    """a prefix of exactly `length` bytes; tags of different `i` never start with one another (nor with b"/bg/")"""
    t = b"/g%05d/" % i
    assert length >= len(t)
    return t + b"p" * (length - len(t))


class _Free:
    """the first free event at or after p (wrapping), by path-compressed next pointers"""

    def __init__(self, n: int):
        self.n, self.nxt = n, list(range(n + 1))

    def _find(self, i: int) -> int:
        root = i
        while self.nxt[root] != root:
            root = self.nxt[root]
        while self.nxt[i] != root:
            self.nxt[i], i = root, self.nxt[i]
        return root

    def take(self, p: int) -> int:
        q = self._find(min(max(p, 0), self.n))
        if q == self.n:
            q = self._find(0)
        if q == self.n:
            raise ValueError("more group events than events")
        self.nxt[q] = q + 1
        return q


def _spread(n: int, lo: int, hi: int, off: float) -> List[int]:
    return [lo + int((k + off) * (hi - lo) / n) for k in range(n)]


def _place(rng: random.Random, free: _Free, E: int, g: Group) -> List[int]:
    n = g.n
    if g.place == "spread":
        want = _spread(n, 0, E, rng.random())
    elif g.place == "cluster":
        wi = rng.randrange((E + WINDOW - 1) // WINDOW)
        lo, hi = wi * WINDOW, min(E, wi * WINDOW + WINDOW)
        s = lo + rng.randrange(max(1, hi - lo - n + 1))
        want = list(range(s, s + n))
    elif g.place == "border":
        s = rng.randrange(max(1, E - WINDOW - n))
        b = (s & ~31) + WINDOW
        want = [s] + [b - (n - 1) // 2 + k for k in range(n - 1)]
    elif g.place == "ends":
        want = [0, E - 1][:n] + _spread(max(n - 2, 0), 1, E - 1, rng.random())
    else:
        raise ValueError(g.place)
    return [free.take(p) for p in want]


def _cuts(rng: random.Random, E: int, cuts: str) -> List[int]:
    if cuts == "one":
        return [0, E]
    if cuts == "b300":
        return list(range(0, E, 300)) + [E]
    # irregular: empty batches (repeated offsets) first, inside and last; no cut on a multiple of 32
    out, c = [0, 0], 0
    while True:
        step = rng.choice([0, 1, 7, 31, 33, 95, 299, 301, 1001, 4097])
        c2 = c + step
        if step and c2 % 32 == 0:
            c2 += 1
        if c2 >= E:
            break
        out.append(c2)
        c = c2
    return out + [E, E]


def _revisions(rng: np.random.Generator, E: int, bo: Sequence[int], mode: str, base: int) -> np.ndarray:
    """consecutive; runs: non-decreasing with runs of equal revisions; random: unordered inside every batch; stepback:
    every batch ascending, each (non-empty) batch after the first starting below the previous batch's last revision"""
    if mode == "consecutive":
        return np.uint64(base) + np.arange(E, dtype=np.uint64)
    if mode == "runs":
        steps = np.where(rng.random(E) < 0.5, 0, rng.integers(1, 4, E)).astype(np.uint64)
        steps[:1] = 0
        return np.uint64(base) + np.cumsum(steps, dtype=np.uint64)
    rev = np.zeros(E, np.uint64)
    last = None
    for lo, hi in zip(bo[:-1], bo[1:]):
        if lo == hi:
            continue
        if mode == "random":
            rev[lo:hi] = rng.integers(base, base + E + 1, hi - lo)
        elif mode == "stepback":
            start = base if last is None else max(1, last - int(rng.integers(1, 65)))
            steps = rng.integers(0, 3, hi - lo).astype(np.uint64)
            steps[0] = 0
            rev[lo:hi] = np.uint64(start) + np.cumsum(steps, dtype=np.uint64)
            last = int(rev[hi - 1])
        else:
            raise ValueError(mode)
    return rev


def running_max(ev: PackedEvents) -> np.ndarray:
    """per collector batch: max(rev[batch start .. i]); filterByRevision keeps event i iff this is >= min_rev"""
    pm = ev.rev.copy()
    bo = ev.batch_off.astype(np.int64)
    for lo, hi in zip(bo[:-1], bo[1:]):
        if hi > lo:
            pm[lo:hi] = np.maximum.accumulate(ev.rev[lo:hi])
    return pm


def match_lists(keys: Sequence[bytes], prefixes: Sequence[bytes]) -> Dict[bytes, np.ndarray]:
    """prefix -> ascending indices of the keys that start with it"""
    by_len: Dict[int, set] = {}
    for p in set(prefixes):
        by_len.setdefault(len(p), set()).add(p)
    out: Dict[bytes, List[int]] = {p: [] for p in set(prefixes)}
    for L, want in by_len.items():
        for i, k in enumerate(keys):
            if len(k) >= L and k[:L] in want:
                out[k[:L]].append(i)
    return {p: np.array(v, np.int64) for p, v in out.items()}


def burst_events(seed: int, E: int, groups: Sequence[Group], mode: str = "consecutive", cuts: str = "b300",
                 rev_base: int = 1000) -> PackedEvents:
    rng = random.Random(seed)
    free, owner = _Free(E), [-1] * E
    order = sorted(range(len(groups)), key=lambda i: PLACES.index(groups[i].place) if groups[i].place != "ends" else -1)
    for gi in order:
        for p in _place(rng, free, E, groups[gi]) if groups[gi].n else []:
            owner[p] = gi
    keys = [groups[o].prefix + b"#%d" % i if o >= 0 else b"/bg/#%d" % i for i, o in enumerate(owner)]
    bo = _cuts(rng, E, cuts)
    rev = _revisions(np.random.default_rng(seed), E, bo, mode, rev_base)
    return PackedEvents(Slab.from_list(keys), rev, np.array(bo, dtype=np.uint64))


def _min_rev(rng: random.Random, spec: str, m: np.ndarray, ev: PackedEvents, pm: np.ndarray) -> int:
    """0; the group's first / middle / last matching event's revision; above every revision; "strip": a value whose
    survivors (the leading-strip rule) include an event below it, or are not a suffix of the group's events"""
    if spec == "0" or ev.n == 0:
        return 0
    if spec == "above":
        return int(ev.rev.max()) + 1
    revs = ev.rev[m] if len(m) else ev.rev
    if spec in ("first", "mid", "last"):
        return int(revs[{"first": 0, "mid": len(revs) // 2, "last": -1}[spec]])
    assert spec == "strip", spec
    if len(m):
        for j in rng.sample(list(m), min(len(m), 64)):
            mr = pm[j]
            keep = pm[m] >= mr
            if (keep & (ev.rev[m] < mr)).any() or np.any(np.diff(keep.astype(np.int8)) < 0):
                return int(mr)
    return int(revs[len(revs) // 2])


def burst_watchers(ev: PackedEvents, groups: Sequence[Group], seed: int, n: int = 0) -> PackedWatchers:
    """one watcher per (group, min_revs entry), then more on random groups up to n watchers, in shuffled order"""
    rng = random.Random(seed ^ 0x5EED)
    items = [(g.prefix, s) for g in groups for s in g.min_revs]
    while len(items) < n:
        items.append((rng.choice(groups).prefix, rng.choice(MR_ALL)))
    rng.shuffle(items)
    m = match_lists(ev.keys.tolist(), [p for p, _ in items])
    pm = running_max(ev)
    mr = [_min_rev(rng, s, m[p], ev, pm) for p, s in items]
    return PackedWatchers(Slab.from_list([p for p, _ in items]), np.array(mr, dtype=np.uint64))


def fanout_burst(seed: int, E: int, groups: Sequence[Group], mode: str = "consecutive", cuts: str = "b300",
                 n_watchers: int = 0) -> Tuple[PackedEvents, PackedWatchers]:
    ev = burst_events(seed, E, groups, mode, cuts)
    return ev, burst_watchers(ev, groups, seed, n_watchers)


def take_watchers(w: PackedWatchers, n: int, seed: int = 0) -> PackedWatchers:
    """n of the watchers: the first of every prefix (a random n of them if there are more prefixes), then others"""
    rng = random.Random(seed)
    pref = w.prefixes.tolist()
    first: Dict[bytes, int] = {}
    for i, p in enumerate(pref):
        first.setdefault(p, i)
    keep = sorted(first.values())
    if len(keep) > n:
        keep = sorted(rng.sample(keep, n))
    rest = [i for i in range(w.n) if i not in set(keep)]
    keep = sorted(keep + rng.sample(rest, min(len(rest), n - len(keep))))
    return PackedWatchers(w.prefixes.take(keep), w.min_rev[keep].copy())


def fanout_classes(ev: PackedEvents, w: PackedWatchers) -> Dict[str, object]:
    """which of the fan-out's paths a burst reaches, from the events and the watchers alone"""
    E = ev.n
    th = fanout_thresholds(E)
    pref = w.prefixes.tolist()
    m = match_lists(ev.keys.tolist(), pref)
    size = {p: len(v) for p, v in m.items()}
    cls = {p: group_class(size[p], th["big_t"]) for p in m}
    pm = running_max(ev)
    strip = nonsuffix = 0
    for p, mr in zip(pref, w.min_rev.tolist()):
        keep = pm[m[p]] >= mr
        strip += bool((keep & (ev.rev[m[p]] < mr)).any())
        nonsuffix += bool(np.any(np.diff(keep.astype(np.int8)) < 0))
    bo = ev.batch_off.astype(np.int64)
    return dict(
        E=E, W=w.n, G=len(m), n_lens=len({len(p) for p in m}), **th,
        batches=len(bo) - 1, empty_batches=int(np.sum(np.diff(bo) == 0)),
        monotone=bool(np.all(ev.rev[1:] >= ev.rev[:-1])),
        classes=dict(sorted(Counter(cls.values()).items())),
        boundaries=sorted({16, 17, 32, 33, th["big_t"], th["big_t"] + 1} & set(size.values())),
        large=sorted(size[p] for p in m if cls[p] == "large"),
        medium_windows=sorted(Counter(medium_windows(m[p]) for p in m if cls[p] == "medium").items()),
        empty_prefix=cls.get(b""),
        ends=any(p and size[p] and m[p][0] == 0 and m[p][-1] == E - 1 for p in m),
        strip=strip, nonsuffix=nonsuffix)


# ---- the named shapes ----
LENS = (8, 15, 16, 17, 24, 31, 32, 33, 65, 80)  # 15/16/17, 31/32/33 and > 64: the hash and verify chunk borders


def shape_a(mode: str, cuts: str, seed: int = 1, n_watchers: int = 301) -> Tuple[PackedEvents, PackedWatchers]:
    """E = 40 001: big_t 1 024, 1 251 bitmap words, 4 chunks per large group"""
    g = [Group(b"", 0, "spread", ("0", "mid", "strip")),
         Group(b"/g", 0, "spread", ("last",)),  # large like "": it holds every tag
         Group(tag(1), 1025, "spread", MR_ALL), Group(tag(2), 1024, "spread", MR_ALL),
         Group(tag(3, 15), 33, "cluster", ("0", "mid")), Group(tag(4, 16), 33, "border", ("first", "strip")),
         Group(tag(5, 17), 500, "cluster", MR_ALL), Group(tag(6, 31), 500, "spread", MR_ALL),
         Group(tag(7, 32), 520, "border", ("0", "last")),
         Group(tag(8, 33), 16, "cluster", ("0", "mid")), Group(tag(9, 65), 17, "spread", ("0", "strip")),
         Group(tag(10, 80), 32, "cluster", ("mid",)), Group(tag(11), 32, "spread", ("0",)),
         Group(tag(12, 24), 20, "ends", MR_ALL),
         Group(b"/none/", 0, "spread", ("0",)), Group(tag(13), 0, "spread", ("0",)),  # no matches
         Group(tag(9, 65) + b"#" + b"9" * 150, 0, "spread", ("0",)),  # longer than every event key
         Group(b"/n/", 30, "spread", ("0",)), Group(b"/n/in/", 10, "cluster", ("mid",)),  # nested: 45, 15, 5 matches
         Group(b"/n/in/most/", 5, "spread", ("0", "strip"))]
    return fanout_burst(seed, 40001, g, mode, cuts, n_watchers)


def shape_b(mode: str, cuts: str, seed: int = 2, n_watchers: int = 2001) -> Tuple[PackedEvents, PackedWatchers]:
    """E = 200 003: big_t 3 125, 17 chunks per large group, 25 windows"""
    rng = random.Random(seed)
    g = [Group(b"", 0, "spread", ("0", "mid", "strip")), Group(b"/g", 0, "spread", ("last",)),
         Group(tag(1), 3125, "spread", MR_ALL), Group(tag(2, 17), 3126, "spread", MR_ALL),
         Group(tag(3, 33), 3127, "cluster", ("0", "mid")), Group(tag(4, 65), 1500, "spread", MR_ALL),
         Group(tag(5, 16), 40, "border", ("0", "strip")), Group(tag(6, 32), 33, "ends", ("0", "last"))]
    for i in range(600):
        n = rng.choice([0, 1, 2, 3, 5, 8, 13, 16, 17, 21, 32, 33, 40, 100])
        g.append(Group(tag(100 + i, rng.choice(LENS)), n, rng.choice(PLACES[:3]), (rng.choice(MR_ALL),)))
    return fanout_burst(seed, 200003, g, mode, cuts, n_watchers)


def shape_c(mode: str, cuts: str, seed: int = 3, n_watchers: int = 20001) -> Tuple[PackedEvents, PackedWatchers]:
    """E = 20 000 with 20 001 watchers: ~12 k groups over 10 prefix lengths"""
    rng = random.Random(seed)
    g = [Group(b"", 0, "spread", ("0",)), Group(b"/g", 0, "spread", ("mid",))]
    sizes, weights = [0, 1, 2, 3, 4, 5, 6, 16, 17, 32, 33], [50, 30, 10, 2, 2, 2, 2, 0.5, 0.5, 0.5, 0.5]
    for i in range(12000):
        n = rng.choices(sizes, weights)[0]
        g.append(Group(tag(i, rng.choice(LENS)), n, rng.choice(PLACES[:3]), (rng.choice(MR_ALL),)))
    return fanout_burst(seed, 20000, g, mode, cuts, n_watchers)


def shape_tiny(E: int, W: int, mode: str, cuts: str, seed: int = 4) -> Tuple[PackedEvents, PackedWatchers]:
    """E in {1, 31, 32, 33}, W in {1, 2}"""
    if W == 1:
        g = [Group(tag(1, 17), E, "spread", ("mid",))]
    else:
        g = [Group(b"", 0, "spread", ("0",)), Group(tag(1, 33), E // 2, "ends" if E >= 4 else "spread", ("strip",))]
    return fanout_burst(seed, E, g, mode, cuts)


# ---- sequences for one engine ----
def seq_rotation(seed: int = 5, n_bursts: int = 6) -> Tuple[List[PackedEvents], PackedWatchers]:
    """bursts of one geometry (E, cuts, watcher set) with different data: a group that is large in burst k is medium in
    burst k+1, the large groups' events move, and the number of large groups goes 4, 3, 4, 4, 3, 4"""
    E, rot = 40001, (3000, 1500, 600, 40, 17, 0)
    pref = [b"", tag(1), tag(2), tag(3), tag(4), tag(5), tag(6), tag(7, 31), tag(8, 65), b"/none/"]
    bursts = []
    for k in range(n_bursts):
        g = [Group(tag(j + 1), rot[(j + k) % 6], PLACES[(j + k) % 4]) for j in range(6)]
        g += [Group(tag(7, 31), 2500 if k % 3 == 0 else 9), Group(tag(8, 65), 2000 if k % 3 == 2 else 33, "cluster")]
        bursts.append(burst_events(seed + k, E, g, REV_MODES[k % 4], "b300"))
    mrs = [0, 1000 + E // 3, 1000 + E, 2**63]
    items = [(p, r) for p in pref for r in mrs] + [(tag(1), 1000 + E // 2)]
    random.Random(seed).shuffle(items)
    return bursts, PackedWatchers(Slab.from_list([p for p, _ in items]), np.array([r for _, r in items], np.uint64))


def seq_regrow(seed: int = 6) -> Tuple[List[PackedEvents], PackedWatchers]:
    """deliveries small -> large -> small -> large: each large burst exceeds 65 536 deliveries and 1.25 x the previous
    burst's + 4 096 (the output buffer is sized from the previous burst's count and has to grow)"""
    E, M = 40001, 10**6
    g = [Group(tag(1), 200, "cluster"), Group(tag(2), 3000, "spread")]
    plan = [(M - E + 50, "consecutive"), (M, "random"), (M - E + 80, "stepback"), (M, "runs")]
    bursts = [burst_events(seed + k, E, g, mode, "b300", rev_base=base) for k, (base, mode) in enumerate(plan)]
    pref = [b""] * 5 + [tag(1), tag(2)]
    return bursts, PackedWatchers(Slab.from_list(pref), np.array([M] * 5 + [0, M], np.uint64))


if __name__ == "__main__":  # prints the classes every named shape reaches
    def show(name, ev, w):
        print(name, fanout_classes(ev, w))

    for mode in REV_MODES:
        for cuts in ("b300", "irregular"):
            show("A %s %s" % (mode, cuts), *shape_a(mode, cuts))
    for mode in REV_MODES:
        show("B %s b300" % mode, *shape_b(mode, "b300"))
    show("C random irregular", *shape_c("random", "irregular"))
    for E in (1, 31, 32, 33):
        for W in (1, 2):
            show("tiny E=%d W=%d" % (E, W), *shape_tiny(E, W, "random", "irregular"))
    bursts, w = seq_rotation()
    for k, ev in enumerate(bursts):
        show("S1 burst %d" % k, ev, w)
