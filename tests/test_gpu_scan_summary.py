"""GPU parity of the scan summary that kb_apply_batch keeps beside the directory (kb_store.cu): value replacements
that flip the facts the summary holds about a record -- the tombstone literal, a revision record's deleted flag, a
/events/ key's expiry inputs -- and inserts / delete runs that change which record sits in front of another, checked
against the oracle with ranges and compaction sweeps (the heap-layout write path of test_gpu_round2, seen from the
scan's side)."""
from __future__ import annotations

import random
import struct

import pytest

from kubebrain_b200 import synth
from kubebrain_b200._lib import Engine
from kubebrain_b200.coder import NormalCoder
from kubebrain_b200.packed import PackedStore
from oracle import binding as ko
from tests.test_gpu_parity import check_compact, check_ranges

pytestmark = pytest.mark.gpu

CODER = NormalCoder()
LO, HI = CODER.encode_object_key(b"/registry/", 0), CODER.encode_object_key(b"/registry0", 0)


@pytest.fixture()
def eng():
    e = Engine(0)
    yield e
    e.close()


def _rev(k: bytes) -> int:
    return struct.unpack(">Q", k[-8:])[0]


def _check(eng, items, meta):
    cur = PackedStore.from_items(list(items.items()))
    st = ko.OracleStore(cur)
    assert eng.store_info()[0] == cur.n
    mid = (meta.first_rev + meta.last_rev) // 2
    top = meta.last_rev + 1000
    check_ranges(eng, cur, st, [(LO, HI, top, 0), (LO, HI, meta.read_rev, 0), (LO, HI, mid, 7), (LO, HI, top, 13)])
    for rev in (mid, meta.read_rev, top):
        check_compact(eng, cur, st, LO, HI, rev)
        eng.set_compact_revision(None)
    check_compact(eng, cur, st, LO, HI, top, timeout_rev=mid, support_ttl=False)
    eng.set_compact_revision(None)
    return cur, st


def test_summary_follows_value_replacements(eng, tmp_path):
    """a value replaced by the tombstone literal and back, a revision record replaced by a 9-byte deleted-flag value (at
    a revision below and above the read revision) and back, near-miss values ("tombstonf", 8 and 10 bytes), /events/
    keys, then inserts next to existing records and runs of deletes: every round answers like the oracle"""
    rng = random.Random(17)
    store, meta = synth.gen_store(3000, 3, 48, 40, 6, config_id=2, tomb_frac=0.1)
    eng.load_sorted(store)
    items = dict(zip(store.keys.tolist(), store.vals.tolist()))
    keys = sorted(items)
    objs = [k for k in keys if _rev(k) != 0]
    revrecs = [k for k in keys if _rev(k) == 0]
    tombed = rng.sample(objs, 300)
    flagged = rng.sample(revrecs, 300)
    near = rng.sample([k for k in objs if k not in set(tombed)], 60)
    lo_rev, hi_rev = meta.first_rev, meta.last_rev + 50

    def flag_val():
        return struct.pack(">Q", rng.choice((lo_rev, meta.read_rev, hi_rev))) + b"\x00"

    # round 1: tombstones, deleted flags, near misses; /events/ objects (revision record + one version each)
    ops = [(k, b"tombstone") for k in tombed]
    ops += [(k, flag_val()) for k in flagged]
    ops += [(k, rng.choice((b"tombstonf", b"tombston", b"tombstone!"))) for k in near]
    ev_rev = meta.last_rev + 1
    ev_keys = []
    for i in range(80):
        uk = b"/registry/events/ns-%02d/e%03d" % (i % 5, i)
        rk, ok = CODER.encode_object_key(uk, 0), CODER.encode_object_key(uk, ev_rev + i)
        ops.append((rk, struct.pack(">Q", ev_rev + i) + (b"\x00" if i % 3 == 0 else b"")))
        ops.append((ok, b"tombstone" if i % 4 == 0 else b"e" * (5 + i)))
        ev_keys.append((rk, ok))
    eng.apply_batch(ops)
    items.update(ops)
    _check(eng, items, meta)

    # round 2: every replacement undone or flipped the other way
    ops = [(k, b"x" * rng.randint(0, 40)) for k in tombed]
    ops += [(k, struct.pack(">Q", rng.choice((lo_rev, meta.read_rev, hi_rev)))) for k in flagged]
    ops += [(k, b"tombstone") for k in near]
    for i, (rk, ok) in enumerate(ev_keys):
        ops.append((rk, struct.pack(">Q", ev_rev + i) + (b"" if i % 3 == 0 else b"\x00")))
        ops.append((ok, b"e" * 9 if i % 4 == 0 else b"tombstone"))
    eng.apply_batch(ops)
    items.update(ops)
    _check(eng, items, meta)

    # round 3: new versions inserted next to existing records, runs of deletes (the record behind each run gets a new
    # predecessor), a deleted record's neighbour rewritten in the same batch
    keys = sorted(items)
    ops = []
    for k in rng.sample(keys, 200):
        if _rev(k) != 0:
            ops.append((k[:-8] + struct.pack(">Q", _rev(k) + 1), rng.choice((b"tombstone", b"n" * 12))))
    gone = set()
    for start in rng.sample(range(len(keys) - 8), 40):
        for k in keys[start:start + rng.randint(1, 6)]:
            gone.add(k)
        if start + 7 < len(keys):
            ops.append((keys[start + 7], flag_val()))
    ops += [(k, None) for k in sorted(gone)]
    eng.apply_batch(ops)
    for k, v in ops:
        if v is None:
            items.pop(k, None)
        else:
            items[k] = v
    cur, st = _check(eng, items, meta)

    # the summary is not part of a dump: restore rebuilds it
    path = str(tmp_path / "snap.kb")
    eng.dump(path)
    e2 = Engine(0)
    try:
        e2.restore(path)
        check_ranges(e2, cur, st, [(LO, HI, meta.last_rev + 1000, 0), (LO, HI, meta.read_rev, 5)])
        check_compact(e2, cur, st, LO, HI, meta.read_rev)
    finally:
        e2.close()
