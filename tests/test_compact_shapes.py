"""The compaction shapes (tests/compact_shapes.py) reach the boundaries of the sweep and the stream's capture they are
built for, and the C oracle the GPU tests compare with agrees with the pure-Python restatement (tests/pyref.py) on every
shape.  The GPU tests in tests/test_gpu_compact_shapes.py can only fail on a wrong boundary if a shape puts something on
it, so a change to a builder that stops reaching a class fails here, on any host."""
from __future__ import annotations

import pytest

from oracle import binding as ko
from tests import compact_shapes as cs
from tests import pyref

ALL = cs.ALL


@pytest.fixture(scope="module")
def classes():
    return cs.compact_classes()


def _pick(classes, prefix):
    return {k: v for k, v in classes.items() if k.startswith(prefix + " ")}


def test_k1_classes_within_a_record(classes):
    k1 = _pick(classes, "K1")
    combos = set().union(*(c["combos"] for c in k1.values()))
    assert {(1,), (2,), (1, 2), (3,), (2, 3), (4,), (5,)} <= combos
    assert {1, 2, 3, 4, 5} <= set().union(*(c["classes"] for c in k1.values()))
    ns = sorted(c["n"] for c in k1.values())
    assert ns[0] == 0 and 1 in ns and 3 in ns  # start == end, the revision record alone, inside one object's versions
    none, every = _pick(classes, "K1 none"), _pick(classes, "K1 every")
    assert [c["victims"] for c in none.values()] == [0]
    assert all(c["classes"] == {1, 2, 3} and c["n"] == c["victims"] == 900 for c in every.values())


def test_k2_tiles_and_slots(classes):
    tiles = _pick(classes, "K2 tiles")
    at0 = next(c for c in tiles.values() if c["start"] == 0)
    assert {0, 1, 2} <= at0["uniform_tiles"]
    assert {(0, 1), (1, 2), (2, 0), (0, 2), (2, 1), (1, 0)} <= at0["seam_changes"]
    assert sorted(c["start"] for c in tiles.values()) == list(cs.K2_STARTS)
    for n in cs.K2_CHAIN_N:
        (c,) = _pick(classes, "K2 chain %d" % n).values()
        assert c["victims"] == 2 * n - 1 and c["n"] == n
    for n in cs.K2_FULL_N:
        (c,) = _pick(classes, "K2 full %d" % n).values()
        assert c["victims"] == 2 * n and c["n"] == n and c["uniform_tiles"] == {2}
    big = _pick(classes, "K2 big")
    assert sorted(c["start"] for c in big.values()) == list(cs.K2_STARTS)
    for c in big.values():
        assert c["n"] > cs.TILE * cs.SCAN_CHUNK and c["chunks"] == 2
        assert min(c["calls_around_chunk_seam"]) > cs.TILE // 2  # dense victims on both sides of the seam
        assert c["combos"] >= {(1,), (2,), (1, 2), (2, 3)}


def test_k3_comparisons(classes):
    c = classes["K3"]
    for k in ("q5", "ttl_obj", "ttl_rev"):
        assert c[k] == {(-1, True), (0, True), (1, False)}, k
    assert {(1, (2,)), (0, (2, 3)), (-1, (2, 3))} <= c["tombrev"]
    for ln in (7, 8, 9, 10):
        assert (ln, False, False) in c["vl"] and (ln, False, True) in c["vl"], ln
    for ln in (8, 9, 10):
        assert (ln, True, True) in c["vl"] and (ln, True, False) in c["vl"], ln
    assert not any(ev and ttl and ln < 8 for ln, ev, ttl in c["vl"])  # the oracle's error case stays out of TTL sweeps
    assert c["short_events_plain"]
    assert {0, 1, 2**63 - 1, 2**63, 2**63 + 1, 2**64 - 2, 2**64 - 1} <= c["sweep_revs"]
    for k in ("timeout_above_rev", "ttl_off_with_timeout", "no_ttl_zero_timeout", "expired_before_live"):
        assert c[k], k
    s = classes["K3 seam"]
    assert s["run_end_in_tile"] == {cs.TILE - 1} and s["expired"] == sum(cs.K3_SEAM_RUNS)


def test_k4_capture_and_entries(classes):
    for v in cs.K4_COUNTS:
        c = classes["K4 count %d" % v]
        assert c["n"] == v and c["tiles"] == -(-v // cs.CAPTURE_TILE)
        if v >= 64:
            assert c["key_pad"] == set(range(16)), v
    assert classes["K4 count 70000"]["tiles"] > 2 * cs.LOOKBACK
    plain, ttl = classes["K4 entries t=0"], classes["K4 entries t=%d" % cs.K4_TIMEOUT]
    assert set(cs.K4_KEY_LENS) <= plain["key_lens"] and plain["guard_lens"] == {9} and 3 in plain["classes"]
    assert set(cs.K4_GUARD_LENS) <= ttl["guard_lens"] and {4, 5} <= ttl["classes"]


def test_k5_layouts(classes):
    e, s = classes["K5 exact"], classes["K5 straddle"]
    assert e["past"] and e["starts_at_line"] and e["entry_at_line"] == 4096 and e["unit"] == 2**20
    assert s["past"] and s["guard_straddles"] and s["entry_at_line"] == 4095 and s["unit"] == 2**20 + 16
    small = cs.k5_store(64, n=5)
    assert all(small.vals[i][8:9] == bytes([i]) and small.vals[i][-1:] == b"\xa5" for i in range(5))


def _pin(store, sweeps):
    st = ko.OracleStore(store)
    keys, vals = store.keys.tolist(), store.vals.tolist()
    for s, e, rev, trev, ttl in sweeps:
        x = ko.worker_run(st, s, e, rev, compact=True, timeout_rev=trev, support_ttl=ttl, collect=True)
        p = pyref.worker_run(keys, vals, s, e, rev, compact=True, timeout_revision=trev, support_ttl=ttl)
        assert x.rc == 0 and p.error is None, (s[:24], rev, trev, ttl)
        assert list(zip(x.victims.tolist(), x.vclass.tolist())) == p.victims, (s[:24], rev, trev, ttl)
        assert (x.count, x.examined) == (p.count, p.examined), (s[:24], rev, trev, ttl)


def test_oracle_agrees_with_pyref():
    full = (cs.MAGIC, b"\xff", ALL, 0, True)
    _pin(cs.k1_store(), cs.k1_sweeps())
    _pin(cs.k1_none_store(), [full])
    _pin(cs.k1_every_store(), [full])
    t = cs.k2_tiles_store()
    _pin(t, [(t.keys[j], b"\xff", ALL, 0, True) for j in cs.K2_STARTS])
    for n in cs.K2_CHAIN_N[:-1] + (3000,):  # 3 000 stands for 300 000
        _pin(cs.chain_store(n), [full])
    for n in cs.K2_FULL_N:
        _pin(cs.full_store(n), [full, (cs.MAGIC, b"\xff", cs.T_TOMB - 1, 0, True)])
    b = cs.big_store(5000)  # the 1.1 M pattern at reduced size
    _pin(b, [(b.keys[j], b"\xff", ALL, 0, True) for j in cs.K2_STARTS])
    _pin(cs.k3_store(), cs.k3_sweeps())
    s3 = cs.k3_seam_store()
    _pin(s3, [(s3.keys[j], b"\xff", ALL - 1, t, ttl) for j in (0, 1)
              for t, ttl in ((cs.K3_SEAM_TIMEOUT, False), (cs.K3_SEAM_TIMEOUT, True), (1024, False), (0, True))])
    c4 = cs.k4_count_store(2000)
    _pin(c4, [(cs.MAGIC, cs.k4_count_end(c4, v), ALL, 0, True) for v in (1, 1023, 1024, 1025)])
    _pin(cs.k4_entry_store(), cs.k4_entry_sweeps())
    _pin(cs.k5_store(64, n=5), [(cs.MAGIC, b"\xff", cs.K5_REV, cs.K5_TIMEOUT, False)])


def test_k3_short_events_values_error_only_in_ttl_sweeps():
    """the `/events/` revision records shorter than 8 bytes: Go would panic in a TTL sweep (the oracle errors); a plain
    sweep passes them"""
    st = ko.OracleStore(cs.k3_store())
    assert ko.worker_run(st, cs.K3_TTL_END, b"\xff", 10, compact=True, timeout_rev=7, support_ttl=False).rc != 0
    assert ko.worker_run(st, cs.K3_TTL_END, b"\xff", 10, compact=True).rc == 0
