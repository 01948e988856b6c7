"""The range shapes (tests/range_shapes.py) reach the boundaries of the scan kernels they are built for.  The GPU tests
in tests/test_gpu_range_shapes.py compare the kernels with the oracle on these shapes; they can only fail on a wrong
boundary if the shape puts something on it, so a change to a builder that stops reaching a class fails here, on any
host.  Every class is derived from the store bytes and the oracle, not from the builders' bookkeeping."""
from __future__ import annotations

import pytest

from tests import range_shapes as rs


@pytest.fixture(scope="module")
def r1():
    sh = rs.r1_store()
    return sh, rs.record_facts(sh.store)


LONG = [t * rs.TILE for t in (31, 32, 33, 40)]


@pytest.mark.parametrize("mode", ["range", "sweep", "ttl"])
def test_r1_reaches_every_seam_class(r1, mode):
    sh, f = r1
    kw = {"range": {}, "sweep": dict(compact=True),
          "ttl": dict(compact=True, timeout_rev=rs.TTL, support_ttl=False)}[mode]
    reqs = rs.r1_requests(sh)
    c = rs.seam_classes(sh.store, reqs, f=f, **kw)
    assert c["tiles"] > rs.SCAN_CHUNK  # one request straddles k_tile_scan's chunk seam
    starts = [c["tile0"][i] for i, (s, e, _, _) in enumerate(reqs) if s >= e]
    assert len(starts) == 9 and len(set(starts)) == 3  # three runs of empty requests, each sharing one first tile
    assert any(a < rs.SCAN_CHUNK < b for a, b in zip(c["tile0"], c["tile0"][1:]))
    for L in rs.RUN_LENS + tuple(LONG):
        assert c["runs"][L] > 0, L
    assert c["runs"][-1] >= 39  # the run that reaches back to the request's first record: no PREVOK in front at all
    follows = {"range": ("diff", "same", "trap", "tomb", "revrec"), "sweep": ("diff", "same", "trap", "tomb", "revrec"),
               "ttl": ("diff", "same", "trap", "tomb", "revrec")}[mode]
    for fo in follows:
        assert c["follows"][fo] > 0, fo
    # each seam record after runs on both sides of the carry window and of one 32-record look-back lane group
    for L in (1, 255, 256, 257, 1024):
        for fo in ("diff", "tomb", "revrec"):
            assert c["pairs"][(L, fo)] > 0, (L, fo)
    assert c["pairs"][(0, "same")] > 0  # an object's versions straddle the seam, the carried record ends the tile
    trap_lens = {L for (L, fo) in c["pairs"] if fo == "trap"}
    assert {1, 32, 256, 1024} <= trap_lens, trap_lens
    if mode != "range":  # the deleted-flag revision records are PREVOK outside the sweep
        assert c["runs"][40 * rs.TILE] >= (4 if mode == "sweep" else 5)


def test_r1_kinds_are_what_they_say(r1):
    """the Q5 revision records and the expired `/events/` records are runs only in the sweeps they belong to"""
    sh, f = r1
    ok_range, ok_sweep = rs.prevok(f, rs.READ), rs.prevok(f, rs.READ, compact=True)
    ok_ttl = rs.prevok(f, rs.READ, compact=True, timeout_rev=rs.TTL, support_ttl=False)
    q5 = f["rev0"] & f["vl9"] & (f["vrev"] > rs.READ)
    assert q5.sum() > 40 * rs.TILE and ok_range[q5].all() and not ok_sweep[q5].any()
    expired = f["events"] & f["dec"] & (f["rev"] <= rs.TTL) & ~f["rev0"]
    assert expired.sum() > 40 * rs.TILE and ok_sweep[expired].all() and not ok_ttl[expired].any()
    assert (~f["dec"]).sum() > 40 * rs.TILE


def test_r2_settles_in_every_round():
    store = rs.r2_store()
    rq = rs.r2_requests(store)
    want = {"w0": None, "w0+1": 0, "round0": 0, "tile_end": 0, "trailing0": 1, "round1": 1, "round2": 2, "never": 1,
            "total-1": 1, "total": 1, "total+1": 1, "unlimited": None}
    st = rs.ko.OracleStore(store)
    for name, q in rq.items():
        r, trailing = rs.probe_round(st, store, q)
        assert r == want[name], name
        if name == "trailing0":
            assert trailing == [True, False]  # window 0 reaches the limit only with its trailing emission
        if name == "round2":
            assert trailing == [False, True, False]
    lo = st.lower_bound(rq["w0"][0])
    assert st.lower_bound(rq["w0"][1]) - lo == rs.WINDOW_MIN and st.lower_bound(rq["w0+1"][1]) - lo == rs.WINDOW_MIN + 1
    tile_end = rs.ko.range_(st, *rq["tile_end"])
    assert tile_end.limit_stop and tile_end.examined == rs.TILE  # the limit-th emission on the last record of tile 0
    total = len(rs.ko.range_(st, rq["total"][0], rq["total"][1], rs.READ).emit)
    assert [rq[n][3] for n in ("total-1", "total", "total+1")] == [total - 1, total, total + 1]
    assert len(rs.ko.range_(st, rq["never"][0], rq["never"][1], rs.READ).emit) < rq["never"][3]


def test_r2_batches_take_the_paths():
    store = rs.r2_store()
    rq = rs.r2_requests(store)
    reuse = {}
    for b, names in rs.R2_BATCHES.items():
        c = rs.range_classes(store, [rq[n] for n in names])
        reuse[b] = c["reuse"]
        assert not rs.range_classes(store, [rq[n] for n in names], wire=True)["reuse"]  # wire batches never reuse
    assert reuse == {"single": True, "round0": True, "limited": False, "mixed": False}
    assert 2 in rs.range_classes(store, [rq[n] for n in rs.R2_BATCHES["limited"]])["rounds"]


def test_r3_pair_sizes():
    store = rs.r3_store()
    c = rs.range_classes(store, rs.r3_requests(store))
    for n in rs.R3_CHUNKS:
        assert c["chunks"][n] > 0, n
    assert max(c["chunks"]) > 2 * rs.GATHER_ROUND  # one pair takes many rounds
    assert c["max_klen"] == 65535 and c["min_klen"] == 13
    assert c["min_vlen"] == 0 and c["max_vlen"] >= 1 << 20
    assert set(rs.R3_KVS) <= set(c["kvs"]) and {0, 1, 31} <= set(c["kvs_mod32"])
    assert c["align"] == list(range(16))
    assert c["room"] == 160 and c["wire"]["at_room"] > 0 and c["wire"]["room_plus_1"] > 0
    # the largest key's two versions share 65 534 bytes: the top of the LCP's 16-bit field, next to KB_LCP_INF
    f = rs.record_facts(store)
    assert int(f["lcp"][(f["klen"] == 65535)].max()) == 65534


@pytest.mark.parametrize("kind", ["small", "mid", "large"])
def test_wire_room(kind):
    store = rs.wire_store(kind)
    c = rs.range_classes(store, [(rs.MAGIC, b"\xff", 2**63, 0)])
    room = {"small": 32, "mid": 100, "large": 160}[kind]
    assert c["room"] == room and c["align"] == list(range(16))
    if kind == "small":
        assert c["max_kv_chunks"] < 32 and c["wire"]["nofit"] == 0
    elif kind == "mid":
        assert 32 <= c["max_kv_chunks"] <= 160 and c["wire"]["at_room"] > 0 and c["wire"]["nofit"] == 0
    else:
        assert c["max_kv_chunks"] > 160 and c["wire"]["at_room"] > 0 and c["wire"]["room_plus_1"] > 0
