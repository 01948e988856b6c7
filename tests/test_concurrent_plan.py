"""The plans of tests/test_gpu_concurrent.py (tests/concurrent_plan.py), on any host: they are deterministic per seed,
the reads they call invariant answer the same on every version (checked with the C oracle), the window reads do change,
and a plan whose writes land at or below a read revision among the invariant reads' records is caught."""
from __future__ import annotations

import pytest

from oracle import binding as ko
from tests import concurrent_plan as cp
from tests import partition_shapes as ps

WINDOW_KINDS = ("count", "info")


@pytest.fixture(scope="module")
def plan():
    return cp.gen_plan(0)


def _designated_window(r: cp.Read) -> bool:
    return r.kind in WINDOW_KINDS or (r.kind == "get" and all(rev == 0 for _, rev in r.args["reqs"]))


def test_plans_are_deterministic(plan):
    again = cp.gen_plan(0)
    assert again.batches == plan.batches and again.items == plan.items
    assert [r.answers for r in again.reads] == [r.answers for r in plan.reads]
    other = cp.gen_plan(1)
    assert other.batches != plan.batches


def test_invariant_and_window_sets_are_as_claimed(plan):
    for r in plan.reads:
        assert len(r.answers) == len(plan.items)
        if _designated_window(r):
            assert not r.invariant, (r.kind, r.args.get("mode"))
        else:
            assert r.invariant, (r.kind, r.args.get("mode"), r.answers)
    c = cp.classes(plan)
    assert {"range/host", "range/device", "range/kvs", "range/events", "range/dev_kvs", "range/count", "get/host",
            "get/kvs", "stream/host", "stream/kvs", "partitions/-", "sweep/-", "cstream/-"} <= set(c["invariant"])
    assert {"get/host", "get/kvs", "count/count", "info/-"} <= set(c["window"])
    assert c["ops"] == ["del", "put", "ttl"] and c["long_key"] and c["undecodable"] > 0


def test_writes_land_above_every_read_revision_and_after_every_invariant_record(plan):
    revs = {r for rd in plan.reads for r in
            [q[2] for q in rd.args.get("reqs", []) if len(q) == 4 and q[2] != cp.ALL] +
            [q[1] for q in rd.args.get("reqs", []) if len(q) == 2 and q[1]] +
            [rd.args.get("rev", 0), rd.args.get("req", (0, 0, 0))[2]]}
    assert max(revs) <= plan.base_rev
    assert min(revs - {0}) >= cp.SWEEP_REV  # no read is below the compact revision the plan's sweeps record
    assert {rd.args["rev"] for rd in plan.reads if rd.kind in ("sweep", "cstream")} == {cp.SWEEP_REV}
    for b in plan.batches:
        for op in b:
            assert op[0] >= cp.INV_HI
            uk, rev, err = ko.decode(op[0])
            assert err == 0 and (rev == 0 or rev > plan.base_rev)


def test_partitions_of_the_plan_pass_check_partitions(plan):
    r = next(x for x in plan.reads if x.kind == "partitions")
    a = r.args
    v0 = plan.stores[0]
    st = ko.OracleStore(v0)
    got = ps.partitions(v0, st, a["start"], a["end"], a["rev"], a["part_bytes"], a["max_parts"])
    assert len(got[0]) > 3
    ps.check_partitions(v0, st, a["start"], a["end"], a["rev"], got)


def test_window_check_rejects_an_answer_outside_its_window(plan):
    r = next(x for x in plan.window_reads if x.kind == "get")
    changes = [v for v in range(1, len(r.answers)) if r.answers[v] != r.answers[v - 1]]
    v = changes[-1]
    # the answer of version v is inside [v - 1, v] and outside [0, w] for every w + 1 < v that answers differently
    assert r.answers[v] in r.answers[v - 1 : v + 1]
    assert r.answers[v] not in [r.answers[w] for w in range(v) if r.answers[w] != r.answers[v]]


def test_a_write_at_or_below_a_read_revision_changes_an_invariant_read():
    """the wrong variant: the same commits at revisions starting below the base revision, among the invariant reads'
    records -- the oracle must see some designated invariant read change"""
    bad = cp.gen_plan(0, low=True)
    broken = [r for r in bad.reads if not _designated_window(r) and not r.invariant]
    assert broken, "no invariant read noticed writes at or below its revision"
    assert {r.kind for r in broken} & {"range", "stream", "partitions"}


def test_bursts_share_one_watcher_set():
    b = cp.gen_bursts()
    assert len(b.events) >= 4 and len(b.expected) == len(b.events)
    assert all(len(s) == b.watchers.n + 1 for s, _ in b.expected)
    assert len({int(s[-1]) for s, _ in b.expected}) > 1  # different data, different deliveries
