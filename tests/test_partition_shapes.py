"""CPU tests of the partition boundary shapes (tests/partition_shapes.py): each shape reaches the classes it is built
for, the partition definition keeps every invariant on every Q1 interval, the cut rule without the key-order drop
breaks them on interleaved user keys, the drop never fires on stores without them, and the restatement of
adjustPartitionsBorders agrees with the C oracle's."""
from __future__ import annotations

import pytest

from kubebrain_b200 import synth
from kubebrain_b200.coder import NormalCoder
from oracle import binding as ko
from tests import partition_shapes as ps


@pytest.fixture(scope="module")
def classes():
    return ps.partition_classes()


def test_q1_classes(classes):
    q1 = {k: v for k, v in classes.items() if k.startswith("Q1 ")}
    for flag in ("order_drop", "on_outer", "on_inner", "both", "straddle", "start_in_versions", "end_in_versions",
                 "start_after_revrec", "start_is_revkey_e1", "start_ge_end", "start_empty"):
        assert any(c[flag] for c in q1.values()), flag
    assert {c["end"] for c in q1.values()} == {"empty", "ff", "key"}
    assert max(c["depth"] for c in q1.values()) == 3
    # without revision records the interleaved pair still runs a border backwards
    assert classes["Q1 q no-revrec rev=1000"]["order_drop"] and classes["Q1 n no-revrec rev=-1"]["order_drop"]
    assert not classes["Q1 start_in_versions rev=1000"]["order_drop"]


def test_q2_classes(classes):
    for n in ps.Q2_N:
        c = classes["Q2 n=%d every" % n]
        assert c["P"] == n and c["at1"] and c["at_last"]
        assert classes["Q2 n=%d exact" % n]["exact"] == (n % 2 == 0)
    big = classes["Q2 n=1100 every"]
    assert big["on_pivot"] and big["past_pivot"]
    assert not classes["Q2 n=33 every"]["on_pivot"]  # 32 candidates: the final round at once
    assert classes["Q2 n=34 every"]["on_pivot"]      # 33 candidates: one pivot round
    assert classes["Q2 n=34 exact"]["exact"] and not classes["Q2 n=34 bumped"]["exact"]
    assert [classes["Q2 T=7pb%+d" % d]["P"] for d in (-1, 0, 1)] == [8, 7, 7]
    assert classes["Q2 big"]["repeated"] and not classes["Q2 big"]["unreached"]
    assert classes["Q2 last huge"]["unreached"]


def test_q3_q4_classes(classes):
    assert {classes["Q3 P=%d" % p]["last_warp"] for p in (16, 17, 18, 32, 33, 34)} == {14, 15, 0}
    assert {classes["Q3 P=%d" % p]["rounds"] for p in (16, 17, 18, 32, 33, 34)} == {1, 2, 3}
    lens = classes["Q4 key lengths"]
    assert lens["mod16"] == list(range(16)) and {13, 16, 17, 31, 32, 33, 65535} <= set(lens["lens"])
    s = classes["Q4 stride"]
    assert s["max_kv_chunks"] == 4097  # 65 535-byte key, 4-byte value
    assert s["report"] == 16 + 4095 * 32 + 4095 * 4097 * 16 == 268_566_496


@pytest.mark.parametrize("rev_records", [True, False])
def test_definition_keeps_the_invariants_on_q1(rev_records):
    store = ps.q1_store(rev_records)
    st = ko.OracleStore(store)
    for name, s, e in ps.q1_intervals(store):
        for rev in ps.Q1_REVS:
            emit = ko.range_(st, s, e, rev, 0).emit.tolist()
            total = sum(ps.pad16(len(store.keys[i])) + ps.pad16(len(store.vals[i])) for i in emit)
            for pb in ps.q1_part_bytes(total, len(emit)):
                for mp in (2, 3, 64):
                    got = ps.partitions(store, st, s, e, rev, pb, mp)
                    ps.check_partitions(store, st, s, e, rev, got, ps.Q1_REVS)


def _old_rule(store, st, s, e, rev, part_bytes, max_parts):
    """the cut rule before the key-order drop: every cut's revision key, whatever lies in front of it"""
    emit = ko.range_(st, s, e, rev, 0).emit.tolist()
    sizes = [ps.pad16(len(store.keys[i])) + ps.pad16(len(store.vals[i])) for i in emit]
    cuts = ps.cuts_of(sizes, part_bytes, max_parts, s, e)
    slot = [0]
    for x in sizes:
        slot.append(slot[-1] + x)
    return ([s] + [ps.revision_key(store.keys[emit[i]]) for i in cuts] + [e], [0] + cuts + [len(emit)],
            [0] + [slot[i] for i in cuts] + [slot[-1]])


@pytest.mark.parametrize("rev_records", [True, False])
def test_old_rule_breaks_the_invariants_on_interleaved_keys(rev_records):
    store = ps.q1_store(rev_records)
    st = ko.OracleStore(store)
    s, e = ps.ik(b"/q/", 0), ps.ik(b"/q0", 0)
    old = _old_rule(store, st, s, e, ps.ALL, 1, 64)
    # the issue's borders: /q/, /q/c$\0*7$<0>, /q/c$<0>, /q/z$<0>, /q0 -- backwards, and partition 1 answers nothing
    assert old[0][1:4] == [ps.ik(ps.nest(b"/q/c", 0), 0), ps.ik(b"/q/c", 0), ps.ik(b"/q/z", 0)]
    with pytest.raises(AssertionError, match="strictly increasing"):
        ps.check_partitions(store, st, s, e, ps.ALL, old)
    assert ko.range_(st, old[0][1], old[0][2], ps.ALL, 0).emit.tolist() == []
    parts = list(zip(old[0], old[0][1:]))
    assert ps.adjust_partitions_borders(parts) != parts
    # the client's streams over the adjusted partitions repeat /q/c and /q/c$\0*7
    cat = []
    for a, b in ps.adjust_partitions_borders(parts):
        cat += ko.range_(st, a, b, ps.ALL, 0).emit.tolist() if a < b else []
    assert sorted(cat) != sorted(set(cat))
    # start == revision_key(e_1): the old border equals start
    s1 = ps.ik(b"/q/c", 0)
    old = _old_rule(store, st, s1, e, ps.ALL, 1, 64)
    assert old[0][1] == s1
    with pytest.raises(AssertionError, match="strictly increasing"):
        ps.check_partitions(store, st, s1, e, ps.ALL, old)
    new = ps.partitions(store, st, s, e, ps.ALL, 1, 64)
    assert len(new[0]) == len(_old_rule(store, st, s, e, ps.ALL, 1, 64)[0]) - 1  # the backwards cut alone is dropped
    ps.check_partitions(store, st, s, e, ps.ALL, new)


def _plain_stores():
    coder = NormalCoder()
    s2, meta = synth.gen_store(1500, 3, 48, 300, 20, config_id=2)
    yield s2, coder.encode_object_key(b"/registry/", 0), coder.encode_object_key(b"/registry0", 0), meta.read_rev
    yield ps.mixed_store(), coder.encode_object_key(b"/m/", 0), coder.encode_object_key(b"/m0", 0), ps.READ
    yield ps.uniform_store(2050), coder.encode_object_key(b"/u/", 0), b"\xff", ps.READ
    yield ps.long_key_store(), b"", b"\xff", 25


def test_the_drop_never_fires_without_interleaved_keys():
    """stores whose user keys are never another's + '$' + bytes keep every cut they had"""
    for store, lo, hi, rev in _plain_stores():
        st = ko.OracleStore(store)
        emit = ko.range_(st, lo, hi, rev, 0).emit.tolist()
        total = sum(ps.pad16(len(store.keys[i])) + ps.pad16(len(store.vals[i])) for i in emit)
        for share in (3, 64, 1000, 4096):
            pb = max(total // share, 1)
            assert ps.partitions(store, st, lo, hi, rev, pb, ps.MAX_PARTS) == \
                _old_rule(store, st, lo, hi, rev, pb, ps.MAX_PARTS)


def test_adjust_restatement_equals_the_oracle():
    ik = ps.ik
    chains = [[b"", b"\xff"], [ik(b"/a", 0), ik(b"/b", 5), ik(b"/c", 0), b"\xff"],
              [b"", ik(b"/a", 7), b"junk", ik(b"/a$\x00", 3), ik(b"/b", 0)], [ik(b"/x", 9), ik(b"/y", 9)]]
    for borders in map(sorted, chains):  # the oracle's restatement takes contiguous partitions in order
        adj = ps.adjust_partitions_borders(list(zip(borders, borders[1:])))
        assert [adj[0][0]] + [b for _, b in adj] == ko.adjust_partition_borders(borders)
    # partitions out of order are sorted by start and chained
    assert ps.adjust_partitions_borders([(b"c", b"d"), (b"a", b"b")]) == [(b"a", b"b"), (b"b", b"d")]
