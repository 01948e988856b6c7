"""CPU check of tests/reconcile_shapes.py: every shape reaches the classes it is built for (derived from the bytes by
the plain merge model, never from the builders' bookkeeping), the shapes together reach every boundary kb_reconcile
has, and the model itself agrees with a restatement of the diff on small cases."""
from __future__ import annotations

import pytest

from tests import reconcile_shapes as rs

SHAPES = {s.name: s for s in rs.all_shapes()}

# every class the suite must reach, by topic
REQUIRED = {
    "edges": {"diff_first", "diff_last", "key_eq_start", "key_eq_end", "outside_divergent"},
    "values": {"byte_0", "byte_15", "byte_16", "byte_17", "byte_last", "len_pm1_equal_pad", "empty_vs_nul",
               "tombstone", "rev8_vs_9"},
    "keys": {"klen_1", "klen_15", "klen_16", "klen_17", "klen_65535", "last_byte_only", "prefix_of_next"},
    "sizes": {"%s_%d" % (p, n) for p in ("n", "span") for n in rs.SIZES} | {"n_1e5", "span_1e5", "all_missing",
                                                                            "all_extra", "identical", "one_in_1e5"},
    "walks": {"chunk_1", "chunk_2", "chunk_7", "chunk_4096", "chunk_end_on_diff"},
    "interplay": {"compact_stream", "range_stream", "range_batch", "ttl_changed", "ttl_unchanged"},
}


@pytest.mark.parametrize("name", list(SHAPES))
def test_shape_reaches_its_tags(name):
    sh = SHAPES[name]
    got = rs.reconcile_classes(sh)
    assert set(sh.tags) <= got, sorted(set(sh.tags) - got)


def test_shapes_cover_every_boundary():
    reached = set()
    for sh in SHAPES.values():
        reached |= rs.reconcile_classes(sh)
    for topic, need in REQUIRED.items():
        assert need <= reached, (topic, sorted(need - reached))


def test_merge_model_small_cases():
    a, b, c, d = (rs.ik(b"/m/%d" % i, 5) for i in range(4))
    mirror = {a: b"1", b: b"2", c: b"3"}
    inp = [(a, b"1"), (b, b"2 new"), (d, b"4")]
    assert rs.diff(mirror, inp, a, rs.ik(b"/m/9", 5)) == [(rs.CHANGED, b, 1), (rs.EXTRA, c, rs.NO_SRC), (rs.MISSING, d, 2)]
    assert rs.diff(mirror, [], b, b) == []                          # start >= end: an empty diff
    assert rs.diff(mirror, [(b, b"2")], b, c) == []                  # c is the end: not read
    assert rs.diff({a: b"abc"}, [(a, b"abc\x00")], a, b) == [(rs.CHANGED, a, 0)]
    assert rs.ops_of([(rs.CHANGED, b, 1), (rs.EXTRA, c, rs.NO_SRC)], inp) == [(b, b"2 new"), (c, None)]


def test_walk_chunks_end_on_the_last_key():
    keys = [rs.ik(b"/w/%d" % i, 5) for i in range(5)]
    eng = {k: b"v" for k in keys}
    lo, hi = rs.ik(b"/w/", 0), rs.ik(b"/w0", 0)
    ch = rs.walk(eng, lo, hi, 2)
    assert [(s, e, [k for k, _ in got]) for s, e, got in ch] == [
        (lo, keys[1] + b"\x00", keys[:2]), (keys[1] + b"\x00", keys[3] + b"\x00", keys[2:4]), (keys[3] + b"\x00", hi, keys[4:])]
    ch = rs.walk(eng, lo, hi, 5)  # exactly one full chunk: a second call finds EOF
    assert [len(got) for _, _, got in ch] == [5, 0] and ch[-1][1] == hi


def test_rejections_are_listed():
    codes = {code for _, code, _, _, _ in rs.rejections()}
    assert codes == {"KB_EUNSORTED", "KB_EINVAL", "KB_ELIMIT"}
