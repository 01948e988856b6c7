"""The watch fan-out's burst shapes (tests/fuzz.py) reach the kernel paths they are meant to reach.  The GPU tests in
tests/test_gpu_fanout_shapes.py compare the kernel with the oracle on these shapes; they can only fail on a wrong path
if the shape takes it, so a change to the generator that stops reaching a class fails here, on any host."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import binding as ko
from tests import fuzz

REV_MODES, CUT_MODES = fuzz.REV_MODES, fuzz.CUT_MODES


def check_revisions(ev, c, mode, cuts):
    """the revision mode and batch cuts show in the burst: the non-monotone flag, the leading-strip rule, cut offsets"""
    bo = ev.batch_off.astype(np.int64)
    multi = int(np.sum(np.diff(bo) > 0)) > 1
    assert c["monotone"] == (mode in ("consecutive", "runs") or (mode == "stepback" and not multi))
    if mode == "runs":
        assert np.any(ev.rev[1:] == ev.rev[:-1])
    if mode == "random":
        assert c["strip"] > 0  # a watcher keeps an event whose own revision is below its min_rev
    if not c["monotone"] and multi:  # (inside one batch the running maximum never drops)
        assert c["nonsuffix"] > 0  # a watcher's survivors are not a suffix of its group
    if mode == "stepback" and multi:
        for lo, hi in zip(bo[:-1], bo[1:]):
            if hi > lo:
                assert np.all(ev.rev[lo + 1 : hi] >= ev.rev[lo : hi - 1])  # every batch ascending, the burst is not
    inner = bo[1:-1][(bo[1:-1] > 0) & (bo[1:-1] < ev.n)]
    if cuts == "irregular":
        assert c["empty_batches"] >= 2 and np.all(inner % 32 != 0)


@pytest.mark.parametrize("cuts", CUT_MODES)
@pytest.mark.parametrize("mode", REV_MODES)
def test_shape_a_reaches(mode, cuts):
    ev, w = fuzz.shape_a(mode, cuts)
    c = fuzz.fanout_classes(ev, w)
    assert (c["E"], c["big_t"], c["bm_words"], c["chunks_per_group"]) == (40001, 1024, 1251, 4)
    assert c["W"] % 2 == 1 and 250 <= c["W"] <= 350
    assert c["boundaries"] == [16, 17, 32, 33, 1024, 1025]
    assert c["empty_prefix"] == "large" and len(c["large"]) >= 3  # "", "/g" and the 1 025-match group
    windows = dict(c["medium_windows"])
    assert 1 in windows and 2 in windows and max(windows) >= 3
    assert c["classes"]["none"] >= 3 and c["ends"]
    assert c["n_lens"] >= 14 and max(len(p) for p in w.prefixes.tolist()) > max(len(k) for k in ev.keys.tolist())
    m = fuzz.match_lists(ev.keys.tolist(), [b"/n/", b"/n/in/", b"/n/in/most/"])
    assert [len(m[p]) for p in (b"/n/", b"/n/in/", b"/n/in/most/")] == [45, 15, 5]  # one event matches 3 lengths
    per_prefix = {}
    for p, r in zip(w.prefixes.tolist(), w.min_rev.tolist()):
        per_prefix.setdefault(p, set()).add(r)
    assert sum(len(v) >= 4 for v in per_prefix.values()) >= 5  # several watchers per prefix, different min_revs
    check_revisions(ev, c, mode, cuts)


@pytest.mark.parametrize("cuts", ["b300", "irregular"])
@pytest.mark.parametrize("mode", REV_MODES)
def test_shape_b_reaches(mode, cuts):
    ev, w = fuzz.shape_b(mode, cuts)
    c = fuzz.fanout_classes(ev, w)
    assert (c["E"], c["big_t"], c["chunks_per_group"]) == (200003, 3125, 17)
    assert c["W"] == 2001 and c["empty_prefix"] == "large"
    assert c["boundaries"] == [16, 17, 32, 33, 3125, 3126] and len(c["large"]) >= 4
    assert max(dict(c["medium_windows"])) == 25 and c["ends"]
    check_revisions(ev, c, mode, cuts)


@pytest.mark.parametrize("cuts", ["b300", "irregular"])
def test_shape_c_reaches(cuts):
    ev, w = fuzz.shape_c("random", cuts)
    c = fuzz.fanout_classes(ev, w)
    assert (c["E"], c["W"], c["chunks_per_group"]) == (20000, 20001, 2)
    assert 11000 <= c["G"] <= 13000 and 10 <= c["n_lens"] <= 12
    assert {"half", "warp", "medium", "large", "none"} <= set(c["classes"])
    assert c["boundaries"] == [16, 17, 32, 33]
    check_revisions(ev, c, "random", cuts)


@pytest.mark.parametrize("E", [1, 31, 32, 33])
@pytest.mark.parametrize("W", [1, 2])
def test_shape_tiny(E, W):
    for mode in REV_MODES:
        ev, w = fuzz.shape_tiny(E, W, mode, "irregular")
        assert (ev.n, w.n) == (E, W) and int(ev.batch_off[-1]) == E
        assert len(ev.rev) == E


def test_rotation_keeps_geometry_and_moves_groups():
    bursts, w = fuzz.seq_rotation()
    cs = [fuzz.fanout_classes(ev, w) for ev in bursts]
    # one scratch geometry: the kernel's own cleanup runs between the bursts, not the host's reset
    assert len({(c["E"], c["G"], c["n_lens"], c["W"], c["batches"]) for c in cs}) == 1
    assert [len(c["large"]) for c in cs] == [4, 3, 4, 4, 3, 4]
    assert len({ev.keys.data.tobytes() for ev in bursts}) == len(bursts)
    for a, b in zip(bursts, bursts[1:]):
        ma = fuzz.match_lists(a.keys.tolist(), w.prefixes.tolist())
        mb = fuzz.match_lists(b.keys.tolist(), w.prefixes.tolist())
        big = [p for p in ma if p and fuzz.group_class(len(ma[p]), 1024) == "large"]
        assert any(fuzz.group_class(len(mb[p]), 1024) == "medium" for p in big)  # large in burst k, medium in k+1
    assert not all(c["monotone"] for c in cs) and any(c["monotone"] for c in cs)


def test_regrow_sequence_grows_the_output():
    bursts, w = fuzz.seq_regrow()
    d = [int(ko.fanout(ev, w, threads=4)[0][-1]) for ev in bursts]
    for k in (1, 3):
        assert d[k] > 65536 and d[k] > 1.25 * d[k - 1] + 4096, d
        assert d[k - 1] < 65536, d
