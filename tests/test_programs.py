"""CPU checks of the seeded programs and their model (tests/program_model.py): generation is deterministic, the committed
(seed, KB_LANES) set reaches every hazard class at every lane count, each rule of the model is one that the programs
can tell from a plausible wrong variant (so an engine implementing the variant would fail tests/test_gpu_programs.py),
and on small stores the stream and partition rules agree with a brute-force restatement in plain Python."""
from __future__ import annotations

import functools
import random

import pytest

from tests import program_model as pm
from tests import pyref
from tests.range_shapes import TOMB, be, ik


@functools.lru_cache(maxsize=None)
def program(seed: int, n_lanes: int) -> pm.Program:
    return pm.gen_program(seed, n_lanes)


@functools.lru_cache(maxsize=None)
def run(seed: int, n_lanes: int, variant=None):
    return pm.run_program(program(seed, n_lanes), variant)


def test_generation_is_deterministic():
    a, b = pm.gen_program(3, 2), pm.gen_program(3, 2)
    assert a.start == b.start and a.ops == b.ops
    assert pm.run_program(a)[0] == pm.run_program(b)[0]
    assert pm.gen_program(3, 4).ops != a.ops  # the lane count is part of the seed


def test_programs_use_every_entry_point():
    kinds = {k for s in pm.SEEDS for L in pm.LANES for k, _ in program(s, L).ops}
    assert kinds == {n[3:] for n in dir(pm.Model) if n.startswith("op_")}
    modes = set()
    for s in pm.SEEDS:
        for L in pm.LANES:
            p = program(s, L)
            assert 2000 <= len(p.start) <= 8000 and 120 <= len(p.ops) <= 300
            assert {len(k) for k, _ in p.start} >= {15, 16, 17, 31, 32, 33, 47, 48, 49, 65535}
            modes |= {a["mode"] for k, a in p.ops if k in ("range_batch", "range_submit")}
    assert modes == set(pm.MODES)


@pytest.mark.parametrize("n_lanes", pm.LANES)
def test_every_hazard_class_is_reached(n_lanes):
    reached = set()
    for s in pm.SEEDS:
        reached |= run(s, n_lanes)[1]
    want = set(pm.CLASSES) | (set(pm.MULTI_LANE_CLASSES) if n_lanes > 1 else set())
    assert want <= reached, sorted(want - reached)


@pytest.mark.parametrize("variant", pm.VARIANTS)
def test_each_rule_changes_an_answer(variant):
    """the mutation check, on the model: a wrong variant of one rule changes at least one expected entry"""
    for s in pm.SEEDS:
        for L in pm.LANES:
            if run(s, L)[0] != run(s, L, variant)[0]:
                return
    pytest.fail("variant %s changes no answer of the committed programs" % variant)


# ---- brute force on small stores --------------------------------------------------------------------------------------
def _small(seed: int):
    rng = random.Random(seed)
    items = {}
    for j in range(40):
        uk = b"/s/%02d" % j + (b"x" * rng.randint(0, 30))
        revs = sorted(rng.sample(range(1, 30), rng.randint(1, 3)))
        items[ik(uk, 0)] = be(revs[-1], rng.random() < 0.1)
        for r in revs:
            items[ik(uk, r)] = TOMB if rng.random() < 0.15 else b"v%d" % r * rng.randint(0, 6)
    items[ik(pm.LONG_UK, 0)] = be(5)
    items[ik(pm.LONG_UK, 5)] = b"long"
    return items


def _brute_answer(items, start, end, rev):
    keys = sorted(items)
    run_ = pyref.worker_run(keys, [items[k] for k in keys], start, end, rev)
    return [keys[i] for i in run_.emit]


@pytest.mark.parametrize("seed", range(4))
def test_stream_rescan_agrees_with_brute_force(seed):
    """R4 on a small store: the pages handed out, then (after a write) the kvs of the new snapshot's whole answer that
    lie behind the last one handed out -- a filter of the full answer, not a re-scan"""
    items = _small(seed)
    rng = random.Random(seed)
    for rev in (pm.ALL, 12):
        for group, budget in ((1, 0), (3, 200), (2, 10**9)):
            p = pm.Program(seed, 1, sorted(items.items()))
            req = (pm.FULL[0], pm.FULL[1], rev, 0)
            p.ops.append(("stream_open", {"req": req, "mode": "host", "group": group, "h": "s"}))
            p.ops.append(("stream_next", {"h": "s", "budget": budget}))
            keys = sorted(items)
            ops = [(rng.choice(keys), None) for _ in range(4)]
            ops += [(ik(b"/s/%02d" % rng.randrange(40) + b"new", rng.randint(1, 30)), b"w") for _ in range(4)]
            p.ops.append(("apply", {"ops": ops}))
            p.ops += [("stream_next", {"h": "s", "budget": budget})] * 60
            t, _ = pm.run_program(p)
            pages = [e for e in t[1:] if isinstance(e, dict)]
            first = pages[0]["rec"]
            old_keys = sorted(items)
            handed = [old_keys[i] for i in first]
            assert handed == _brute_answer(items, req[0], req[1], rev)[: len(first)]
            new = dict(items)
            for k, v in ops:
                if v is None:
                    new.pop(k, None)
                else:
                    new[k] = v
            new_keys = sorted(new)
            rest = [new_keys[i] for e in pages[1:] for i in e["rec"]]
            assert rest == [k for k in _brute_answer(new, req[0], req[1], rev) if k > handed[-1]]


def _brute_partitions(items, start, end, rev, part_bytes, max_parts):
    keys = _brute_answer(items, start, end, rev)
    sizes = [len(pm.pad16(k)) + len(pm.pad16(items[k])) for k in keys]
    n, total = len(sizes), sum(sizes)
    P = 1 if n <= 1 or start >= end else min(max_parts, n, max(1, -(-total // part_bytes)))
    cuts = []
    for k in range(1, P):
        i = next((i for i in range(1, n) if sum(sizes[:i]) * P >= k * total), None)
        if i is not None and (not cuts or cuts[-1] != i):
            cuts.append(i)
    borders = [start] + [keys[i][:-8] + b"\x00" * 8 for i in cuts] + [end]
    return borders, [0] + cuts + [n], [0] + [sum(sizes[:i]) for i in cuts] + [total]


@pytest.mark.parametrize("seed", range(4))
def test_partitions_agree_with_brute_force(seed):
    """R6 on a small store: the model's partitions equal a linear restatement of the header's definition, also with a
    compact revision above the read revision (there is no compact-race check)"""
    items = _small(seed)
    p = pm.Program(seed, 1, sorted(items.items()))
    cases = [(pm.FULL[0], pm.FULL[1], rev, pb, mp) for rev in (pm.ALL, 12, 3) for pb in (1, 100, 1000, 10**6)
             for mp in (1, 3, 4096)]
    p.ops.append(("set_compact_revision", {"rev": 20}))
    for c in cases:
        p.ops.append(("partitions", dict(zip(("start", "end", "rev", "part_bytes", "max_parts"), c))))
    t, _ = pm.run_program(p)
    for c, e in zip(cases, t[1:]):
        b, kf, af = _brute_partitions(items, *c)
        assert (e["borders"], e["kv_first"], e["arena_first"]) == (b, kf, af), c


def test_key_after():
    assert pm.key_after(b"abc") == b"abc\x00"
    k = b"k" * (pm.MAX_KEY - 2) + b"a\xff"
    assert pm.key_after(k) == b"k" * (pm.MAX_KEY - 2) + b"b"
    assert pm.key_after(b"\xff" * pm.MAX_KEY) is None
