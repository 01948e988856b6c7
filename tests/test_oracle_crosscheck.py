"""The C oracle against an independent pure-Python restatement of the same reference loop (tests/pyref.py) on
adversarial stores: emitted records, counts, examined records, the limit-stop quirk, ordered delete calls with their
classes, TTL expiry.  Neither file was derived from the other; both cite the reference lines they follow."""
from __future__ import annotations

import pytest

from oracle import binding as ko
from tests import fuzz, pyref, range_shapes


def _check(store, st, keys, vals, s, e, rev, lim, compact, timeout=0, support_ttl=True):
    exp = pyref.worker_run(keys, vals, s, e, rev, lim, compact, timeout, support_ttl)
    got = ko.worker_run(st, s, e, rev, lim, compact=compact, timeout_rev=timeout, support_ttl=support_ttl,
                        collect=not compact)
    if exp.error:
        assert got.rc != 0
        return
    assert got.rc == 0
    ctx = (s, e, rev, lim, compact, timeout, support_ttl)
    assert got.emit.tolist() == exp.emit, ctx
    assert got.examined == exp.examined, ctx
    assert got.limit_stop == exp.limit_stop, ctx
    assert got.count == exp.count, ctx
    assert list(zip(got.victims.tolist(), got.vclass.tolist())) == exp.victims, ctx


@pytest.mark.parametrize("seed", range(16))
def test_range_and_compaction_agree(seed):
    store = fuzz.fuzz_store(7000 + seed, n_keys=30 + 12 * seed)
    st = ko.OracleStore(store)
    keys, vals = store.keys.tolist(), store.vals.tolist()
    for s, e in fuzz.fuzz_bounds(store, seed):
        if s > e:
            continue
        for rev in (0, 7, 23, 41, 59, 2**64 - 1):
            for lim in (0, 1, 2, 5, 40):
                _check(store, st, keys, vals, s, e, rev, lim, compact=False)
            _check(store, st, keys, vals, s, e, rev, 0, compact=True)
            for timeout in (11, 35):
                _check(store, st, keys, vals, s, e, rev, 0, compact=True, timeout=timeout, support_ttl=False)
                _check(store, st, keys, vals, s, e, rev, 0, compact=True, timeout=timeout, support_ttl=True)


@pytest.mark.parametrize("start", ["s0", "s255", "reach_back"])
def test_r1_seam_shapes_agree(start):
    """tests/range_shapes.py R1 at reduced size: non-PREVOK runs up to 257 records and over 2 tiles, every seam record"""
    sh = range_shapes.r1_store(5, lens=(0, 1, 31, 32, 255, 256, 257), long_tiles=2)
    store, st = sh.store, ko.OracleStore(sh.store)
    keys, vals = store.keys.tolist(), store.vals.tolist()
    s, e, R, T = sh.starts[start], sh.end, range_shapes.READ, range_shapes.TTL
    for lim in (0, 3):
        _check(store, st, keys, vals, s, e, R, lim, compact=False)
    _check(store, st, keys, vals, s, e, T - 50, 0, compact=False)
    _check(store, st, keys, vals, s, e, R, 0, compact=True)
    _check(store, st, keys, vals, s, e, R, 0, compact=True, timeout=T, support_ttl=False)


def test_r2_limit_shapes_agree():
    """tests/range_shapes.py R2: limits reached in probe rounds 0-2, by a trailing emission, never, and total +- 1"""
    store = range_shapes.r2_store()
    st = ko.OracleStore(store)
    keys, vals = store.keys.tolist(), store.vals.tolist()
    for s, e, rev, lim in range_shapes.r2_requests(store).values():
        _check(store, st, keys, vals, s, e, rev, lim, compact=False)


def test_decode_agrees():
    cases = [b"", b"\x57\xfb\x80\x8b", b"\x57\xfb\x80\x8b$" + b"\x00" * 8, b"\x57\xfb\x80\x8ba$" + b"\x00" * 7 + b"\x05",
             b"\x57\xfb\x80\x8ca$" + b"\x00" * 8, b"\x57\xfb\x80\x8ba%" + b"\x00" * 8, b"x" * 12, b"x" * 13]
    for k in cases:
        uk, rev, err = ko.decode(k)
        try:
            euk, erev = pyref.decode(k)
            assert err == 0 and (uk, rev) == (euk, erev), k
        except pyref.DecodeError:
            assert err != 0, k


def _fanout_shape(case: str):
    """the fan-out's exact-group-size shapes (large groups, non-monotone and empty batches) at reduced watcher counts"""
    kind, mode, cuts = case.split("-")
    if kind == "A":
        ev, w = fuzz.shape_a(mode, cuts)
        return ev, fuzz.take_watchers(w, 31)
    if kind == "B":
        ev, w = fuzz.shape_b(mode, cuts)
        return ev, fuzz.take_watchers(w, 13)
    if kind == "C":
        ev, w = fuzz.shape_c(mode, cuts)
        return ev, fuzz.take_watchers(w, 41)
    return fuzz.shape_tiny(int(kind[1:]), 2, mode, cuts)


SHAPE_CASES = (["A-%s-%s" % (m, c) for m in fuzz.REV_MODES for c in ("b300", "irregular")] +
               ["B-random-irregular", "B-stepback-b300", "C-runs-irregular", "E1-random-irregular",
                "E33-stepback-irregular"])


@pytest.mark.parametrize("seed", list(range(12)) + SHAPE_CASES)
def test_fanout_agrees(seed):
    if isinstance(seed, str):
        ev, w = _fanout_shape(seed)
    else:
        ev = fuzz.fuzz_events(40 + seed, n=80 + 50 * seed, monotone=(seed % 2 == 0))
        w = fuzz.fuzz_watchers(ev, seed, n=8 + 6 * seed)
    lists, messages = pyref.fanout(ev.keys.tolist(), ev.rev.tolist(), ev.batch_off.tolist(), w.prefixes.tolist(),
                                   w.min_rev.tolist())
    start, idx, msgs = ko.fanout(ev, w)
    assert msgs == messages
    for i, exp in enumerate(lists):
        assert idx[int(start[i]) : int(start[i + 1])].tolist() == exp, i
    start4, idx4, msgs4 = ko.fanout(ev, w, threads=4, alloc_per_batch=True)  # the timing variant gives the same answer
    assert (start4.tolist(), idx4.tolist(), msgs4) == (start.tolist(), idx.tolist(), msgs)


@pytest.mark.parametrize("seed", range(10))
def test_get_agrees(seed):
    store = fuzz.fuzz_store(7100 + seed, n_keys=40 + 10 * seed)
    st = ko.OracleStore(store)
    keys, vals = store.keys.tolist(), store.vals.tolist()
    uks = set()
    for k in keys:
        try:
            uk, _ = pyref.decode(k)
        except pyref.DecodeError:
            continue
        uks.update((uk, uk + b"$", uk[:-1], uk + b"\x00"))
    for uk in sorted(uks):
        for rev in (0, 1, 9, 17, 33, 58, 59, 2**63, 2**64 - 1):
            assert ko.get(st, uk, rev) == pyref.get(keys, vals, uk, rev), (uk, rev)
