"""CPU tests of answer-balanced range partitions (kb_range_partitions / kb_partition_view_get): the symbols cross the
boundary, bad arguments are refused before any CUDA call, the view's ctypes layout is gcc's, the reference helper
(tests/partition_shapes.py) agrees with a brute-force restatement, the definition itself keeps every answer whole on
the oracle, and Backend.get_partitions keeps its default answer."""
from __future__ import annotations

import ctypes
import os
import random
import shutil
import subprocess

import pytest

from kubebrain_b200 import _lib, synth
from kubebrain_b200._lib import KB_EINVAL, KB_ELIMIT
from kubebrain_b200.backend import Backend
from kubebrain_b200.coder import NormalCoder
from oracle import binding as ko
from tests import partition_shapes as ps
from tests.test_abi import ROOT, _declared

NAMES = ["kb_range_partitions", "kb_partition_view_get"]


def test_symbols_declared_exported_and_bound():
    assert set(NAMES) <= set(_declared())
    assert set(NAMES) <= set(_lib.ABI_SYMBOLS)
    L = ctypes.CDLL(_lib.LIB_PATH)
    for n in NAMES:
        assert hasattr(L, n)
    assert L.kb_abi_version() == 2


def test_invalid_arguments_need_no_device():
    L = _lib.lib()
    req = (_lib.KbRangeReq * 1)()
    h = ctypes.c_void_p()
    v = _lib.KbPartitionView()
    assert L.kb_range_partitions(None, req, 1 << 20, 64, ctypes.byref(h)) == KB_EINVAL
    assert L.kb_partition_view_get(None, ctypes.byref(v)) == KB_EINVAL
    # every argument check comes before the context is touched: a placeholder handle never gets read
    fake = ctypes.create_string_buffer(64)
    ctx = ctypes.cast(fake, ctypes.c_void_p)
    assert L.kb_range_partitions(ctx, None, 1 << 20, 64, ctypes.byref(h)) == KB_EINVAL
    assert L.kb_range_partitions(ctx, req, 1 << 20, 64, None) == KB_EINVAL
    assert L.kb_range_partitions(ctx, req, 0, 64, ctypes.byref(h)) == KB_EINVAL
    assert L.kb_range_partitions(ctx, req, 1 << 20, 0, ctypes.byref(h)) == KB_EINVAL
    lim = (_lib.KbRangeReq * 1)()
    lim[0].limit = 1
    assert L.kb_range_partitions(ctx, lim, 1 << 20, 64, ctypes.byref(h)) == KB_EINVAL
    bad = (_lib.KbRangeReq * 1)()
    bad[0].end_len = 3  # NULL key with a length
    assert L.kb_range_partitions(ctx, bad, 1 << 20, 64, ctypes.byref(h)) == KB_EINVAL
    assert L.kb_range_partitions(ctx, req, 1 << 20, 4097, ctypes.byref(h)) == KB_ELIMIT
    assert L.kb_range_partitions(ctx, req, 1 << 20, 1 << 40, ctypes.byref(h)) == KB_ELIMIT
    assert h.value is None


def test_partition_view_layout_matches_gcc(tmp_path):
    gcc = shutil.which("gcc")
    if not gcc:
        pytest.skip("no gcc")
    fields = [f for f, _ in _lib.KbPartitionView._fields_]
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "kb_b200.h"\nint main(void){printf("%zu'
           + " %zu" * len(fields) + '\\n",sizeof(kb_partition_view)'
           + "".join(",offsetof(kb_partition_view,%s)" % f for f in fields) + ");return 0;}\n")
    c, exe = tmp_path / "v.c", tmp_path / "v"
    c.write_text(src)
    subprocess.check_call([gcc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    want = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    got = [ctypes.sizeof(_lib.KbPartitionView)] + [getattr(_lib.KbPartitionView, f).offset for f in fields]
    assert got == want


# ---- the helper against a brute-force restatement ----------------------------------------------------------------------
def brute_cuts(sizes, part_bytes, max_parts):
    n, total = len(sizes), sum(sizes)
    p = 1 if n <= 1 else min(max_parts, n, max(1, (total + part_bytes - 1) // part_bytes))
    out = []
    for k in range(1, p):
        cand = [i for i in range(1, n) if sum(sizes[:i]) * p >= k * total]
        if cand and (not out or out[-1] != cand[0]):
            out.append(cand[0])
    return out


@pytest.mark.parametrize("seed", range(40))
def test_helper_equals_brute_force(seed):
    rng = random.Random(seed)
    n = rng.choice([0, 1, 2, 3, rng.randint(4, 60)])
    spread = rng.choice([1, 10, 1000])
    sizes = [16 * rng.randint(2, 2 + spread) for _ in range(n)]
    if n and rng.random() < 0.3:
        sizes[rng.randrange(n)] *= 500  # one kv larger than a share: cuts fall together and are dropped
    total = sum(sizes)
    for part_bytes in (1, 16, max(total // 7, 1), max(total // 2, 1), total or 1, total + 1, 1 << 60):
        for max_parts in (1, 2, 3, 8, 64, ps.MAX_PARTS):
            got = ps.cuts_of(sizes, part_bytes, max_parts)
            assert got == brute_cuts(sizes, part_bytes, max_parts), (sizes, part_bytes, max_parts)
            assert got == sorted(set(got)) and all(0 < i < n for i in got)
            assert len(got) + 1 <= max(1, min(max_parts, n))


def test_empty_interval_is_one_partition():
    assert ps.cuts_of([32] * 10, 16, 8, b"b", b"a") == []
    assert ps.cuts_of([32] * 10, 16, 8, b"a", b"a") == []
    assert ps.cuts_of([32] * 10, 16, 8, b"a", b"b") != []


# ---- the definition on the oracle ----------------------------------------------------------------------------------
def _stores():
    coder = NormalCoder()
    s2, meta = synth.gen_store(1500, 3, 48, 300, 20, config_id=2)
    lo, hi = coder.encode_object_key(b"/registry/", 0), coder.encode_object_key(b"/registry0", 0)
    yield "synth", s2, lo, hi, [meta.read_rev, meta.read_rev // 2 + 500, ps.ALL]
    m = ps.mixed_store()
    yield "mixed", m, coder.encode_object_key(b"/m/", 0), coder.encode_object_key(b"/m0", 0), [ps.READ, 300, ps.ALL]
    u = ps.uniform_store(2050)
    yield "uniform", u, coder.encode_object_key(b"/u/", 0), b"\xff", [ps.READ, 200, ps.ALL]
    lk = ps.long_key_store()
    yield "long_keys", lk, b"", b"\xff", [25, 15, ps.ALL]
    yield "interleaved", ps.q1_store(), b"", b"\xff", list(ps.Q1_REVS)


@pytest.mark.parametrize("name", ["synth", "mixed", "uniform", "long_keys", "interleaved"])
def test_borders_keep_every_answer_whole(name):
    store, lo, hi, revs = next((s, a, b, r) for n, s, a, b, r in _stores() if n == name)
    st = ko.OracleStore(store)
    whole_bytes = ps.partitions(store, st, lo, hi, ps.ALL, 1 << 60, 1)[2][-1]
    for rev in revs:
        for share in (3, 7, 64, 1000):
            borders, kv_first, arena_first = ps.partitions(store, st, lo, hi, rev, max(whole_bytes // share, 1), 64)
            split = ps.check_partitions(store, st, lo, hi, rev, (borders, kv_first, arena_first), revs)
            assert not split or name == "interleaved", (name, rev, share)
            if split:  # a user key's records straddle a border: the answer is whole at the cut's revision only
                continue
            assert all(a < b for a, b in zip(borders, borders[1:])), (name, rev, share)
            assert all(a < b for a, b in zip(kv_first, kv_first[1:])) or len(kv_first) == 2
            assert ko.adjust_partition_borders(borders) == borders
            for r in revs:  # borders cut at one revision keep the answer whole at every revision
                whole = ko.range_(st, lo, hi, r, 0).emit.tolist()
                assert ko.scan(st, borders, r).emit.tolist() == whole, (name, rev, share, r)
                parts = []
                for a, b in zip(borders, borders[1:]):
                    parts += ko.worker_run(st, a, b, r).emit.tolist()
                assert parts == whole, (name, rev, share, r)
            emit = ko.range_(st, lo, hi, rev, 0).emit.tolist()
            for k, (a, b) in enumerate(zip(borders, borders[1:])):  # each partition holds exactly its kvs
                assert ko.worker_run(st, a, b, rev).emit.tolist() == emit[kv_first[k] : kv_first[k + 1]]


# ---- Backend.get_partitions ---------------------------------------------------------------------------------------
class _FakeEngine:
    def __init__(self):
        self.calls = []

    def range_partitions(self, start, end, read_rev, part_bytes, max_parts):
        self.calls.append((start, end, read_rev, part_bytes, max_parts))
        return [start, b"mid", end], [0, 5, 9], [0, 100, 170]


def test_get_partitions_default_is_the_whole_interval():
    eng = _FakeEngine()
    b = Backend(eng)
    c = NormalCoder()
    assert b.get_partitions(b"/a", b"/b") == [c.encode_object_key(b"/a", 0), c.encode_object_key(b"/b", 0)]
    assert eng.calls == []


def test_get_partitions_cuts_on_the_device_when_asked():
    eng = _FakeEngine()
    b = Backend(eng, partition_bytes=1 << 20, max_partitions=16)
    c = NormalCoder()
    s, e = c.encode_object_key(b"/a", 0), c.encode_object_key(b"/b", 0)
    assert b.get_partitions(b"/a", b"/b") == [s, b"mid", e]
    assert eng.calls == [(s, e, 2**64 - 1, 1 << 20, 16)]
