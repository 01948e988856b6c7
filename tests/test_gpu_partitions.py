"""kb_range_partitions against the reference helper (tests/partition_shapes.py) and the C oracle: the device's cuts,
arena offsets and border bytes are the helper's exactly, every partition's range stream and unlimited range batch
concatenate to the whole answer at several revisions, the call interleaves with batches in flight and open streams
without touching the snapshot, and Backend.get_partitions serves the reference's partitionsTestcase."""
from __future__ import annotations

import os

import pytest

from kubebrain_b200 import synth
from kubebrain_b200._lib import KB_OUT_COUNT, KB_OUT_HOST, Engine
from kubebrain_b200.backend import Backend
from kubebrain_b200.coder import NormalCoder
from kubebrain_b200.packed import PackedStore
from oracle import binding as ko
from tests import partition_shapes as ps
from tests.range_shapes import ik
from tests.refmodel import MiniBackend

pytestmark = pytest.mark.gpu

ALL = ps.ALL
coder = NormalCoder()


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def check(eng, store, st, s, e, rev, part_bytes, max_parts, what=""):
    borders, kv_first, arena_first = ps.partitions(store, st, s, e, rev, part_bytes, max_parts)
    got = eng.range_partitions(s, e, rev, part_bytes, max_parts)
    assert got[1].tolist() == kv_first, (what, "kv_first")
    assert got[2].tolist() == arena_first, (what, "arena_first")
    assert got[0] == borders, (what, "borders")
    return borders, kv_first


def stream_recs(eng, s, e, rev):
    out = []
    stream = eng.range_stream((s, e, rev, 0), KB_OUT_HOST, 300)
    while True:
        page = stream.next(1 << 20)
        if page is None:
            break
        out += page.rec_idx.tolist()
        page.close()
    stream.close()
    return out


def answers_whole(eng, st, borders, revs, streams=True):
    s, e = borders[0], borders[-1]
    reqs = lambda r: [(a, b, r, 0) for a, b in zip(borders, borders[1:])]
    for r in revs:
        whole = ko.range_(st, s, e, r, 0).emit.tolist()
        res = eng.range_batch(reqs(r))
        got = []
        for q in range(res.n_req):
            got += res.rec_indices(q).tolist()
        res.close()
        assert got == whole, ("batch", r)
        cnt = eng.range_batch(reqs(r), KB_OUT_COUNT)
        one = eng.range_batch([(s, e, r, 0)], KB_OUT_COUNT)
        assert int(cnt.req_count.sum()) == int(one.req_count[0])
        cnt.close()
        one.close()
        if streams:
            got = []
            for a, b in zip(borders, borders[1:]):
                got += stream_recs(eng, a, b, r)
            assert got == whole, ("stream", r)


def _load(eng, store):
    eng.load_sorted(store)
    return ko.OracleStore(store)


# ---- shapes --------------------------------------------------------------------------------------------------------
def test_small_answers(eng):
    store = ps.uniform_store(3)
    st = _load(eng, store)
    k = [ik(b"/u/o%07d" % j, 0) for j in range(4)]
    for n in range(4):  # n = 0 .. 3 kvs
        for pb in (1, 16, 1 << 30):
            b, _ = check(eng, store, st, k[0], k[n], 500, pb, 64, n)
            answers_whole(eng, st, b, [500, ALL])
    # start >= end: one partition, the interval itself
    for s, e in ((k[2], k[0]), (k[1], k[1])):
        assert eng.range_partitions(s, e, ALL, 1, 64)[0] == [s, e]


@pytest.mark.parametrize("n", [2046, 2048, 2050])
def test_cuts_on_tile_edges(eng, n):
    store = ps.uniform_store(4200)
    st = _load(eng, store)
    s, e = ik(b"/u/o%07d" % 0, 0), ik(b"/u/o%07d" % n, 0)
    total = ps.partitions(store, st, s, e, ALL, 1 << 60, 1)[2][-1]
    _, kv_first = check(eng, store, st, s, e, ALL, total // 2, 64)
    assert kv_first[1] == {2046: 1023, 2048: 1024, 2050: 1025}[n]
    b, _ = check(eng, store, st, s, e, ALL, total // 4, 64)
    answers_whole(eng, st, b, [ALL, 300])


def test_clamps(eng):
    store = ps.uniform_store(4200)
    st = _load(eng, store)
    s, e = ik(b"/u/", 0), b"\xff"
    total = ps.partitions(store, st, s, e, ALL, 1 << 60, 1)[2][-1]
    for pb, mp, parts in ((total, 64, 1), (total + 1, 64, 1), (1 << 62, 4096, 1), (1, 3, 3), (1, 4096, 4096),
                          (total // 100, 64, 64), (total // 100, 100, 100)):
        b, _ = check(eng, store, st, s, e, ALL, pb, mp, (pb, mp))
        assert len(b) - 1 == parts, (pb, mp)
    few = ik(b"/u/o%07d" % 5, 0)
    b, _ = check(eng, store, st, s, few, ALL, 1, 64)  # the n clamp
    assert len(b) - 1 == 5
    answers_whole(eng, st, b, [ALL])


@pytest.mark.parametrize("rev", [ps.READ, 300, 1500, ALL])
def test_mixed_history(eng, rev):
    """hidden versions, tombstoned last versions, revision-record-only keys, undecodable records beside the cuts,
    user keys that prefix others, and kvs larger than a share (dropped cuts)"""
    store = ps.mixed_store()
    st = _load(eng, store)
    s, e = coder.encode_object_key(b"/m/", 0), coder.encode_object_key(b"/m0", 0)
    total = ps.partitions(store, st, s, e, rev, 1 << 60, 1)[2][-1]
    dropped = False
    for share in (2, 7, 64, 300):
        b, kv_first = check(eng, store, st, s, e, rev, max(total // share, 1), 64, share)
        dropped |= len(b) - 1 < min(share, 64)
        if share in (7, 64):
            answers_whole(eng, st, b, [rev, 300, ALL])
    if rev == ps.READ:
        assert dropped


def test_long_keys(eng):
    store = ps.long_key_store()
    st = _load(eng, store)
    longest = 0
    for pb in (1, 50_000, 200_000):
        b, _ = check(eng, store, st, b"", b"\xff", ALL, pb, 64, pb)
        answers_whole(eng, st, b, [ALL, 25])
        longest = max([longest] + [len(x) for x in b])
    assert longest == 65535


# ---- interleaving --------------------------------------------------------------------------------------------------
def test_interleaves_with_batches_and_streams(eng):
    store, meta = synth.gen_store(20000, 3, 64, 400, 50, config_id=2)
    st = _load(eng, store)
    s, e = coder.encode_object_key(b"/registry/", 0), coder.encode_object_key(b"/registry0", 0)
    rev = meta.read_rev
    info = eng.store_info()
    want = ps.partitions(store, st, s, e, rev, 1 << 20, 64)
    reqs = [(s, e, rev, 0), (s, e, rev, 77)]
    # between kb_range_submit and kb_range_collect of batches on other lanes
    p1 = eng.range_submit(reqs)
    p2 = eng.range_submit(reqs[::-1])
    got = eng.range_partitions(s, e, rev, 1 << 20, 64)
    r1, r2 = p1.collect(), p2.collect()
    assert got[0] == want[0] and got[1].tolist() == want[1]
    for q, (a, b, r, lim) in enumerate(reqs):
        exp = ko.range_(st, a, b, r, lim).emit.tolist()
        assert r1.rec_indices(q).tolist() == exp and r2.rec_indices(1 - q).tolist() == exp
    r1.close()
    r2.close()
    # with a range stream and a compaction stream open
    rs = eng.range_stream((s, e, rev, 0), KB_OUT_HOST, 300)
    first = rs.next(1 << 20)
    cs = eng.compact_stream(s, e, meta.last_rev)
    got = eng.range_partitions(s, e, rev, 1 << 20, 64)
    assert got[0] == want[0] and got[2].tolist() == want[2]
    recs = first.rec_idx.tolist()
    first.close()
    while True:
        p = rs.next(1 << 20)
        if p is None:
            break
        recs += p.rec_idx.tolist()
        p.close()
    rs.close()
    assert recs == ko.range_(st, s, e, rev, 0).emit.tolist()
    exp = ko.scan(st, [s, e], meta.last_rev, compact=True, collect=False)
    assert cs.n_victims == len(exp.victims)
    cs.close()
    assert eng.store_info() == info
    # the sweep recorded its compact revision, above the read revision: GetPartitions makes no checkCompactRace
    got = eng.range_partitions(s, e, rev, 1 << 20, 64)
    assert got[0] == want[0]
    eng.set_compact_revision(None)
    # after kb_apply_batch: the new snapshot's answer
    keys = store.keys.tolist()
    ops = [(keys[7], None), (keys[100], b"x" * 5000), (keys[2000] + b"\x01", b"inserted")]
    eng.apply_batch(ops)
    items = dict(zip(keys, store.vals.tolist()))
    for k, v in ops:
        if v is None:
            items.pop(k)
        else:
            items[k] = v
    cur = PackedStore.from_items(list(items.items()))
    cst = ko.OracleStore(cur)
    b, _ = check(eng, cur, cst, s, e, ALL, 1 << 20, 64, "after apply")
    answers_whole(eng, cst, b, [ALL, rev], streams=False)


def test_config2_full_range(eng):
    store, meta = synth.gen_store(200000, 4, 256, 2048, 1000, config_id=2)
    st = _load(eng, store)
    s, e = coder.encode_object_key(b"/registry/", 0), coder.encode_object_key(b"/registry0", 0)
    b, kv_first = check(eng, store, st, s, e, meta.read_rev, 64 << 20, 64)
    assert len(b) > 2
    answers_whole(eng, st, b, [meta.read_rev], streams=False)


# ---- the reference's partitionsTestcase (backend_test.go:502-533, 883-899) through Backend -----------------------------
@pytest.mark.parametrize("partition_bytes", [0, 1, 100, 1 << 20])
def test_reference_partitions_testcase(eng, partition_bytes):
    inject = 10
    mb = MiniBackend(1_700_000_000)
    test_key = b"/registry/test/key"
    fmt = lambda p, i: p + b"/" + (b"%05d" % i)
    kv_list = []
    for i in range(inject):
        rev, ok = mb.create(fmt(test_key, i), fmt(b"val", i))
        assert ok
        kv_list.append((fmt(test_key, i), fmt(b"val", i), rev))
    eng.load_sorted(mb.snapshot())
    b = Backend(eng, partition_bytes=partition_bytes)
    b.set_current_revision(mb.rev)
    for end, want in ((ko.prefix_end(test_key), kv_list), (fmt(test_key, inject - 2), kv_list[: inject - 2])):
        borders = b.get_partitions(test_key, end)
        if partition_bytes == 0:
            assert len(borders) == 2
        kvs = []
        for i in range(1, len(borders)):
            for wr in b.list_by_stream(borders[i - 1], borders[i], 0):
                kvs += [(kv.key, kv.value, kv.revision) for kv in wr.kvs]
        assert sorted(kvs) == sorted(want)
        if partition_bytes == 1:
            assert len(borders) - 1 == len(want)


# ---- the storage adaptor's call sequence ----------------------------------------------------------------------------
def test_partitions_replay_cpp(tmp_path):
    """tests/cpp/partitions_replay_test.cpp, compiled here against the in-tree library and the oracle"""
    import shutil
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    gxx = shutil.which("g++")
    assert gxx, "the replay driver needs a C++ compiler"
    libdir, oradir = os.path.join(root, "kubebrain_b200"), os.path.join(root, "oracle")
    ko.build()
    exe = str(tmp_path / "partitions_replay_test")
    subprocess.check_call([gxx, "-O1", "-std=c++17", "-Wall", "-o", exe,
                           os.path.join(root, "tests", "cpp", "partitions_replay_test.cpp"),
                           "-L" + libdir, "-lkbb200", "-L" + oradir, "-lkboracle",
                           "-Wl,-rpath," + libdir, "-Wl,-rpath," + oradir])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "partitions replay OK" in r.stdout, r.stdout + r.stderr
