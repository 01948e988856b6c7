"""The write shapes (tests/write_shapes.py) reach the boundaries of the write path they are built for, and the heap
model and the dump-image restatement agree with hand-worked cases.  The GPU tests in tests/test_gpu_write_shapes.py
compare kb_apply_batch / kb_expire / kb_dump with them; they can only fail on a wrong boundary if the shape puts
something on it, so a change to a builder that stops reaching a class fails here, on any host.  Every class is derived
from the bytes and the model, not from the builders' bookkeeping."""
from __future__ import annotations

import struct

import pytest

from tests import write_shapes as ws


@pytest.fixture(scope="module")
def classes():
    return {sh.name: ws.shape_classes(sh) for sh in ws.all_shapes(slow=True)}


def test_w1_merge_and_fix_list(classes):
    c = ws.merged(classes["W1 merge"][0])
    for k in ("lb0", "lbN", "ins_on_deleted", "del_0", "del_last", "del_then_put", "put_then_del",
              "rep_behind_ins", "rep_all", "del_all", "ins_into_empty"):
        assert c[k], k
    assert all(ws.merged(classes["W1 N=%d" % n][0])["del_0_ins_0"] for n in (255, 256, 257))
    assert {1, 2, 31, 32, 33, 257} <= c["per_bound"]
    big = ws.merged(classes["W1 200k"][0])
    assert big["more_ins_than_N"] and big["per_bound"] == {200}
    assert big["merge_threads"][0] == 201_000
    threads = set()
    for n in (255, 256, 257):
        cl = classes["W1 N=%d" % n][0]
        assert [x["merge_threads"] for x in cl[:2]] == [n, n + 1]  # n_ins 0 and 1
        threads |= {x["merge_threads"] for x in cl}
    b = ws.MERGE_BLOCK  # one thread short of a block, on it, one and two past it
    assert {b - 1, b, b + 1, b + 2} <= threads


def test_w2_key_bytes(classes):
    c = ws.merged(classes["W2 keys"][0])
    assert {0, 1, 12, 13, 16, 17, 511, 512, 513, 1024, ws.MAX_KEY - 1, ws.MAX_KEY} <= c["op_klens"]
    assert {0, 31, 32, 33, "last"} <= c["near_chunk"]  # k_key_exists's first, second and third pass
    assert {"prefix", "extends", "extends_nul"} <= c["prefix"]
    for t in ws.LCP_TARGETS:
        for how in ("insert", "delete", "replace"):
            assert (t, how) in c["lcp"], (t, how)
    assert {0, 1, 2} <= c["lcp_pass"]  # summarize_record finds the first difference in its first, second, third pass
    assert {0, 31, 32, 33, 63, 64, "last", "into$"} <= c["events_at"]


def test_w3_trigger_at_threshold_and_one_past(classes):
    for name, big in (("W3 displaced floor", False), ("W3 displaced N/32", True)):
        cl = classes[name][0]
        assert [x["displaced_vs_threshold"] for x in cl[:2]] == [0, 1], name
        assert [x["fired"] for x in cl[:2]] == [None, ("displaced",)], name
        assert cl[0]["big_branch"] == big and cl[1]["big_branch"] == big
        gk, gv = cl[0]["garbage"]
        assert gk > 0 and gv > 0 and cl[0]["gk_vs_quarter"] < 0 and cl[0]["gv_vs_quarter"] < 0, name
    k = classes["W3 garbage keys"][0]
    assert [x["gk_vs_quarter"] for x in k[:2]] == [0, ws.GARBAGE_DIV] and [x["fired"] for x in k[:2]] == [None, ("garbage_k",)]
    v = classes["W3 garbage values"][0]
    assert [x["gv_vs_quarter"] for x in v[:2]] == [0, ws.GARBAGE_DIV] and [x["fired"] for x in v[:2]] == [None, ("garbage_v",)]
    p = classes["W3 pinned"][0]
    assert p[0]["pinned"] and p[0]["gk_vs_quarter"] > 0 and p[0]["fired"] is None
    assert not p[1]["pinned"] and p[1]["fired"] == ("garbage_k",)  # the first batch after the stream closed


def _infos(shape, threshold):
    """kb_store_info after every step of a shape, predicted by a model whose displaced threshold is `threshold`"""
    m = ws.HeapModel(shape.start)
    m.threshold = threshold
    out = []
    for s in shape.steps:
        m.apply(s.ops)
        out.append(m.info())
    return out


@pytest.mark.parametrize("variant", ["fires at the threshold", "never", "no floor", "N / 16"])
def test_w3_store_info_tells_a_wrong_displaced_trigger(variant):
    """The GPU tests see the trigger only through kb_store_info.  A trigger that is off by one, never fires or takes
    the wrong branch of max(4096, N / 32) must predict other numbers than the right one on some displaced shape."""
    wrong = {"fires at the threshold": lambda n2: max(ws.DISPLACED_FLOOR, n2 // ws.DISPLACED_DIV) - 1,
             "never": lambda n2: 2**64,
             "no floor": lambda n2: n2 // ws.DISPLACED_DIV,
             "N / 16": lambda n2: max(ws.DISPLACED_FLOOR, n2 // 16)}[variant]
    shapes = [s for s in ws.w3_heap() if s.name.startswith("W3 displaced")]
    differs = [_infos(s, wrong) != _infos(s, ws.HeapModel(s.start).threshold) for s in shapes]
    want = {"fires at the threshold": [True, True], "never": [True, True], "no floor": [True, False],
            "N / 16": [False, True]}[variant]
    assert differs == want


def test_w3_growth_and_empty_values(classes):
    _, m = classes["W3 growth"]
    assert m.grows_k >= 3 and m.grows_v >= 3  # slab_reserve grows each slab several times
    sh = [s for s in ws.w3_heap() if s.name == "W3 empty values"][0]
    m = ws.HeapModel(sh.start)
    keys = sorted(m.items)
    for s in sh.steps[:3]:
        (k, v), = s.ops
        assert m.items[k] == b"" and ws.chunks(len(m.items[k])) == 0  # replaces an empty value
        f = m.apply(s.ops)
        assert f["n_rep"] == 1 and f["garbage_v"] == 0 and f["displaced"] == 0 and f["fired"] is None
    assert [keys.index(s.ops[0][0]) for s in sh.steps[:3]] == [3, 6, len(keys) - 1]  # not the last record, and the last


def test_w4_ttl(classes):
    cl = classes["W4 ttl"][0]
    ex = [x for x in cl if x.get("expire")]
    assert ex[0]["dropped"] == 0 and ex[1]["dropped"] == 40 and ex[1]["at_now"] == 40  # 40 due at exactly t
    assert any(x["stale"] for x in ex)
    assert ex[-1]["emptied"]
    assert [x["reinstall"] for x in cl if "reinstall" in x] == ["reload", "restore"]
    assert all(x["dropped_ttls"] for x in cl if "reinstall" in x)
    c = ws.merged(cl)
    assert c["del_then_put"] and c["put_then_del"]


# ---- the model on hand-worked cases ---------------------------------------------------------------------------------
def test_model_hand_worked():
    a, b, c = b"a" * 16, b"b" * 17, b"c"
    m = ws.HeapModel([(a, b"x" * 20), (c, b"")])
    assert m.info() == (2, 32, 32)  # keys 1 + 1 chunks, values 2 + 0
    f = m.apply([(b, b"yy")])  # an insert appends both: key 2 chunks, value 1
    assert m.info() == (3, 64, 48) and f["n_ins"] == 1 and f["displaced"] == 1 and f["fired"] is None
    f = m.apply([(c, b"z" * 33)])  # replacement: 3 value chunks appended, the old value (0 chunks) is garbage
    assert m.info() == (3, 64, 96) and f["garbage_v"] == 0 and f["fired"] is None
    f = m.apply([(b"absent", None), (b"other", None)])  # only absent deletes: nothing changes
    assert m.info() == (3, 64, 96) and f["n_del"] == 0 and "threshold" not in f
    f = m.apply([(b, b"q"), (b, None), (a, b"new")])  # last op per key wins: b deleted, a replaced
    # garbage_k = 2 (b's key) of a key tail of 4: 8 > 4; garbage_v = 1 (b's value) + 2 (a's old value) of a value
    # tail of 6 + 1: 12 > 7
    assert f["n_del"] == 1 and f["n_rep"] == 1 and f["garbage_k"] == 2 and f["garbage_v"] == 3 and f["vtail"] == 7
    assert f["ktail"] == 4 and f["fired"] == ("garbage_k", "garbage_v")
    assert m.info() == (2, 32, 16 + 48)  # compacted: a (1 + 1), c (1 + 3)
    m.apply([(a, b"t", 100), (c, b"u", 100), (a, b"t2", 200)])  # a re-put later: its 100 entry is stale
    assert m.expire(99)[0] == 0 and m.expire(100)[0] == 1 and m.expire(200)[0] == 1 and not m.items


def test_model_threshold_solver():
    for n in (0, 1000, 131_072, 140_000, 1_000_000):
        t = ws._solve_threshold(n)
        assert t == max(ws.DISPLACED_FLOOR, (n + t) // 32) and t + 1 > max(ws.DISPLACED_FLOOR, (n + t + 1) // 32)


# ---- the dump image ---------------------------------------------------------------------------------------------------
def test_fnv_words():
    assert ws.fnv1a64_words(ws.FNV_OFFSET, b"") == ws.FNV_OFFSET
    w = 0x0807060504030201
    assert ws.fnv1a64_words(ws.FNV_OFFSET, bytes(range(1, 9))) == ((ws.FNV_OFFSET ^ w) * ws.FNV_PRIME) % 2**64
    h = ((ws.FNV_OFFSET ^ w) * ws.FNV_PRIME) % 2**64
    assert ws.fnv1a64_words(ws.FNV_OFFSET, bytes(range(1, 10))) == ((h ^ 9) * ws.FNV_PRIME) % 2**64


@pytest.mark.parametrize("n", [0, 1, 2, 7])
def test_dump_roundtrip(n):
    items = sorted((ws.ik(b"/d/%02d" % i + b"k" * (i * 9), i), b"v" * (i * 7)) for i in range(n))
    img = ws.dump_image(items, compact_rev=17 if n & 1 else None)
    d = ws.parse_dump(img)
    assert d.sums_ok and d.items() == items
    h = d.header
    assert h["magic"] == ws.DUMP_MAGIC and h["version"] == 1 and h["header_bytes"] == 88 and h["n"] == n
    assert (h["compact_present"], h["compact_rev"]) == ((1, 17) if n & 1 else (0, 0))
    assert h["key_chunks"] == sum(ws.chunks(len(k)) for k, _ in items) == d.koff16[-1]
    assert h["val_chunks"] == sum(ws.chunks(len(v)) for _, v in items) == d.voff16[-1]
    assert h["max_kv_chunks"] == max((ws.chunks(len(k)) + ws.chunks(len(v)) for k, v in items), default=0)
    # the directory is contiguous, the padding zero
    assert all(d.koff16[i + 1] - d.koff16[i] == ws.chunks(d.klen[i]) for i in range(n))
    assert all(d.voff16[i + 1] - d.voff16[i] == ws.chunks(d.vlen[i]) for i in range(n))
    assert d.kslab == b"".join(ws.pad16(k) for k, _ in items)
    assert len(img) == 88 + 4 * (n + 1) + 2 * n + 8 * (n + 1) + 4 * n + len(d.kslab) + len(d.vslab)
    if n:  # a flipped byte anywhere behind the header breaks a sum
        for at in (88, len(img) - 1):
            bad = img[:at] + bytes([img[at] ^ 1]) + img[at + 1:]
            assert not ws.parse_dump(bad).sums_ok


def test_dump_header_layout():
    img = ws.dump_image([(b"k", b"v")], max_kv_chunks=9)
    assert img[:8] == b"KBB200D1" and struct.unpack_from("<II", img, 8) == (1, 88)
    assert struct.unpack_from("<I", img, 56)[0] == 9  # max_kv_chunks behind n, both chunk counts and the compact record
