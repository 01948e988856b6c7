"""Range batches in flight on every lane count (KB_LANES = 1 .. 4), against the CPU oracle: submitted batches answer
exactly like the oracle in any collection order, in every output mode, while the other entry points -- which run on
the current lane's stream and staging -- are called between submission and collection; a pending can be given up, a
context can be closed with batches still in flight, and every lane is reused many times."""
from __future__ import annotations

import numpy as np
import pytest

from kubebrain_b200 import synth
from kubebrain_b200._lib import KB_OUT_COUNT, KB_OUT_DEVICE, KB_OUT_HOST, KB_WIRE_ETCD_KVS, Engine
from kubebrain_b200.coder import NormalCoder, prefix_end
from kubebrain_b200.packed import PackedStore
from oracle import binding as ko
from tests.test_gpu_parity import check_gets, check_ranges
from tests.test_gpu_round2 import _check_result

pytestmark = pytest.mark.gpu

CODER = NormalCoder()
LO, HI = CODER.encode_object_key(b"/registry/", 0), CODER.encode_object_key(b"/registry0", 0)
WIRE_HOST = KB_OUT_HOST | KB_WIRE_ETCD_KVS


def _check_device(eng, r, store, st, reqs):
    """a KB_OUT_DEVICE answer: per-kv arrays and arena bytes read back from the device"""
    arr = {name: r.device_array(name, dt) for name, dt in (("rec_idx", np.uint32), ("rev", np.uint64), ("key_off", np.uint64),
                                                           ("key_len", np.uint32), ("val_off", np.uint64), ("val_len", np.uint32))}
    arena = eng.read_device(r.bytes_ptr, r.n_bytes, sync=False)
    for q, (s, e, rev, lim) in enumerate(reqs):
        exp = ko.range_(st, s, e, rev, lim)
        a, b = int(r.req_first[q]), int(r.req_first[q + 1])
        assert arr["rec_idx"][a:b].astype(np.uint64).tolist() == exp.emit.tolist(), (q, rev, lim)
        assert int(r.req_count[q]) == exp.count and int(r.req_examined[q]) == exp.examined, q
        kvs = []
        for k in range(a, b):
            ko_, kl, vo, vl = int(arr["key_off"][k]), int(arr["key_len"][k]), int(arr["val_off"][k]), int(arr["val_len"][k])
            kvs.append((arena[ko_ : ko_ + kl], arena[vo : vo + vl], int(arr["rev"][k])))
        assert kvs == exp.kvs(store), (q, "kv bytes")


def _check_any(eng, r, store, st, reqs, mode):
    if mode == KB_OUT_DEVICE:
        _check_device(eng, r, store, st, reqs)
    elif mode == WIRE_HOST:
        (s, e, rev, lim), = reqs
        exp = ko.range_(st, s, e, rev, lim)
        body, off = ko.wire_encode(st, exp.emit, ko.WIRE_KVS)
        assert r.rec_idx.astype(np.uint64).tolist() == exp.emit.tolist()
        assert r.arena.tobytes() == body and r.elem_off.tolist() == off.tolist(), "wire elements"
    else:
        _check_result(r, store, st, reqs)
    r.close()


@pytest.mark.parametrize("n_lanes", [1, 2, 3, 4])
def test_lanes(monkeypatch, n_lanes):
    monkeypatch.setenv("KB_LANES", str(n_lanes))  # kb_open reads it every time
    store, meta = synth.gen_store(6000, 4, 64, 90, 9, config_id=2, tomb_frac=0.1)
    p = b"/registry/pods/ns-00002/"
    ps, pe = CODER.encode_object_key(p, 0), CODER.encode_object_key(prefix_end(p), 0)
    a = [(LO, HI, meta.read_rev, 0), (ps, pe, meta.last_rev, 5), (HI, HI, meta.last_rev, 0)]  # a limit, an empty interval
    b = [(LO, HI, meta.last_rev, 7), (LO, HI, meta.first_rev, 0)]
    c = [(LO, HI, meta.last_rev, 0)]
    w = [(ps, pe, meta.last_rev, 0)]
    specs = [(a, KB_OUT_HOST), (w, WIRE_HOST), (b, KB_OUT_DEVICE), (c, KB_OUT_HOST), (b, KB_OUT_HOST)]
    ev = synth.gen_events(3000, 256, 60, 5000)
    wat = synth.gen_watchers(50, 4, 5000, 6500)
    fan_start, fan_idx, _ = ko.fanout(ev, wat, threads=2)
    m = n_lanes + 1  # one more batch than lanes: a submission first reads back the rows of its lane's previous batch

    eng = Engine(0)
    eng.load_sorted(store)
    eng.watch_add_many(wat)
    items = dict(zip(store.keys.tolist(), store.vals.tolist()))
    cur, st = store, ko.OracleStore(store)
    victims = iter(sorted(items)[100::400])
    for first in (0, 2):
        batches = (specs[first:] + specs[:first])[:m]
        for order in (list(range(m)), list(range(m))[::-1], list(range(0, m, 2)) + list(range(1, m, 2))):
            pend = [eng.range_submit(x, mode) for x, mode in batches]
            # entry points that only take the current lane (no quiesce): the fan-out on a host slab and on an uploaded one
            got = eng.watch_match(ev)
            assert got.start.tolist() == fan_start.tolist() and got.event_idx.tolist() == fan_idx.tolist()
            got.close()
            h = eng.events_upload(ev)
            d = eng.watch_match_dev(h, KB_OUT_DEVICE)
            assert d.start.tolist() == fan_start.tolist() and d.device_event_idx().tolist() == fan_idx.tolist()
            d.close()
            eng.events_free(h)
            # entry points that read every batch in flight back first, on the snapshot the batches were submitted on
            check_gets(eng, cur, st, [(cur.keys[i][4:-9], 0) for i in range(0, cur.n, 997)] + [(b"/registry/none", 0)])
            exp = ko.scan(st, [LO, HI], meta.read_rev, compact=True, collect=False)
            cs = eng.compact_sweep(LO, HI, meta.read_rev, out_mode=KB_OUT_COUNT)
            assert (cs.n_victims, cs.count, cs.examined) == (len(exp.victims), exp.count, exp.examined)
            cs.close()
            eng.set_compact_revision(None)
            eng.range_prefetch(a)
            check_ranges(eng, cur, st, a)
            k = next(victims)
            eng.apply_batch([(k, None)])
            for i in order:
                _check_any(eng, pend[i].collect(), cur, st, *batches[i])
            items.pop(k)
            cur = PackedStore.from_items(list(items.items()))
            st = ko.OracleStore(cur)

    # a pending given up, then one collected
    pa = eng.range_submit(a, KB_OUT_HOST)
    pgone = eng.range_submit(b, KB_OUT_DEVICE)
    pgone.close()
    with pytest.raises(Exception):
        pgone.collect()
    _check_any(eng, pa.collect(), cur, st, a, KB_OUT_HOST)

    # every lane reused many times at full depth
    q = [eng.range_submit(specs[i % 2 * 3][0], KB_OUT_HOST) for i in range(n_lanes)]
    for i in range(50):
        q.append(eng.range_submit(specs[(n_lanes + i) % 2 * 3][0], KB_OUT_HOST))
        _check_any(eng, q.pop(0).collect(), cur, st, specs[i % 2 * 3][0], KB_OUT_HOST)
    for i, p_ in enumerate(q):
        _check_any(eng, p_.collect(), cur, st, specs[(50 + i) % 2 * 3][0], KB_OUT_HOST)

    # closed with two batches uncollected; a new context answers
    left = [eng.range_submit(a, KB_OUT_HOST), eng.range_submit(c, KB_OUT_DEVICE)]
    eng.close()
    del left
    e2 = Engine(0)
    e2.load_sorted(cur)
    _check_any(e2, e2.range_submit(a, KB_OUT_HOST).collect(), cur, st, a, KB_OUT_HOST)
    e2.close()
