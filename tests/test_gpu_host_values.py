"""The value heap in mapped pinned host memory (KB_CFG_HOST_VALUES): every answer, view, error code and dump image is
the one the HBM placement gives.

- the seeded programs of tests/program_model.py (every entry point interleaved with writes, expiry, streams, dumps and
  restores) on a host-placement engine at every lane count, against the model;
- the boundary suites of the range scan, bound searches and point reads, write path, compaction sweep and stream, and
  partitions, run as they are with every engine they use opened in host placement.  The 4 GiB answer shapes are left
  out: they measure arena offsets, not where the values live;
- dumps of one history from the two placements are byte-identical, and each restores into the other placement with the
  same answers in every output mode;
- kb_store_mem: where the bytes are."""
from __future__ import annotations

import functools
import inspect
import struct

import numpy as np
import pytest

from kubebrain_b200 import synth
from kubebrain_b200._lib import (KB_ESTATE, KB_OUT_DEVICE, KB_OUT_HOST, KB_WIRE_ETCD_EVENTS, KB_WIRE_ETCD_KVS, Engine,
                                 KbError)
from kubebrain_b200.packed import PackedStore
from tests import test_gpu_compact_shapes as tcs
from tests import test_gpu_compact_stream as gcs
from tests import test_gpu_lookup_shapes as tls
from tests import test_gpu_partition_shapes as tpq
from tests import test_gpu_partitions as tps
from tests import test_gpu_programs as tgp
from tests import test_gpu_range_shapes as trs
from tests import test_gpu_write_shapes as tws
# module fixtures of the suites, resolved here by name when a suite's test asks for them
from tests.test_gpu_compact_shapes import big, k4  # noqa: F401
from tests.test_gpu_compact_stream import cases  # noqa: F401
from tests.test_gpu_lookup_shapes import p2  # noqa: F401
from tests.test_gpu_range_shapes import r1  # noqa: F401

pytestmark = pytest.mark.gpu

HostEngine = functools.partial(Engine, host_values=True)


@pytest.fixture
def eng():
    e = HostEngine(0)
    yield e
    e.close()


@pytest.fixture
def engs():
    a, b = HostEngine(0), HostEngine(0)
    yield a, b
    a.close()
    b.close()


def _param_sets(fn):
    """every parameter set pytest runs `fn` with, from its parametrize marks"""
    sets = [{}]
    for mark in getattr(fn, "pytestmark", []):
        if mark.name != "parametrize":
            continue
        names = mark.args[0]
        names = [a.strip() for a in names.split(",")] if isinstance(names, str) else list(names)
        values = [v.values if hasattr(v, "values") else v for v in mark.args[1]]
        sets = [{**s, **dict(zip(names, v if len(names) > 1 else (v,)))} for s in sets for v in values]
    return sets


def _cases(mod, names):
    short = mod.__name__.rsplit(".", 1)[1]
    out = []
    for name in names:
        for params in _param_sets(getattr(mod, name)):
            pid = ",".join("%s=%s" % (k, v if not isinstance(v, bytes) else v[:8]) for k, v in sorted(params.items()))
            out.append(pytest.param(mod, name, params, id="%s::%s[%s]" % (short, name, pid)))
    return out


SUITES = (
    _cases(trs, ["test_r1_seams", "test_r1_sweep", "test_r2_limit_windows", "test_r3_pairs_and_point_reads",
                 "test_wire_room", "test_sequence_two_in_flight", "test_fuzz_store_tiles", "test_synthetic_key_lengths"])
    + _cases(tls, ["test_s1_pivots", "test_s1_emptied_store", "test_s2_compare_chunks", "test_p1_resolve",
                   "test_p2_finalize_chunks", "test_p2_one_record_read_many_times", "test_c_range_stream_every_cut",
                   "test_c_compact_stream_every_cut"])
    + _cases(tws, ["test_write_shape", "test_write_shape_large", "test_empty_value_replacement_dumps_canonically",
                   "test_batches_between_submit_and_collect", "test_invalid_ops_change_nothing"])
    + _cases(tcs, ["test_k1_classes", "test_k1_streams", "test_k1_none_and_every", "test_k2_tiles",
                   "test_k2_chain_2n_minus_1", "test_k2_every_record_two_calls",
                   "test_k2_one_sweep_across_the_tile_scan_chunk", "test_k3_comparisons",
                   "test_k3_expired_runs_on_tile_seams", "test_k4_capture_counts", "test_k4_entries",
                   "test_k6_device_answers_held_across_sweeps"])
    + _cases(gcs, ["test_pages_concatenate_to_the_victims", "test_config4_ttl_sweeps", "test_apply_pages_as_they_arrive",
                   "test_backend_compact_apply", "test_layout_compaction_deferred_while_open",
                   "test_heap_rewrite_invalidates", "test_close_context_with_open_streams", "test_edges",
                   "test_pages_between_batches_and_point_reads"])
    + _cases(tps, ["test_small_answers", "test_cuts_on_tile_edges", "test_clamps", "test_mixed_history",
                   "test_long_keys", "test_interleaves_with_batches_and_streams", "test_config2_full_range",
                   "test_reference_partitions_testcase"])
    + _cases(tpq, ["test_q1_key_order", "test_q2_search", "test_q2_equal_bumped_big_and_unreached",
                   "test_q3_warps_and_clamps", "test_q4_key_lengths", "test_q4_report_regrows_on_one_engine",
                   "test_q5_snapshots"])
    + _cases(tgp, ["test_program"])
)


@pytest.mark.parametrize("mod,name,params", SUITES)
def test_suite_in_host_placement(request, monkeypatch, mod, name, params):
    """one test of a boundary suite (or one seeded program) with every engine in host placement: the `eng` / `engs`
    fixtures here, and the suite module's own Engine for the engines a test opens itself"""
    monkeypatch.setattr(mod, "Engine", HostEngine)
    fn = getattr(mod, name)
    kwargs = {a: params[a] if a in params else request.getfixturevalue(a) for a in inspect.signature(fn).parameters}
    fn(**kwargs)


# ---- one history in both placements ---------------------------------------------------------------------------------
LO, HI = b"", b"\xff" * 4
MODES = [KB_OUT_HOST, KB_OUT_DEVICE, KB_OUT_HOST | KB_WIRE_ETCD_KVS, KB_OUT_DEVICE | KB_WIRE_ETCD_KVS,
         KB_OUT_HOST | KB_WIRE_ETCD_EVENTS, KB_OUT_DEVICE | KB_WIRE_ETCD_EVENTS]


def _history(eng: Engine, store: PackedStore):
    """load, a batch with deletes, replacements and inserts, a TTL expiry, another batch: the layout ends out of order"""
    eng.load_sorted(store)
    keys = store.keys.tolist()
    ops = [(keys[i], None) for i in range(0, len(keys), 9)]
    ops += [(keys[i], b"r" * (i % 300)) for i in range(4, len(keys), 13)]
    ops += [(keys[7][:-8] + struct.pack(">Q", 2**40 + i), b"i%d" % i * (i % 40), 1000 if i % 3 == 0 else 0)
            for i in range(60)]
    eng.apply_batch(ops)
    dropped = eng.expire(1000)
    eng.apply_batch([(keys[i], b"\x09" * 5000) for i in range(2, len(keys), 97)])
    return dropped


def _answer(eng: Engine, reqs, mode: int):
    r = eng.range_batch(reqs, mode)
    rows = (r.req_first.tolist(), r.req_count.tolist(), r.req_examined.tolist())
    if r.on_device:
        rec = r.device_array("rec_idx", np.uint32).tolist()
        arena = eng.read_device(r.bytes_ptr, r.n_bytes, sync=False)
        eo = r.device_array("elem_off", np.uint64).tolist() if mode & 0x30 and r.n_kvs else None
    else:
        rec, arena = r.rec_idx.tolist(), r.arena[: r.n_bytes].tobytes()
        eo = r.elem_off.tolist() if mode & 0x30 and r.n_kvs else None
    r.close()
    return rows, rec, arena, eo


def test_dumps_match_and_restore_across_placements(tmp_path):
    store, meta = synth.gen_store(2500, 4, 128, 1500, 20, config_id=2)
    dev, host = Engine(0), HostEngine(0)
    dev2, host2 = Engine(0), HostEngine(0)
    try:
        assert _history(dev, store) == _history(host, store) > 0
        for e in (dev, host):
            e.set_compact_revision(None)
        assert dev.store_info() == host.store_info()
        pd, ph = str(tmp_path / "dev.kbd"), str(tmp_path / "host.kbd")
        dev.dump(pd)
        host.dump(ph)
        blob = open(pd, "rb").read()
        assert blob == open(ph, "rb").read(), "the placements dump different files"
        host2.restore(pd)  # device dump -> host placement
        dev2.restore(ph)   # host dump -> device placement
        reqs = [(LO, HI, meta.read_rev, 0), (LO, HI, 2**64 - 1, 301), (LO, HI, meta.first_rev, 0)]
        for mode in MODES:
            want = _answer(dev, reqs, mode)
            for e in (host, host2, dev2):
                assert _answer(e, reqs, mode) == want, hex(mode)
        # the restored contexts keep accepting writes, and dump the same file again
        for e in (dev2, host2):
            e.apply_batch([(store.keys.tolist()[3], b"again")])
        dev2.dump(pd)
        host2.dump(ph)
        assert open(pd, "rb").read() == open(ph, "rb").read()
    finally:
        for e in (dev, host, dev2, host2):
            e.close()


def test_store_mem_by_placement():
    """equal keys, 16 B against 4 KiB values: the HBM bytes of a host-placement store do not depend on its values"""
    keys = [b"\x57\xfb\x80\x8b/registry/pods/p%06d" % i + b"\x24" + struct.pack(">Q", 5) for i in range(3000)]
    small = PackedStore.from_items([(k, b"s" * 16) for k in keys])
    large = PackedStore.from_items([(k, b"L" * 4096) for k in keys])
    got = {}
    for host_values in (False, True):
        for name, store in (("small", small), ("large", large)):
            e = Engine(0, host_values=host_values)
            try:
                with pytest.raises(KbError) as ei:
                    e.store_mem()
                assert ei.value.code == KB_ESTATE
                e.load_sorted(store)
                got[host_values, name] = e.store_mem()
            finally:
                e.close()
    assert got[False, "small"][1] == 0 and got[False, "large"][1] == 0
    assert got[True, "small"][0] == got[True, "large"][0]
    assert got[True, "large"][1] >= 3000 * 4096 and got[True, "small"][1] >= 3000 * 16
    # device placement holds the same key slab and directory plus the heap
    assert got[False, "large"][0] == got[True, "large"][0] + got[True, "large"][1]
