"""What a Verify walk (kb_reconcile chunk by chunk) costs on the config-2 store (200 000 objects x 4 versions + revision
records = 1 000 000 records, 256-byte user keys, 2 KiB values), next to a kb_load_sorted of the same items.

Per placement (HBM / KB_CFG_HOST_VALUES), per case (in sync; 0.1 % and 10 % of the records planted divergent, a third
each changed in the value, deleted from the snapshot and added to it) and per chunk size (4 096, 65 536): the snapshot is
loaded and planted, then [b"", b"\\xff") is walked the way the storage adaptor's Verify walks it (a chunk ends at the
last key + 0x00, the last one at the interval's end) with repair.  Reported: wall seconds of the walk, records/s and
input GB/s (keys + values handed in), split into the host packing of the input, the compare (upload, bound search,
kernels, readbacks; the kernels' own event time beside it) and the apply of the repairs; the diff counts, which must
equal the planted ones.  The split comes from the library's profiling segments, so every kernel is bracketed by CUDA
events during the walks.  The card's name and power limit are read in the same run.  Prints one JSON object (and writes
it to --out when given).

usage: python tools/reconcile_probe.py [--out profiles/h100_reconcile.json]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kubebrain_b200 import synth  # noqa: E402
from kubebrain_b200._lib import Engine, KbReconcileView, lib, u8p, u64p  # noqa: E402
from tools.stream_probe import card  # noqa: E402

START, END = b"", b"\xff"
KERNELS = ("k_search", "k_reconcile_match", "k_reconcile_extra", "k_reconcile_keys")


def plant(store, frac: float, seed: int):
    """(value slab with changed bytes, keys to delete from the snapshot, records to add to it) for `frac` of the records"""
    n = int(store.n)
    k = int(n * frac)
    rng = np.random.default_rng(seed)
    pick = rng.choice(n, size=k, replace=False) if k else np.zeros(0, np.int64)
    chg, dele, ext = pick[0::3], pick[1::3], pick[2::3]
    vdata = store.vals.data.copy()
    voff = store.vals.off
    for i in chg:
        a, b = int(voff[i]), int(voff[i + 1])
        if b > a:
            vdata[a] ^= 0x5A
    keys = store.keys.tolist()
    return vdata, len([i for i in chg if voff[i + 1] > voff[i]]), [keys[i] for i in dele], \
        [(keys[i] + b"~", b"only in the snapshot") for i in ext]


def walk(eng, store, chunk: int):
    """the Verify walk of [START, END) with repair; returns the summed diff counts"""
    L = lib()
    kd, ko = store.keys.data, np.ascontiguousarray(store.keys.off, dtype=np.uint64)
    vd, vo = store.vals.data, np.ascontiguousarray(store.vals.off, dtype=np.uint64)
    kp, vp = kd.ctypes.data_as(u8p), vd.ctypes.data_as(u8p)
    n = int(store.n)
    cur, i = START, 0
    tot = np.zeros(4, np.int64)
    while True:
        m = min(chunk, n - i)
        end = END if m < chunk else bytes(kd[int(ko[i + m - 1]): int(ko[i + m])]) + b"\x00"
        h = C.c_void_p()
        rc = L.kb_reconcile(eng._ctx, cur, len(cur), end, len(end), kp, ko[i:].ctypes.data_as(u64p), vp,
                            vo[i:].ctypes.data_as(u64p), m, 0, C.byref(h))
        eng._check(rc)
        v = KbReconcileView()
        eng._check(L.kb_reconcile_view_get(h, C.byref(v)))
        tot += (v.n_missing, v.n_extra, v.n_changed, v.n_diff)
        L.kb_result_free(eng._ctx, h)
        i += m
        if m < chunk:
            return tot
        cur = end


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--objects", type=int, default=200_000)
    a = ap.parse_args()
    store, _ = synth.gen_store(a.objects, 4, 256, 2048, 1000, config_id=2)
    n = int(store.n)
    in_bytes = int(store.keys.off[-1] - store.keys.off[0] + store.vals.off[-1] - store.vals.off[0])
    res = {"card": card(), "records": n, "input_bytes": in_bytes, "profiling_events": True, "runs": []}
    from kubebrain_b200.packed import PackedStore, Slab
    for hv in (False, True):
        eng = Engine(0, host_values=hv)
        try:
            t0 = time.perf_counter()
            eng.load_sorted(store)
            load_s = time.perf_counter() - t0
            res["runs"].append({"placement": "host" if hv else "device", "case": "kb_load_sorted", "wall_s": load_s,
                                "records_per_s": n / load_s, "input_gb_per_s": in_bytes / load_s / 1e9})
            for frac, case in ((0.0, "in sync"), (0.001, "0.1 %"), (0.1, "10 %")):
                for chunk in (4096, 65536):
                    vdata, n_chg, dels, extra = plant(store, frac, 7)
                    mirror = PackedStore(store.keys, Slab(vdata, store.vals.off))
                    eng.load_sorted(mirror)
                    if dels or extra:
                        eng.apply_batch([(k, None) for k in dels] + extra)
                    eng.prof_enable(1)
                    eng.prof_reset()
                    t0 = time.perf_counter()
                    tot = walk(eng, store, chunk)
                    wall = time.perf_counter() - t0
                    prof = {p["name"]: p for p in eng.prof_read()}
                    eng.prof_enable(0)
                    seg = lambda name: prof.get(name, {"total_ms": 0.0})["total_ms"] / 1e3  # noqa: E731
                    want = (len(dels), len(extra), n_chg)
                    got = tuple(int(x) for x in tot[:3])
                    if got != want:
                        sys.exit("%s %s chunk %d: diff %s, planted %s" % ("host" if hv else "device", case, chunk,
                                                                          got, want))
                    res["runs"].append({
                        "placement": "host" if hv else "device", "case": case, "chunk": chunk, "wall_s": wall,
                        "records_per_s": n / wall, "input_gb_per_s": in_bytes / wall / 1e9,
                        "pack_s": seg("host:reconcile_pack"), "compare_s": seg("host:reconcile_compare"),
                        "kernels_s": sum(seg(k) for k in KERNELS), "apply_s": seg("host:reconcile_apply"),
                        "kernel_ms": {k: prof.get(k, {"total_ms": 0.0})["total_ms"] for k in KERNELS},
                        "missing": got[0], "extra": got[1], "changed": got[2]})
                    print(json.dumps(res["runs"][-1]), flush=True)
        finally:
            eng.close()
    js = json.dumps(res, indent=1)
    print(js)
    if a.out:
        with open(a.out, "w") as f:
            f.write(js + "\n")


if __name__ == "__main__":
    main()
