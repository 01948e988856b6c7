"""What keeping the value heap in mapped pinned host memory (KB_CFG_HOST_VALUES) costs on the config-2 store (200 000
objects x 4 versions + revision records, 256-byte user keys, 2 KiB values), against the HBM placement, in one run.

The store is loaded in each placement in turn, the order alternating over --rounds rounds (one engine alive at a time).
Per placement and round: load seconds and kb_store_mem; range-batch throughput (the bench's batch: the full range plus
256 namespace Lists of limit 10 001) in KB_OUT_HOST and KB_OUT_DEVICE; single-List latency (one namespace List) in
both; one write-path batch of 300 CAS + Put pairs; a forced layout compaction (one batch of inserts past the displaced
trigger) with k_relocate's event time; dump and restore seconds; SHA-256 digests of the answers' arenas (raw, etcd KVS
wire, device-resident) and of the dump file, which must be equal between the placements.  Host clock around calls that
end with their answer complete (KB_OUT_DEVICE: after kb_result_wait).  The card's name and power limit are read in the
same run.  Prints one JSON object (and writes it to --out when given).

usage: python tools/host_values_probe.py [--rounds 2] [--reps 10] [--out profiles/h100_host_values.json]"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import struct
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kubebrain_b200 import synth  # noqa: E402
from kubebrain_b200._lib import KB_OUT_DEVICE, KB_OUT_HOST, KB_WIRE_ETCD_KVS, Engine  # noqa: E402
from kubebrain_b200.coder import NormalCoder, prefix_end  # noqa: E402
from tools.stream_probe import card  # noqa: E402

CODER = NormalCoder()


def stats(ts):
    ms = 1e3 * np.array(ts)
    return {"median_ms": float(np.median(ms)), "p90_ms": float(np.percentile(ms, 90)), "calls": len(ts)}


def workload():
    store, meta = synth.gen_store(200_000, 4, 256, 2048, 1000, config_id=2)
    lo, hi = CODER.encode_object_key(b"/registry/", 0), CODER.encode_object_key(b"/registry0", 0)
    reqs = [(lo, hi, meta.read_rev, 0)]
    resn = [b"pods", b"configmaps", b"secrets", b"services", b"deployments", b"events"]
    for i in range(256):
        p = b"/registry/" + resn[i % 6] + b"/ns-%05d/" % ((i * 7) % 1000)
        reqs.append((CODER.encode_object_key(p, 0), CODER.encode_object_key(prefix_end(p), 0), meta.read_rev, 10001))
    return store, meta, reqs


def timed_batch(eng, reqs, mode, reps):
    """seconds per call, kvs and answer bytes of range_batch(reqs, mode); the answer is complete when the clock stops"""
    ts = []
    for _ in range(reps + 1):
        t0 = time.perf_counter()
        r = eng.range_batch(reqs, mode)
        if r.on_device:
            r.wait()
        ts.append(time.perf_counter() - t0)
        kvs, nb = r.n_kvs, r.n_bytes
        r.close()
    return ts[1:], kvs, nb  # the first call warms the pools


def digest(eng, reqs, mode) -> str:
    r = eng.range_batch(reqs, mode)
    if r.on_device:
        r.wait()
        raw = eng.read_device(r.bytes_ptr, r.n_bytes, sync=False)
    else:
        raw = r.arena[: r.n_bytes].tobytes()
    r.close()
    return hashlib.sha256(raw).hexdigest()


def one_placement(store, meta, reqs, host_values: bool, reps: int, tmp: str):
    out = {}
    eng = Engine(0, host_values=host_values)
    try:
        t0 = time.perf_counter()
        eng.load_sorted(store)
        out["load_s"] = time.perf_counter() - t0
        d, h = eng.store_mem()
        out["store_mem"] = {"device_bytes": d, "host_bytes": h}
        full = reqs[:1]
        out["digests"] = {"raw_host": digest(eng, full, KB_OUT_HOST),
                          "kvs_host": digest(eng, full, KB_OUT_HOST | KB_WIRE_ETCD_KVS),
                          "raw_device": digest(eng, full, KB_OUT_DEVICE)}
        for name, mode in (("host", KB_OUT_HOST), ("device", KB_OUT_DEVICE)):
            ts, kvs, nb = timed_batch(eng, reqs, mode, reps)
            out["range_batch_" + name] = {**stats(ts), "kvs": kvs, "answer_bytes": nb,
                                          "answer_gb_per_s": nb / float(np.median(ts)) / 1e9}
            ts1, kvs1, nb1 = timed_batch(eng, reqs[1:2], mode, 5 * reps)
            out["single_list_" + name] = {**stats(ts1), "kvs": kvs1, "answer_bytes": nb1}
        # the write path: 300 CAS(revision record) + Put(object record) pairs with 2 KiB values
        keys = store.keys.tolist()
        rev_keys = [k for k in keys if k.endswith(b"\0" * 8)]
        tw = []
        for b in range(reps):
            ops = []
            for i in range(150):
                k = rev_keys[(b * 150 + i) * 7 % len(rev_keys)]
                ops.append((k, struct.pack(">Q", meta.last_rev + 1 + b * 150 + i)))
                ops.append((k[:-8] + struct.pack(">Q", meta.last_rev + 1 + b * 150 + i), b"w" * 2048))
            t0 = time.perf_counter()
            eng.apply_batch(ops)
            tw.append(time.perf_counter() - t0)
        out["write_batch_300"] = stats(tw)
        # forced layout compaction: inserts past the displaced trigger (N / 32 records appended out of key order)
        n = eng.store_info()[0]
        ins = [(keys[i * 13 % len(keys)][:-8] + struct.pack(">Q", 2**48 + i), b"x" * 64) for i in range(n // 32 + 4096)]
        eng.prof_enable(1)
        eng.prof_reset()
        t0 = time.perf_counter()
        eng.apply_batch(ins)
        t_apply = time.perf_counter() - t0
        prof = {p["name"]: p for p in eng.prof_read()}
        eng.prof_enable(0)
        rel = prof.get("k_relocate", {"launches": 0, "total_ms": 0.0, "alg_bytes": 0})
        out["layout_compaction"] = {"apply_s": t_apply, "k_relocate_launches": rel["launches"],
                                    "k_relocate_ms": rel["total_ms"], "k_relocate_alg_bytes": rel["alg_bytes"]}
        path = os.path.join(tmp, "probe.kbd")
        t0 = time.perf_counter()
        eng.dump(path)
        out["dump_s"] = time.perf_counter() - t0
        with open(path, "rb") as f:
            out["digests"]["dump"] = hashlib.file_digest(f, "sha256").hexdigest()
        out["dump_bytes"] = os.path.getsize(path)
    finally:
        eng.close()
    eng = Engine(0, host_values=host_values)
    try:
        t0 = time.perf_counter()
        eng.restore(path)
        out["restore_s"] = time.perf_counter() - t0
        out["digests"]["restored_raw_host"] = digest(eng, reqs[:1], KB_OUT_HOST)
    finally:
        eng.close()
        os.remove(path)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    store, meta, reqs = workload()
    res = {"card": card(), "records": int(store.n), "key_bytes": int(store.keys.off[-1]),
           "value_bytes": int(store.vals.off[-1]), "rounds": []}
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(a.rounds):
            order = (False, True) if r % 2 == 0 else (True, False)
            rnd = {}
            for hv in order:
                rnd["host" if hv else "device"] = one_placement(store, meta, reqs, hv, a.reps, tmp)
            res["rounds"].append({"order": ["host" if hv else "device" for hv in order], **rnd})
    res["digests_equal"] = all(x["host"]["digests"] == x["device"]["digests"] for x in res["rounds"])
    js = json.dumps(res, indent=1)
    print(js)
    if a.out:
        with open(a.out, "w") as f:
            f.write(js + "\n")
    if not res["digests_equal"]:
        sys.exit("the placements answered differently")


if __name__ == "__main__":
    main()
