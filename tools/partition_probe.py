"""Cost of kb_range_partitions on the config-2 store (1M records, 256-byte user keys, 2 KiB values): the full range cut at
16, 64 and 256 MiB partitions, alternated call by call with a KB_OUT_COUNT batch of the same interval (the Count the
cut is expected to cost about as much as, plus placement).  Host clock around each call: both return with their answer
on the host.  Reports the partition count, per-partition arena bytes, the median and p90 microseconds per call, and the
card's name and power limit.  Prints one JSON object (and writes it to --out when given).

usage: python tools/partition_probe.py [--reps 20] [--out /tmp/partition_probe.json]"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kubebrain_b200 import synth  # noqa: E402
from kubebrain_b200._lib import KB_OUT_COUNT, Engine  # noqa: E402
from kubebrain_b200.coder import NormalCoder  # noqa: E402
from tools.stream_probe import card  # noqa: E402


def stats(ts):
    us = 1e6 * np.array(ts)
    return {"median_us": float(np.median(us)), "p90_us": float(np.percentile(us, 90)), "calls": len(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    store, meta = synth.gen_store(200000, 4, 256, 2048, 1000, config_id=2)
    coder = NormalCoder()
    s, e = coder.encode_object_key(b"/registry/", 0), coder.encode_object_key(b"/registry0", 0)
    eng = Engine(0)
    eng.load_sorted(store)
    out = {"card": card(), "records": int(store.n), "read_rev": int(meta.read_rev), "cases": []}
    for mib in (16, 64, 256):
        part_bytes = mib << 20
        eng.range_partitions(s, e, meta.read_rev, part_bytes, 64)  # warm-up: pools, module load, report buffer
        eng.range_batch([(s, e, meta.read_rev, 0)], KB_OUT_COUNT).close()
        tp, tc = [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            borders, kv_first, arena_first = eng.range_partitions(s, e, meta.read_rev, part_bytes, 64)
            tp.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            r = eng.range_batch([(s, e, meta.read_rev, 0)], KB_OUT_COUNT)
            tc.append(time.perf_counter() - t0)
            count = int(r.req_count[0])
            r.close()
        assert int(kv_first[-1]) == count
        out["cases"].append({"partition_mib": mib, "partitions": len(borders) - 1, "kvs": count,
                             "answer_bytes": int(arena_first[-1]),
                             "partition_bytes": np.diff(arena_first.astype(np.int64)).tolist(),
                             "partition_kvs": np.diff(kv_first.astype(np.int64)).tolist(),
                             "range_partitions": stats(tp), "count_batch": stats(tc)})
    eng.close()
    text = json.dumps(out, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
