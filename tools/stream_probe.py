"""Full-range stream of the config-2 store (1M records, 256-byte user keys, 2 KiB values) at 4, 16 and 64 MiB pages,
in host and EVENTS modes, against one unlimited kb_range_batch of the same range.  Host clock around synchronised
work: every page is complete (host copy done) when kb_range_stream_next returns; the device-resident EVENTS pages are
waited for before the clock stops.  Prints one JSON object (and writes it to --out when given).

usage: python tools/stream_probe.py [--reps 5] [--out /tmp/stream_probe.json]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kubebrain_b200 import synth  # noqa: E402
from kubebrain_b200._lib import KB_OUT_HOST, KB_WIRE_ETCD_EVENTS, Engine  # noqa: E402
from kubebrain_b200.coder import NormalCoder  # noqa: E402


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                      text=True, timeout=30).strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # the numbers still stand, without the card's name beside them
        return {"error": str(e)}


def one_shot(eng, req, mode, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = eng.range_batch([req], mode)
        if r.on_device:
            r.wait()
        ts.append(time.perf_counter() - t0)
        n, nb = r.n_kvs, r.n_bytes
        r.close()
    return {"ms": 1e3 * float(np.median(ts)), "kvs": n, "bytes": nb}


def streamed(eng, req, mode, page_bytes, reps):
    ts, pages, largest = [], 0, 0
    for _ in range(reps):
        t0 = time.perf_counter()
        s = eng.range_stream(req, mode, 300)
        pages = 0
        while True:
            p = s.next(page_bytes)
            if p is None:
                break
            if p.on_device:
                p.wait()
            pages += 1
            largest = max(largest, p.n_bytes)
            p.close()
        s.close()
        ts.append(time.perf_counter() - t0)
    ms = 1e3 * float(np.median(ts))
    return {"page_mib": page_bytes >> 20, "ms": ms, "pages": pages, "ms_per_page": ms / max(pages, 1),
            "largest_page_bytes": largest}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    store, meta = synth.gen_store(200000, 4, 256, 2048, 1000, config_id=2)
    coder = NormalCoder()
    req = (coder.encode_object_key(b"/registry/", 0), coder.encode_object_key(b"/registry0", 0), meta.read_rev, 0)
    klen = np.diff(store.keys.off.astype(np.int64))
    vlen = np.diff(store.vals.off.astype(np.int64))
    padded_store = int((((klen + 15) // 16) + ((vlen + 15) // 16)).sum() * 16)
    eng = Engine(0)
    eng.load_sorted(store)
    out = {"card": card(), "records": int(store.n),
           "one_shot_arena_bound_bytes": padded_store,  # kb_range_batch's arena for a range over the whole store
           "modes": {}}
    for name, mode in (("host", KB_OUT_HOST), ("events", KB_OUT_HOST | KB_WIRE_ETCD_EVENTS)):
        one_shot(eng, req, mode, 1)  # warm-up: pools, module load
        streamed(eng, req, mode, 16 << 20, 1)
        res = {"one_shot": one_shot(eng, req, mode, a.reps)}
        res["paged"] = [streamed(eng, req, mode, mb << 20, a.reps) for mb in (4, 16, 64)]
        out["modes"][name] = res
    eng.close()
    text = json.dumps(out, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
