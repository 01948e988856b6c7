"""Point-read latency and throughput on the config-2 store (1M records, 256-byte user keys, 2 KiB values; bench.py's
workload), host clock around calls that return complete answers:
  (a) one Get (n = 1, KB_OUT_HOST): median and p99 over --calls calls
  (b) reads per second of one batch of n random FOUND reads, n = 64, 1 024, 16 384
  (c) one Get submitted while two bench-shaped range batches (1 full Range + 256 List(limit 10 001)) are in flight,
      timed from its submission to its collection (kb_get_submit / _collect; a tree without them: kb_get_batch)
With --baseline-root DIR (another checkout of the project, built by this script), every case is measured in both trees,
in alternating child processes on the same seeded data; the card's name and power limit are read in the same run.  Prints one JSON object (and writes it to --out when given).

usage: python tools/get_probe.py [--baseline-root DIR] [--rounds 2] [--calls 2000] [--out /tmp/get_probe.json]"""
from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                      text=True, timeout=30).strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # the numbers still stand, without the card's name beside them
        return {"error": str(e)}


def stats_us(ts):
    a = np.asarray(ts) * 1e6
    return {"median_us": round(float(np.median(a)), 2), "p99_us": round(float(np.percentile(a, 99)), 2),
            "mean_us": round(float(a.mean()), 2), "calls": len(a)}


def child(root: str, calls: int) -> dict:
    sys.path.insert(0, root)
    import bench
    from kubebrain_b200._lib import KB_OUT_HOST, Engine

    wl = bench.build_workload(0, 1)
    store, reqs = wl["store"], wl["reqs"]
    eng = Engine(0)
    eng.load_sorted(store)
    rng = random.Random(7)
    keys = list(dict.fromkeys(store.keys[i][4:-9] for i in rng.sample(range(store.n), 20000)))
    r = eng.get_batch([(k, 0) for k in keys], KB_OUT_HOST)
    keys = [k for k, s in zip(keys, r.status.tolist()) if s == 0]  # FOUND at the latest revision (not deleted)
    r.close()
    rng = random.Random(1)
    pipelined = hasattr(eng, "get_submit")

    def one_get(k):
        if pipelined:
            r = eng.get_submit([(k, 0)], KB_OUT_HOST).collect()
        else:
            r = eng.get_batch([(k, 0)], KB_OUT_HOST)
        assert int(r.status[0]) == 0
        r.close()

    out = {"tree": "this" if root == HERE else "baseline", "pipelined_get": pipelined, "records": int(store.n),
           "range_requests_per_batch": len(reqs)}
    # warm-up of every shape the timed windows use
    for _ in range(200):
        one_get(keys[rng.randrange(len(keys))])
    for n in (64, 1024, 16384):
        for _ in range(3):
            eng.get_batch([(keys[rng.randrange(len(keys))], 0) for _ in range(n)]).close()
    for _ in range(3):
        a, b = eng.range_submit(reqs), eng.range_submit(reqs)
        one_get(keys[0])
        a.collect().close()
        b.collect().close()

    ts = []
    for _ in range(calls):
        k = keys[rng.randrange(len(keys))]
        t0 = time.perf_counter()
        one_get(k)
        ts.append(time.perf_counter() - t0)
    out["a_one_get"] = stats_us(ts)

    out["b_reads_per_s"] = {}
    for n in (64, 1024, 16384):
        batches = [[(keys[rng.randrange(len(keys))], 0) for _ in range(n)] for _ in range(8)]
        done, t0 = 0, time.perf_counter()
        while time.perf_counter() - t0 < 1.0:
            r = eng.get_batch(batches[done % 8], KB_OUT_HOST)
            r.close()
            done += 1
        dt = time.perf_counter() - t0
        out["b_reads_per_s"][str(n)] = {"reads_per_s": round(done * n / dt), "batches": done, "us_per_batch":
                                        round(dt / done * 1e6, 1)}

    ts = []
    for i in range(max(calls // 10, 100)):
        a, b = eng.range_submit(reqs), eng.range_submit(reqs)
        k = keys[rng.randrange(len(keys))]
        t0 = time.perf_counter()
        one_get(k)
        ts.append(time.perf_counter() - t0)
        a.collect().close()
        b.collect().close()
    out["c_get_beside_two_ranges"] = stats_us(ts)
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-root", default=None, help="another checkout to measure in alternation with this one")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--calls", type=int, default=2000)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", metavar="ROOT", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        print(json.dumps(child(args.child, args.calls)))
        return
    roots = [HERE]
    if args.baseline_root:
        base = os.path.abspath(args.baseline_root)
        subprocess.check_call(["make", "-s", "-C", os.path.join(base, "kubebrain_b200", "csrc"), "-j4"],
                              stdout=subprocess.DEVNULL)
        roots.append(base)
    result = {"card": card(), "workload": "config-2 store of bench.py (1M records, 256 B user keys, 2 KiB values); "
              "(c): two batches of 1 full Range + 256 List(limit 10001) in flight", "runs": []}
    for rnd in range(args.rounds):
        for root in roots:  # alternating trees
            out = subprocess.check_output([sys.executable, os.path.abspath(__file__), "--calls", str(args.calls),
                                           "--child", root], text=True)
            run = json.loads(out.strip().splitlines()[-1])
            run["round"] = rnd
            result["runs"].append(run)
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
