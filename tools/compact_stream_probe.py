"""Compaction stream of the config-4 store at full size (10 M objects x (1 revision record + 9 versions) = 100 M records,
64-byte user keys and values): the open against kb_compact_sweep alone (alternated), pages of 16 / 64 / 256 MiB (time per
page, export rate against a plain pinned device -> host copy of the same size), and the whole stream with every page's
deletes committed through kb_apply_batch before the next page.  Host clock around synchronised work: every page is in
host memory when kb_compact_stream_next returns.  Prints one JSON object (and writes it to --out when given).

usage: python tools/compact_stream_probe.py [--objects 10000000] [--reps 5] [--out profiles/h100_compact_stream.json]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kubebrain_b200 import synth  # noqa: E402
from kubebrain_b200._lib import KB_OUT_HOST, KbWriteOp, Engine, lib  # noqa: E402
from kubebrain_b200.coder import NormalCoder  # noqa: E402


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                       "--format=csv,noheader"], text=True, timeout=30).strip().splitlines()[0]
        name, power, sm = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock_limit": sm}
    except Exception as e:  # the numbers still stand, without the card's name beside them
        return {"error": str(e)}


def pcie_d2h_gbs(nbytes: int, reps: int) -> float:
    """a plain pinned device -> host copy of nbytes (the ceiling a page export can approach)"""
    import torch

    src = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dst = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    dst.copy_(src)
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        dst.copy_(src)
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return nbytes / float(np.median(ts)) / 1e9


def open_vs_sweep(eng, lo, hi, rev, reps):
    t_open, t_sweep = [], []
    for _ in range(reps):  # alternated
        t0 = time.perf_counter()
        r = eng.compact_sweep(lo, hi, rev, 0, True, KB_OUT_HOST)
        t_sweep.append(time.perf_counter() - t0)
        nv = r.n_victims
        r.close()
        t0 = time.perf_counter()
        s = eng.compact_stream(lo, hi, rev)
        t_open.append(time.perf_counter() - t0)
        s.close()
    return {"victims": int(nv), "sweep_host_ms": 1e3 * float(np.median(t_sweep)),
            "open_ms": 1e3 * float(np.median(t_open)), "sweep_ms_all": [1e3 * t for t in t_sweep],
            "open_ms_all": [1e3 * t for t in t_open]}


def next_raw(eng, stream, budget):
    """one page without the Python copies of CompactPage: (n, bytes) or None"""
    from kubebrain_b200._lib import KbCompactPageView

    r = C.c_void_p()
    eng._check(lib().kb_compact_stream_next(eng._ctx, stream._h, int(budget), C.byref(r)))
    if not r.value:
        return None
    v = KbCompactPageView()
    eng._check(lib().kb_compact_page_view_get(r, C.byref(v)))
    return r, v


def paged(eng, lo, hi, rev, mib, reps):
    ts, pages, nbytes = [], 0, 0
    for _ in range(reps):
        s = eng.compact_stream(lo, hi, rev)
        pages, nbytes, t = 0, 0, 0.0
        while True:
            t0 = time.perf_counter()
            x = next_raw(eng, s, mib << 20)
            t += time.perf_counter() - t0
            if x is None:
                break
            r, v = x
            pages += 1
            nbytes += int(v.n_bytes)
            lib().kb_result_free(eng._ctx, r)
        s.close()
        ts.append(t)
    ms = 1e3 * float(np.median(ts))
    return {"page_mib": mib, "pages": pages, "bytes": nbytes, "ms": ms, "ms_per_page": ms / max(pages, 1),
            "export_gbs": nbytes / (ms / 1e3) / 1e9, "pcie_d2h_gbs": pcie_d2h_gbs(mib << 20, reps)}


WRITE_OP = np.dtype([("type", "<u4"), ("pad", "<u4"), ("key", "<u8"), ("key_len", "<u8"), ("val", "<u8"),
                     ("val_len", "<u8"), ("expire_unix", "<u8")])


def applied(eng, lo, hi, rev, mib):
    """the whole stream with every page's deletes committed (one kb_apply_batch per page) before the next page; nothing
    rewrites a revision record meanwhile, so every DelCurrent guard holds and every victim is deleted"""
    assert WRITE_OP.itemsize == C.sizeof(KbWriteOp)
    n0 = eng.store_info()[0]
    t_next = t_apply = 0.0
    pages = victims = 0
    t_all = time.perf_counter()
    s = eng.compact_stream(lo, hi, rev)
    while True:
        t0 = time.perf_counter()
        x = next_raw(eng, s, mib << 20)
        t_next += time.perf_counter() - t0
        if x is None:
            break
        r, v = x
        n = int(v.n)
        ops = np.zeros(n, WRITE_OP)
        ops["type"] = 1  # KB_OP_DEL
        ops["key"] = int(v.bytes) + np.ctypeslib.as_array(v.key_off, shape=(n,))
        ops["key_len"] = np.ctypeslib.as_array(v.key_len, shape=(n,))
        t0 = time.perf_counter()
        eng._check(lib().kb_apply_batch(eng._ctx, ops.ctypes.data_as(C.POINTER(KbWriteOp)), n))
        t_apply += time.perf_counter() - t0
        lib().kb_result_free(eng._ctx, r)
        pages += 1
        victims += n
    s.close()
    total = time.perf_counter() - t_all
    return {"page_mib": mib, "pages": pages, "victims": victims, "records_before": int(n0),
            "records_after": int(eng.store_info()[0]), "total_s": total, "next_s": t_next, "apply_s": t_apply}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--objects", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    store, meta = synth.gen_store(a.objects, 9, 64, 64, max(1, a.objects // 200), config_id=4, tomb_frac=0.02)
    coder = NormalCoder()
    lo, hi = coder.encode_object_key(b"/registry/", 0), coder.encode_object_key(b"/registry0", 0)
    rev = meta.last_rev
    eng = Engine(0)
    eng.load_sorted(store)
    out = {"card": card(), "records": int(store.n), "reps": a.reps}
    open_vs_sweep(eng, lo, hi, rev, 1)  # warm-up: pools, module load
    out["open"] = open_vs_sweep(eng, lo, hi, rev, a.reps)
    out["paged"] = [paged(eng, lo, hi, rev, mib, a.reps) for mib in (16, 64, 256)]
    out["applied"] = applied(eng, lo, hi, rev, 64)
    eng.close()
    text = json.dumps(out, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
