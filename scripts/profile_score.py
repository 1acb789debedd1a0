#!/usr/bin/env python
"""Where the time of one scoring call goes: warmed clp_score_euclidean_dev calls (score tile + compact build) at the
bench workloads, per kernel, against the bytes each kernel must move.

  python scripts/profile_score.py [--workloads c2,c4] [--calls 10] [--warmup 3] [--trace DIR]

Per workload: the call time by CUDA events with the profiler off, then the same calls under torch.profiler (CUDA
activities) for the per-kernel device time.  Bytes per kernel are computed from m, clp_sparse_info and the row counts:
  score_tile_kernel          4 m^2 written (the dense fp32 store)
  sparse_fill_items_kernel   4 m^2 read back + the compact copy written (clp_sparse_info's bytes of one pass)
  sort / item lengths / scans / partition / warp columns: counts, window bitmaps, row ids and item pointers (a few MB)
Share of peak = bytes / time against the H100 SXM data-sheet 3.35 TB/s.  Prints ONE JSON line.
"""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_GBS = 3350.0


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim, smax = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock_max": smax}
    except Exception as e:  # the measurement itself does not depend on it
        return {"name": None, "error": str(e)}


def short_name(name):
    """'void clp::sparse_fill_items_kernel<float, true>(...)' -> 'sparse_fill_items_kernel<float, true>'"""
    n = name.split("(")[0]
    n = re.sub(r"^void\s+", "", n)
    return n.replace("clp::", "").replace("(anonymous namespace)::", "")


def kernel_bytes(key, m, rows_pad, NI, nseg, wwords, pass_bytes, packed):
    """bytes the kernel must move in one scoring call (None: not modelled)"""
    dense = 4 * m * m
    cnt = 4 * nseg * (rows_pad + 1)
    win = 4 * rows_pad * wwords if packed else 0
    items = 4 * nseg * (NI + 1)
    rowid = 4 * nseg * rows_pad
    if key.startswith("score_tile_kernel"):
        return dense
    if key.startswith("sparse_fill_items_kernel"):
        return dense + pass_bytes
    if key.startswith("sell_sort") or key.startswith("sell_hist") or key.startswith("sell_place"):
        return cnt + win + rowid
    if key.startswith("sell_itemlen"):
        return rowid // 4 + nseg * NI * 4 * (1 + wwords if packed else 1) + items
    if key.startswith("sparse_scan"):
        return 2 * items
    return None


def profile_workload(name, calls, warmup, trace_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from clipper_b200 import _capi, datagen
    import clipper_b200 as clipperpy

    L = _capi.load()
    dev = torch.device("cuda", 0)
    prob = datagen.config_problem(name)
    cfg = prob["cfg"]; m = cfg["m"]
    ip = clipperpy.invariants.EuclideanDistanceParams(); ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
    clip = clipperpy.CLIPPER(clipperpy.invariants.EuclideanDistance(ip), clipperpy.Params(), device=0)
    h = clip.handle
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    clip.set_stream(stream.cuda_stream)
    D1 = torch.from_numpy(np.ascontiguousarray(prob["D1"].T)).to(dev)
    D2 = torch.from_numpy(np.ascontiguousarray(prob["D2"].T)).to(dev)
    A = torch.from_numpy(np.ascontiguousarray(prob["A"].T)).to(dev)

    def score():
        _capi.check(h, L.clp_score_euclidean_dev(h, D1.data_ptr(), 3, D1.shape[0], D2.data_ptr(), D2.shape[0],
                                                 A.data_ptr(), m, cfg["sigma"], cfg["epsilon"], 0.0))

    for _ in range(warmup):
        score()
    torch.cuda.synchronize()
    # call time, profiler off
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    for _ in range(calls):
        score()
    ev1.record(stream)
    torch.cuda.synchronize()
    call_ms = ev0.elapsed_time(ev1) / calls

    mode = clip.dense_mode()
    kept, pass_bytes = clip.sparse_info() if mode in (3, 6) else (None, 0)
    rows_pad = (m + 31) // 32 * 32
    NI = rows_pad // 4
    ld = (m + 127) // 128 * 128
    wwords = (ld + 511) // 512
    # resident layout (mode 6): one segment = the whole row; segmented (mode 3): 4096-column segments or fewer
    nseg = 1 if mode == 6 else -(-m // 4096)
    packed = mode == 6 and pass_bytes < 5 * (kept or 0)  # 4-byte entries (+ fillers and padding) vs 6-byte ones

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            score()
        torch.cuda.synchronize()
    if trace_dir:
        os.makedirs(trace_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(trace_dir, "score_%s.json" % name))

    per = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        key = short_name(ev.name)
        d = per.setdefault(key, {"us": 0.0, "launches": 0})
        d["us"] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        d["launches"] += 1
    kernels = []
    for key, d in per.items():
        ms = d["us"] / 1e3 / calls
        b = kernel_bytes(key, m, rows_pad, NI, nseg, wwords, pass_bytes, packed)
        k = {"kernel": key, "ms_per_call": ms, "launches_per_call": d["launches"] / calls, "bytes": b}
        if b is not None and ms > 0:
            k["GBps"] = b / (ms * 1e-3) / 1e9
            k["frac_of_peak"] = k["GBps"] / PEAK_GBS
        kernels.append(k)
    kernels.sort(key=lambda k: -k["ms_per_call"])
    dev_ms = sum(k["ms_per_call"] for k in kernels)
    floor_bytes = 2 * 4 * m * m + pass_bytes
    return {"workload": name, "m": m, "sweep_mode": mode, "kept_entries": kept, "bytes_per_pass": pass_bytes,
            "call_ms": call_ms, "device_ms_in_kernels": dev_ms,
            "floor_bytes": floor_bytes, "floor_ms_at_peak": floor_bytes / (PEAK_GBS * 1e9) * 1e3,
            "kernels": kernels}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c2,c4")
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--trace", default=None, help="also write a chrome trace per workload under DIR")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("profile_score.py: no CUDA device")
    out = {"card": card(), "peak_GBps": PEAK_GBS, "peak_source": "H100 SXM data sheet", "calls": args.calls,
           "workloads": [profile_workload(w, args.calls, args.warmup, args.trace) for w in args.workloads.split(",")]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
