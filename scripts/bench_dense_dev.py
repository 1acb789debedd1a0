#!/usr/bin/env python
"""Matrices already on the GPU against matrices from the host, on one H100.  Prints one JSON line:
- batch: for m in {256, 1024, 2048, 4096}, 128 seeded weighted problems each (datagen.weighted_matrix_problem, 12.8 %
  density as scripts/bench_batch_matrices.py), problems/s of MatrixBatchCLIPPER.solve_many from numpy (CSC conversion,
  host check and upload included) and of solve_dense_dev from fp32 and from fp64 (B, m, m) tensors; the CLP_PROF_BATCH=1
  split (load, build, solve per problem) of one extra dense call per input type; the bytes the load step must move per
  problem (both strict upper triangles read, the rows_pad x ld fp32 scratch written) and what they are per load time
  of one CTA and, over the whole batch, per kernel time as a share of 3.35 TB/s;
- single handle at m = 20 000 (fp32 tensors): time of set_matrix_data from numpy against set_matrix_data_dev.
Asserts equal nodes between the host and the device paths.  --sizes and --no-single run a part of it.  The GPU's name
and power limit are read in the same run."""
import json
import os
import re
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_batch_matrices import DENSITY, gpu_info  # noqa: E402

HBM_TBPS = 3.35   # H100 SXM data sheet


def load_bytes(m, esize):
    ld, rows_pad = (m + 127) // 128 * 128, (m + 3) // 4 * 4
    return 2 * esize * m * (m - 1) // 2 + 4 * rows_pad * ld


def prof_split(clp, tM, tC, u0):
    os.environ["CLP_PROF_BATCH"] = "1"
    try:
        b = clp.MatrixBatchCLIPPER()
    finally:
        os.environ.pop("CLP_PROF_BATCH", None)
    with tempfile.TemporaryFile(mode="w+b") as tmp:
        saved = os.dup(2)
        sys.stderr.flush()
        os.dup2(tmp.fileno(), 2)
        try:
            b.solve_dense_dev(tM, tC, u0)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        tmp.seek(0)
        text = tmp.read().decode(errors="replace")
    mt = re.search(r"kernel ([\d.]+) ms; mean per problem: load ([\d.]+)\s+build ([\d.]+)\s+solve ([\d.]+)\s+total ([\d.]+) ms",
                   text)
    if not mt:
        return dict(prof_raw=text.strip())
    k, lo, bu, so, to = (float(x) for x in mt.groups())
    return dict(kernel_ms=k, load_ms=lo, build_ms=bu, solve_ms=so, total_ms=to)


def timed(f, reps=3):
    f()   # warm-up: buffers and scratch are allocated once
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); out = f(); ts.append(time.perf_counter() - t0)
    return sorted(ts)[len(ts) // 2], out


def main():
    import torch
    import clipper_b200 as clp
    from clipper_b200 import datagen
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="256,1024,2048,4096")
    ap.add_argument("--no-single", action="store_true")
    args = ap.parse_args()
    res = dict(gpu_info())
    rows = []
    for m in [int(x) for x in args.sizes.split(",") if x]:
        n = 128
        distinct = [datagen.weighted_matrix_problem(m, DENSITY, 7000 + 31 * m + k) for k in range(32)]
        probs = [dict(distinct[k % 32], u0=np.random.default_rng(k).random(m)) for k in range(n)]
        dense = [torch.stack([torch.from_numpy(d[w].toarray()).cuda() for d in distinct]) for w in ("M", "C")]
        idx = torch.tensor([k % 32 for k in range(n)], device="cuda")
        u0 = torch.from_numpy(np.stack([p["u0"] for p in probs])).cuda()
        b = clp.MatrixBatchCLIPPER()
        t_host, sols = timed(lambda: b.solve_many(probs))
        row = dict(m=m, problems=n, solve_many_problems_per_s=n / t_host)
        for name, dt, es in (("f32", torch.float32, 4), ("f64", torch.float64, 8)):
            tM, tC = dense[0].to(dt)[idx], dense[1].to(dt)[idx]
            bd = clp.MatrixBatchCLIPPER()
            t_dev, sd = timed(lambda: bd.solve_dense_dev(tM, tC, u0))
            if name == "f64":
                assert [s.nodes for s in sd] == [s.nodes for s in sols], "m=%d: device and host paths differ" % m
            sp = prof_split(clp, tM, tC, u0)
            nb = load_bytes(m, es)
            row.update({"dense_dev_%s_problems_per_s" % name: n / t_dev, "dense_dev_%s_kernel_ms" % name: sd[0].kernel_ms,
                        "prof_%s" % name: sp, "load_bytes_per_problem_%s" % name: nb})
            if "load_ms" in sp:
                row["load_GBps_per_cta_%s" % name] = nb / (sp["load_ms"] * 1e-3) / 1e9
                row["load_bytes_over_kernel_share_of_hbm_%s" % name] = n * nb / (sp["kernel_ms"] * 1e-3) / (HBM_TBPS * 1e12)
            del tM, tC, bd
        del dense
        torch.cuda.empty_cache()
        rows.append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
    res["batch"] = rows
    if args.no_single:
        print(json.dumps(res), flush=True)
        return
    # single handle, m = 20 000
    m = 20000
    p = datagen.weighted_matrix_problem(m, 0.01, 99)
    M = p["M"].toarray().astype(np.float32).astype(np.float64); Cm = p["C"].toarray()
    tM, tC = torch.from_numpy(M).float().cuda(), torch.from_numpy(Cm).float().cuda()
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()), clp.Params())
    t_np, _ = timed(lambda: c.set_matrix_data(M, Cm))
    c.solve(p["u0"]); nodes_host = c.get_solution().nodes
    t_dev, _ = timed(lambda: (c.set_matrix_data_dev(tM, tC), torch.cuda.synchronize()))
    c.solve(p["u0"])
    assert c.get_solution().nodes == nodes_host, "m=20000: device and host loads differ"
    res["single_m20000"] = dict(set_matrix_data_ms=1e3 * t_np, set_matrix_data_dev_ms=1e3 * t_dev)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
