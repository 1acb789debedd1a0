#!/usr/bin/env python
"""Point clouds and associations already on the GPU against the host inputs of a scored batch, on one H100.  Prints one
JSON line.  Problems: config c1's parameters (datagen.euclidean_problem, m = 1000 associations, rho 0.9, sigma 0.01,
epsilon 0.02, full 9 992-point clouds), B = 64 and 512 per call (32 distinct seeds repeated).  For each B, the median
wall time of repeated calls after a warm-up of three paths:
  (a) BatchCLIPPER.solve_many from numpy arrays;
  (b) what a torch user does without the device path: .cpu().numpy() per problem, then solve_many;
  (c) BatchCLIPPER.solve_many_dev from the (B, 3, n), (B, m, 2) and (B, m) tensors.
Also the CLP_PROF_BATCH=1 upload time and bytes of (a) and (c) (from the call's start to the launch: the host copies
and uploads, or the staging kernel), from the second of two extra calls each.  Asserts that the three give identical
u, scores and nodes.  The GPU's name and power limit are read in the same run."""
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

from bench_batch_matrices import gpu_info  # noqa: E402


def timed(f, reps):
    f()   # warm-up: buffers and scratch are allocated once
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); out = f(); ts.append(time.perf_counter() - t0)
    return sorted(ts)[len(ts) // 2], out


def upload_split(clp, inv, call):
    """(upload ms, upload bytes, kernel ms) of the second of two calls on a batch made with CLP_PROF_BATCH=1 (the first
    allocates the batch's buffers)"""
    os.environ["CLP_PROF_BATCH"] = "1"
    try:
        b = clp.BatchCLIPPER(inv, clp.Params())
    finally:
        os.environ.pop("CLP_PROF_BATCH", None)
    with tempfile.TemporaryFile(mode="w+b") as tmp:
        saved = os.dup(2)
        sys.stderr.flush()
        os.dup2(tmp.fileno(), 2)
        try:
            call(b)
            call(b)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        tmp.seek(0)
        text = tmp.read().decode(errors="replace")
    mt = list(re.finditer(r"upload (\d+) bytes ([\d.]+) ms, kernel ([\d.]+) ms", text))
    mt = mt[-1] if len(mt) == 2 else None
    if not mt:
        return dict(prof_raw=text.strip())
    return dict(upload_bytes=int(mt.group(1)), upload_ms=float(mt.group(2)), kernel_ms=float(mt.group(3)))


def same(x, y, what):
    for k, (s, t) in enumerate(zip(x, y)):
        u1 = s.u if isinstance(s.u, np.ndarray) else s.u.cpu().numpy()
        u2 = t.u if isinstance(t.u, np.ndarray) else t.u.cpu().numpy()
        assert u1.tobytes() == u2.tobytes() and s.score == t.score and s.nodes == t.nodes, "%s: problem %d differs" % (what, k)


def main():
    import argparse
    import torch
    import clipper_b200 as clp
    from clipper_b200 import datagen
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="64,512")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    cfg = datagen.CONFIGS["c1"]
    ip = clp.invariants.EuclideanDistanceParams()
    ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
    inv = clp.invariants.EuclideanDistance(ip)
    distinct = [datagen.euclidean_problem(cfg["m"], cfg["rho"], cfg["seed"] + k) for k in range(32)]
    res = dict(gpu_info(), config="c1", m=cfg["m"], n=int(distinct[0]["D1"].shape[1]), rows=[])
    for B in [int(x) for x in args.batches.split(",") if x]:
        probs = [dict(D1=distinct[k % 32]["D1"], D2=distinct[k % 32]["D2"], A=distinct[k % 32]["A"],
                      u0=np.random.default_rng(k).random(cfg["m"])) for k in range(B)]
        D1 = torch.from_numpy(np.stack([p["D1"] for p in probs])).cuda()
        D2 = torch.from_numpy(np.stack([p["D2"] for p in probs])).cuda()
        A = torch.from_numpy(np.stack([p["A"] for p in probs])).cuda()
        U0 = torch.from_numpy(np.stack([p["u0"] for p in probs])).cuda()
        torch.cuda.synchronize()
        b = clp.BatchCLIPPER(inv, clp.Params())

        def from_torch():
            return b.solve_many([dict(D1=D1[k].cpu().numpy(), D2=D2[k].cpu().numpy(), A=A[k].cpu().numpy(),
                                      u0=U0[k].cpu().numpy()) for k in range(B)])

        t_a, sa = timed(lambda: b.solve_many(probs), args.reps)
        t_b, sb = timed(from_torch, args.reps)
        t_c, sc = timed(lambda: b.solve_many_dev(D1, D2, A, U0), args.reps)
        same(sa, sb, "B=%d host vs torch-to-host" % B)
        same(sa, sc, "B=%d host vs device" % B)
        row = dict(B=B, host_ms=1e3 * t_a, torch_to_host_ms=1e3 * t_b, device_ms=1e3 * t_c,
                   host_problems_per_s=B / t_a, torch_to_host_problems_per_s=B / t_b, device_problems_per_s=B / t_c,
                   speedup_vs_torch_to_host=t_b / t_c, speedup_vs_host=t_a / t_c,
                   prof_host=upload_split(clp, inv, lambda x: x.solve_many(probs)),
                   prof_device=upload_split(clp, inv, lambda x: x.solve_many_dev(D1, D2, A, U0)))
        print(json.dumps(row), file=sys.stderr, flush=True)
        res["rows"].append(row)
        del D1, D2, A, U0, b
        torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
