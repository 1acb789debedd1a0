#!/usr/bin/env python
"""Batches scored with a CUDA-source invariant (clp_batch_solve_custom) next to the built-in batch and a single-handle loop.

  python scripts/bench_batch_custom.py [--reps 5] [--loop 32] [--out results.json]

Per workload (seeded problems of clipper_b200.datagen, EuclideanDistance sigma 0.015, epsilon 0.05), on cuda:0:
  * builtin: BatchCLIPPER.solve_many with the built-in EuclideanDistance (fp32 screen, one launch);
  * custom: the same problems through the CUDA restatement of EuclideanDistance (EUCLID_SRC of the tests): rounds of a
    gather, the run-time compiled scoring launch over the whole device, and the stored-matrix solve launch;
  * loop: a CLIPPER with the same CudaInvariant, score_pairwise_consistency + solve per problem, over the first
    --loop problems of the list.
Problems/s from the median wall time of --reps calls after a warm-up call (every call ends in a synchronisation).  The
custom batch's answers must equal the built-in batch's bit for bit.  One extra custom call per workload runs under
torch.profiler and reports the device time of the scoring kernels (gather + score) and of the solve kernel.  The first
custom call's run-time compilation is reported apart.  Prints the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_gpu_custom_invariant import EUCLID_SRC  # noqa: E402  (the restatement the tests pin bit for bit)

SIGMA, EPS = 0.015, 0.05
WORKLOADS = [("m256", [256] * 396), ("m1024", [1024] * 396), ("m2048", [2048] * 256), ("m4096", [4096] * 128)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def problems(sizes, seed0):
    from clipper_b200 import datagen
    out = []
    for k, m in enumerate(sizes):
        prob = datagen.euclidean_problem(m, 0.9, seed0 + k)
        A = prob["A"]
        used1, inv1 = np.unique(A[:, 0], return_inverse=True)
        used2, inv2 = np.unique(A[:, 1], return_inverse=True)
        out.append(dict(D1=np.asfortranarray(prob["D1"][:, used1]), D2=np.asfortranarray(prob["D2"][:, used2]),
                        A=np.asfortranarray(np.stack([inv1, inv2], axis=1).astype(np.int32)), u0=prob["u0"]))
    return out


def wall(f):
    t0 = time.perf_counter()
    out = f()
    return time.perf_counter() - t0, out


def kernel_split(f):
    """device ms of the custom batch's scoring kernels and of its solve kernel in one call of f"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
    score = solve = 0.0
    for e in prof.key_averages():
        name = e.key
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if "batch_score_custom_kernel" in name or "batch_gather_kernel" in name:
            score += t / 1e3
        elif "batch_stored_solve_kernel" in name:
            solve += t / 1e3
    return round(score, 3), round(solve, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--loop", type=int, default=32)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    import clipper_b200 as clp
    from clipper_b200.api import jit_stats
    dev = card()
    print("card:", dev, flush=True)
    res = {"card": dev}
    rng = np.random.default_rng(11)
    workloads = WORKLOADS + [("mixed", rng.integers(128, 4097, 396).tolist())]
    ip = clp.invariants.EuclideanDistanceParams()
    ip.sigma, ip.epsilon = SIGMA, EPS
    inv = clp.invariants.CudaInvariant(EUCLID_SRC, (SIGMA, EPS, 0.0))
    b = clp.BatchCLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params())
    c = clp.BatchCLIPPER(inv, clp.Params())
    for seed, (name, sizes) in enumerate(workloads):
        probs = problems(sizes, 10000 * (seed + 1))
        n = len(probs)
        r = {"nprob": n, "m_min": int(min(sizes)), "m_max": int(max(sizes))}
        n0, ms0 = jit_stats()
        t_first, sc = wall(lambda: c.solve_many(probs))
        n1, ms1 = jit_stats()
        if n1 > n0:
            r["compile_ms"] = round(ms1 - ms0, 1)
            r["first_call_ms"] = round(1e3 * t_first, 1)
        sb = b.solve_many(probs)
        for k, (x, y) in enumerate(zip(sb, sc)):
            assert x.u.tobytes() == y.u.tobytes() and x.nodes == y.nodes and x.score == y.score, (name, k)
        r["slots"] = c.info()[0]
        r["rounds"] = -(-n // r["slots"])
        tb, tc = [], []
        for _ in range(args.reps):   # alternated, so that drift affects both alike
            tb.append(wall(lambda: b.solve_many(probs))[0])
            tc.append(wall(lambda: c.solve_many(probs))[0])
        r["builtin_per_s"] = round(n / float(np.median(tb)), 1)
        r["custom_per_s"] = round(n / float(np.median(tc)), 1)
        r["custom_ms"] = round(1e3 * float(np.median(tc)), 2)
        r["custom_score_kernel_ms"], r["custom_solve_kernel_ms"] = kernel_split(lambda: c.solve_many(probs))
        nl = min(args.loop, n)
        h = clp.CLIPPER(inv, clp.Params())
        h.score_pairwise_consistency(probs[0]["D1"], probs[0]["D2"], probs[0]["A"])
        h.solve(probs[0]["u0"])

        def loop():
            for p in probs[:nl]:
                h.score_pairwise_consistency(p["D1"], p["D2"], p["A"])
                h.solve(p["u0"])
        r["loop_per_s"] = round(nl / wall(loop)[0], 1)
        r["loop_problems"] = nl
        res[name] = r
        print(name, json.dumps(r), flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
