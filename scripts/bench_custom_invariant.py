#!/usr/bin/env python
"""Cost of scoring a CUDA-source invariant (CudaInvariant, clp_score_custom) next to the built-in EuclideanDistance.

  python scripts/bench_custom_invariant.py [--reps 5] [--configs c1,c2]

Per config (clipper_b200.datagen.CONFIGS: c1 m = 1000, c2 m = 20000), on cuda:0:
  * compile_ms: the one run-time compilation of the restatement (NVRTC, reported once and apart from the calls);
  * builtin_f32 / builtin_f64 / custom_f32 / custom_f64: median wall time of a warm score_pairwise_consistency call
    (host inputs, returns with the matrix and its compact copy built) of the built-in invariant and of its CUDA
    restatement, with fp32 and fp64 storage.  The fp32 built-in runs the screened kernel; every other case runs the
    unscreened fp64 kernel;
  * c1 only: the notebook's Custom invariant (sigma = 0.015, epsilon = 0.02) through the two host custom paths, the
    Python mirror and the C++ shell's pybind module (clipperpy), one call each.
Before timing, the restatement's M and C must equal the built-in's bit for bit at each size and storage.
Prints the card's name and power limit read in the same run, then one JSON line.
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def timed_call(c, D1, D2, A):
    t0 = time.perf_counter()
    c.score_pairwise_consistency(D1, D2, A)
    return 1e3 * (time.perf_counter() - t0)


def same(a, b, what):
    for get in ("get_constraint_matrix", "get_affinity_matrix"):
        x, y = getattr(a, get)(), getattr(b, get)()
        assert np.array_equal(x.view(np.int64), y.view(np.int64)), "%s: %s differs" % (what, get)
        del x, y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--configs", default="c1,c2")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    import clipper_b200 as clp
    from clipper_b200 import datagen
    from clipper_b200.api import jit_stats
    print("card:", card(), flush=True)
    res = {"card": card()}
    for name in args.configs.split(","):
        prob = datagen.config_problem(name)
        cfg = prob["cfg"]
        sigma, eps = (0.015, 0.02) if name == "c1" else (cfg["sigma"], cfg["epsilon"])
        D1, D2, A = prob["D1"], prob["D2"], prob["A"]
        ip = clp.invariants.EuclideanDistanceParams()
        ip.sigma, ip.epsilon = sigma, eps
        r = {"m": int(A.shape[0]), "sigma": sigma, "epsilon": eps}
        for storage, tag in ((clp.STORE_F32, "f32"), (clp.STORE_F64, "f64")):
            b = clp.CLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params(), storage=storage)
            c = clp.CLIPPER(clp.invariants.CudaInvariant(EUCLID_SRC, (sigma, eps, 0.0)), clp.Params(), storage=storage)
            n0, ms0 = jit_stats()
            b.score_pairwise_consistency(D1, D2, A)
            c.score_pairwise_consistency(D1, D2, A)
            n1, ms1 = jit_stats()
            r["compile_ms_" + tag] = round(ms1 - ms0, 1) if n1 > n0 else 0.0
            same(b, c, "%s %s" % (name, tag))
            tb, tc = [], []
            for _ in range(args.reps):   # alternated, so that drift affects both alike
                tb.append(timed_call(b, D1, D2, A))
                tc.append(timed_call(c, D1, D2, A))
            r["builtin_%s_ms" % tag] = round(float(np.median(tb)), 3)
            r["custom_%s_ms" % tag] = round(float(np.median(tc)), 3)
            del b, c
        if name == "c1":
            class Custom(clp.invariants.PairwiseInvariant):   # the reference notebook's invariant
                def __call__(self, ai, aj, bi, bj):
                    cc = np.abs(np.linalg.norm(ai - aj) - np.linalg.norm(bi - bj))
                    return np.exp(-0.5 * cc ** 2 / sigma ** 2) if cc < eps else 0
            h = clp.CLIPPER(Custom(), clp.Params())
            r["host_python_ms"] = round(timed_call(h, D1, D2, A), 1)
            sys.path.insert(0, os.path.join(ROOT, "clipper_b200", "lib"))
            import clipperpy as cp

            class PyCustom(cp.invariants.PairwiseInvariant):
                def __call__(self, ai, aj, bi, bj):
                    cc = np.abs(np.linalg.norm(ai - aj) - np.linalg.norm(bi - bj))
                    return np.exp(-0.5 * cc ** 2 / sigma ** 2) if cc < eps else 0
            s = cp.CLIPPER(PyCustom(), cp.Params())
            r["host_cpp_shell_ms"] = round(timed_call(s, D1, D2, A), 1)
        res[name] = r
        print(name, json.dumps(r), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
