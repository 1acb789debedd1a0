"""Semidefinite relaxation on the GPU (clp_sdp_solve, clp_batch_sdp_matrices): iterations, Jacobi sweeps per
iteration, kernel and eigensolver time, problems per second, and the time of the numpy restatement in
tests/sdr_oracle.py on the same inputs (a CPU restatement with numpy.linalg.eigh; it is not SCS).

  single problems: the reference's 20 x 20 matrix and scored Euclidean problems at m = 64 and 128
  batches: 132 k problems (k = 1, 4) of scored Euclidean problems at m = 64 and m = 128

Prints one JSON line per measurement; --out also writes them to a JSON file.
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def scored(clp, m, seed):
    from clipper_b200 import datagen
    p = datagen.euclidean_problem(m, 0.8, seed)
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()), clp.Params())
    c.score_pairwise_consistency(p["D1"], p["D2"], p["A"])
    return c


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-reps", type=int, default=2)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_sdr needs a CUDA device"
    import clipper_b200 as clp
    import fixtures as fx
    import sdr_oracle as so
    import scipy.sparse as sp
    dev = card()
    rows = []

    def emit(r):
        r["card"] = dev
        print(json.dumps(r), flush=True)
        rows.append(r)

    p = clp.SDPParams()
    singles = [("m20", None)] + [("euclid%d" % m, m) for m in (64, 128)]
    for name, m in singles:
        if m is None:
            M, Cm = fx.m20()
            c = clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()), clp.Params())
            c.set_matrix_data(M, Cm)
        else:
            c = scored(clp, m, 31 + m)
        M, Cm = c.get_affinity_matrix(), c.get_constraint_matrix()
        c.solve_as_msrc_sdr(p)  # warm-up
        ts, infos = [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            c.solve_as_msrc_sdr(p)
            ts.append(time.perf_counter() - t0)
            infos.append(c.get_solution().sdp_info)
        i = infos[-1]
        to = []
        for _ in range(args.oracle_reps):
            t0 = time.perf_counter()
            o = so.solve(M, Cm)
            to.append(time.perf_counter() - t0)
        emit(dict(case="single", name=name, m=int(M.shape[0]), iters=i["iters"], sweeps_per_iter=i["n_sweeps"] / i["iters"],
                  kernel_ms=float(np.median([x["kernel_ms"] for x in infos])),
                  proj_ms=float(np.median([x["proj_ms"] for x in infos])), call_ms=1e3 * float(np.median(ts)),
                  problems_per_s=1.0 / float(np.median(ts)), nodes=len(c.get_solution().nodes),
                  cpu_numpy_restatement_ms=1e3 * float(np.median(to)), cpu_iters=o["iters"]))

    b = clp.MatrixBatchCLIPPER()
    for m in (64, 128):
        for k in (1, 4):
            n = 132 * k
            probs = []
            base = [scored(clp, m, 1000 + m + q) for q in range(8)]
            mats = [(c.get_affinity_matrix(), c.get_constraint_matrix()) for c in base]
            for q in range(n):
                M, Cm = mats[q % len(mats)]
                probs.append(dict(M=sp.csc_matrix(np.triu(M, 1)), C=sp.csc_matrix(np.triu(Cm, 1))))
            b.sdr_many(probs[:8], p)  # warm-up
            ts = []
            for _ in range(max(1, args.reps // 2)):
                t0 = time.perf_counter()
                out = b.sdr_many(probs, p)
                ts.append(time.perf_counter() - t0)
            it = [s.sdp_info["iters"] for s in out]
            sw = sum(s.sdp_info["n_sweeps"] for s in out) / sum(it)
            t0 = time.perf_counter()
            for M, Cm in mats:
                so.solve(M, Cm)
            cpu_ms = 1e3 * (time.perf_counter() - t0) / len(mats)
            emit(dict(case="batch", m=m, nprob=n, ctas=b.info()[0], mean_iters=float(np.mean(it)), sweeps_per_iter=sw,
                      kernel_ms=out[0].sdp_info["kernel_ms"], call_ms=1e3 * float(np.median(ts)),
                      problems_per_s=n / float(np.median(ts)),
                      mean_proj_ms=float(np.mean([s.sdp_info["proj_ms"] for s in out])),
                      cpu_numpy_restatement_ms_per_problem=cpu_ms))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
