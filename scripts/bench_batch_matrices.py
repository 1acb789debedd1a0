#!/usr/bin/env python
"""problems/s of batches of problems given as (M, C) matrices (clp_batch_solve_matrices, MatrixBatchCLIPPER):
(a) one MatrixBatchCLIPPER.solve_many call against (b) the same problems one at a time through one fp32 CLIPPER handle
(set_sparse_matrix_data + solve) and (c) the CPU oracle on a few problems.  Seeded weighted problems
(datagen.weighted_matrix_problem, 12.8 % density: c2-like) at m in {256, 1024, 2048, 4096}, 128 per size, plus 256 at
m = 2048.  Reports the bytes uploaded per call and the CLP_PROF_BATCH=1 split (scatter, build, solve) of one extra call,
and asserts equal nodes between (a) and (b).  One JSON line per configuration; the first names the GPU and its power
limit, read in the same run."""
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DENSITY = 0.128


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return dict(gpu=name, power_limit=power)
    except Exception as e:  # the measurement stands without it, but says so
        return dict(gpu="unknown (%s)" % e, power_limit="unknown")


def upload_bytes(csc, m):
    """what one call copies to the device for a problem: two column pointer arrays, row indices and values of M and C,
    u0 (padded to 16 bytes) and its table entry"""
    _, cpM, riM, vM, cpC, riC, vC = csc
    return 8 * (cpM.size + cpC.size) + 12 * (riM.size + riC.size) + 8 * ((m + 1) & ~1) + 48


def profiled_split(clp, probs):
    """one call with CLP_PROF_BATCH=1 (read when a batch handle is created); the library prints its split to stderr"""
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
            b.solve_many(probs)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        tmp.seek(0)
        text = tmp.read().decode(errors="replace")
    mt = re.search(r"upload (\d+) bytes ([\d.]+) ms, kernel ([\d.]+) ms; mean per problem: scatter ([\d.]+)\s+build ([\d.]+)"
                   r"\s+solve ([\d.]+)\s+total ([\d.]+) ms", text)
    if not mt:
        return dict(prof_raw=text.strip())
    up, up_ms, kms, sc, bu, so, to = mt.groups()
    return dict(prof_upload_bytes=int(up), prof_upload_ms=float(up_ms), prof_kernel_ms=float(kms),
                prof_scatter_ms_per_problem=float(sc), prof_build_ms_per_problem=float(bu),
                prof_solve_ms_per_problem=float(so), prof_total_ms_per_problem=float(to))


def main():
    import clipper_b200 as clp
    from clipper_b200 import datagen
    from clipper_b200.batch import matrices_to_csc
    from oracle import clipper_oracle as orc
    print(json.dumps(gpu_info()), flush=True)
    configs = [(256, 128), (1024, 128), (2048, 128), (4096, 128), (2048, 256)]
    if len(sys.argv) > 1:   # e.g. 2048:128,256:128
        configs = [tuple(int(x) for x in c.split(":")) for c in sys.argv[1].split(",")]
    for m, n in configs:
        distinct = [datagen.weighted_matrix_problem(m, DENSITY, 7000 + 31 * m + k) for k in range(min(n, 32))]
        probs = [dict(distinct[k % len(distinct)], u0=np.random.default_rng(k).random(m)) for k in range(n)]
        nbytes = sum(upload_bytes(matrices_to_csc(p["M"], p["C"]), m) for p in probs)
        b = clp.MatrixBatchCLIPPER()
        b.solve_many(probs)   # warm-up with the full batch: buffers, pinned staging and scratch are allocated once
        runs = []
        for _ in range(3):    # median of three timed calls
            t0 = time.perf_counter(); sols = b.solve_many(probs); t = time.perf_counter() - t0
            runs.append((t, sols[0].kernel_ms, sols))
        runs.sort(key=lambda r: r[0])
        t_batch, kms, sols = runs[1]
        t_call = sols[0].t * n   # wall clock inside clp_batch_solve_matrices: check + staging, upload, kernel, results
        t0 = time.perf_counter()
        for p in probs:
            matrices_to_csc(p["M"], p["C"])
        t_convert = time.perf_counter() - t0
        # (b) one fp32 handle, one problem at a time
        c = clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()), clp.Params())
        nl = min(n, 32)
        for p in probs[:2]:
            c.set_sparse_matrix_data(p["M"], p["C"]); c.solve(p["u0"])
        t0 = time.perf_counter()
        same = True
        for k, p in enumerate(probs[:nl]):
            c.set_sparse_matrix_data(p["M"], p["C"]); c.solve(p["u0"])
            same &= c.get_solution().nodes == sols[k].nodes
        t_loop = (time.perf_counter() - t0) / nl
        assert same, "m=%d: the batch and the single handle selected different nodes" % m
        # (c) the CPU oracle on a few problems (fp32-rounded M, as the GPU stores it)
        no = 2 if m >= 2048 else 4
        t0 = time.perf_counter()
        for p in probs[:no]:
            M = p["M"].toarray(); M = np.triu(M, 1).astype(np.float32).astype(np.float64); M = M + M.T + np.eye(m)
            Cu = np.triu(p["C"].toarray(), 1)
            o = orc.Oracle(); o.set_matrix_data(M, Cu + Cu.T + np.eye(m)); o.solve(p["u0"])
        t_cpu = (time.perf_counter() - t0) / no
        ctas, scratch, nnz = b.info()
        row = dict(m=m, problems=n, density=nnz / (n * m * (m - 1) / 2), batch_problems_per_s=n / t_batch,
                   batch_kernel_ms=kms, batch_kernel_problems_per_s=n / (kms * 1e-3), batch_call_ms=1e3 * t_call,
                   python_convert_ms=1e3 * t_convert, batch_wall_ms=1e3 * t_batch, upload_bytes=nbytes,
                   upload_bytes_per_problem=nbytes / n, single_handle_problems_per_s=1.0 / t_loop,
                   speedup_vs_single=(n / t_batch) * t_loop, cpu_oracle_problems_per_s=1.0 / t_cpu,
                   same_nodes_as_single=bool(same), ctas=ctas, scratch_GB=scratch / 1e9,
                   mean_evals=float(np.mean([s.n_evals for s in sols])))
        row.update(profiled_split(clp, probs))
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
