#!/usr/bin/env python
"""Bytes the resident solver reads per solve, and where its time goes, at the bench workloads.

  python scripts/profile_solve.py [--workloads c1,c2] [--solves 10]

Per workload: one scoring call, one warm-up solve, then timed solves (clp_solution.kernel_ms by CUDA events, and the
in-kernel phase split prof_matvec_ms / prof_combine_ms / prof_exchange_ms of CTA 0).  The matrix bytes of a solve come
from clp_last_solve_sweeps and clp_sparse_info:
  full passes       (n_matvec - rebuild - restricted) x the bytes of one pass of the compact copy
                    (the power step and the first normalisation always sweep the whole copy)
  rebuilds          one pass of the compact copy read + 6 bytes written per kept entry (not counted: a few %)
  restricted sweeps 6 bytes (fp32 value + 16-bit column) per entry and padding entry read
"dense_equivalent" is what the same evaluations would read with one full pass each, as bench.py assumes.  One more solve
on a handle made with CLP_PROF_CTAS=1 gives the spread over the CTAs (min / mean / max) of the sweep time and of the
restricted entries each CTA swept; the phase times above come from solves without it.  Prints ONE JSON line per workload.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim, smax = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock_max": smax}
    except Exception as e:  # the measurement itself does not depend on it
        return {"name": None, "error": str(e)}


def scored(clp, prob):
    cfg = prob["cfg"]
    ip = clp.invariants.EuclideanDistanceParams(); ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params())
    c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
    return c


def cta_spread(clp, prob):
    """one solve with the per-CTA timers (CLP_PROF_CTAS=1, read when a handle is made): the library's "[clp prof]" lines,
    which it writes to stderr, as {quantity: {min, mean, max}}"""
    os.environ["CLP_PROF_CTAS"] = "1"
    try:
        c = scored(clp, prob)
    finally:
        del os.environ["CLP_PROF_CTAS"]
    with tempfile.TemporaryFile(mode="w+") as tmp:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(tmp.fileno(), 2)
        try:
            c.solve(prob["u0"])
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        tmp.seek(0)
        text = tmp.read()
    out = {}
    for ln in text.splitlines():
        m = re.match(r"\[clp prof\] (.+?) per solve: min (\S+)\s+mean (\S+)\s+max (\S+)", ln)
        if m:
            key = m.group(1).strip().replace(" ", "_") + ("_ms" if "entries" not in m.group(1) else "")
            lo, mean, hi = (float(x) for x in m.group(2, 3, 4))
            out[key] = {"min": lo, "mean": mean, "max": hi, "max_over_mean": hi / mean if mean else None}
    return out


def profile(clp, datagen, name, solves):
    prob = datagen.config_problem(name); cfg = prob["cfg"]
    c = scored(clp, prob)
    _, pass_bytes = c.sparse_info()
    c.solve(prob["u0"])
    rows = []
    for _ in range(solves):
        c.solve(prob["u0"])
        s = c.get_solution()
        rows.append((s.kernel_ms,) + tuple(s.prof_ms))
    sw = c.last_solve_sweeps()
    full_passes = s.n_matvec - sw["rebuild"] - sw["restricted"]
    restricted_bytes = 6 * (sw["entries"] + sw["padding"])
    total = full_passes * pass_bytes + sw["rebuild"] * pass_bytes + restricted_bytes
    k = np.array(rows)
    return {
        "workload": name, "m": cfg["m"], "dense_mode": c.dense_mode(), "n_evals": int(s.n_evals),
        "n_matvec": int(s.n_matvec), "sweeps": sw, "pass_bytes": int(pass_bytes),
        "bytes_per_solve": int(total), "full_pass_equivalents": total / pass_bytes,
        "dense_equivalent_bytes": int(s.n_matvec * pass_bytes),
        "restricted_mb_per_sweep": restricted_bytes / max(1, sw["rebuild"] + sw["restricted"]) / 1e6,
        "kernel_ms": {"median": float(np.median(k[:, 0])), "min": float(k[:, 0].min()), "max": float(k[:, 0].max())},
        "phase_ms_cta0": {"sweeps_and_staging": float(np.median(k[:, 1])), "epilogues": float(np.median(k[:, 2])),
                          "exchanges": float(np.median(k[:, 3]))},
        "per_cta": cta_spread(clp, prob),
        "card": card(),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c1,c2")
    ap.add_argument("--solves", type=int, default=10)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("profile_solve.py needs a CUDA device")
    import clipper_b200 as clp
    from clipper_b200 import datagen
    for name in args.workloads.split(","):
        print(json.dumps(profile(clp, datagen, name, args.solves)))


if __name__ == "__main__":
    main()
