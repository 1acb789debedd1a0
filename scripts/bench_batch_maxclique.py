"""Batched maximum clique: batches of small scored problems, one batch call against the same problems one at a time.

    python scripts/bench_batch_maxclique.py [--sizes 256,1024,2048] [--nprob 256] [--time-limit 10] [--out file]

Per size m: nprob seeded Euclidean problems (rho = 0.9, the benchmark's sigma = 0.015 and epsilon = 0.05), for HEU and
for EXACT under --time-limit (for the whole batch call, and per problem on the single handle):
  (a) one BatchCLIPPER.max_clique_many call,
  (b) the same problems one at a time through one fp32 handle (score, then clp_max_clique),
  (c) the CPU restatement in tests/clique_oracle.py, core numbers and heuristic only (at most --oracle-nprob problems).
Problems per second for each, how many problems were proven, and an assertion that (a) and (b) agree as the tests
require (cores, bounds, HEU nodes; EXACT nodes where both are proven).  The card's name and power limit are read in
the same run and printed with the numbers.  One JSON line per (m, method).
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
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # the numbers are still printed, marked with the failure
        return "unknown (%s)" % e


def problems(m, nprob, seed0):
    from clipper_b200 import datagen
    out = []
    for k in range(nprob):
        prob = datagen.euclidean_problem(m, 0.9, seed0 + k)
        A = prob["A"]
        used1, inv1 = np.unique(A[:, 0], return_inverse=True)
        used2, inv2 = np.unique(A[:, 1], return_inverse=True)
        out.append(dict(D1=np.asfortranarray(prob["D1"][:, used1]), D2=np.asfortranarray(prob["D2"][:, used2]),
                        A=np.asfortranarray(np.stack([inv1, inv2], axis=1).astype(np.int32))))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="256,1024,2048")
    ap.add_argument("--nprob", type=int, default=256)
    ap.add_argument("--time-limit", type=float, default=10.0)
    ap.add_argument("--oracle-nprob", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import clipper_b200 as clp
    import clique_oracle as co
    sigma, eps = 0.015, 0.05
    gpu = card()
    print("card:", gpu, flush=True)

    def inv():
        ip = clp.invariants.EuclideanDistanceParams()
        ip.sigma, ip.epsilon = sigma, eps
        return clp.invariants.EuclideanDistance(ip)

    rows = []
    b = clp.BatchCLIPPER(inv(), clp.Params())
    c = clp.CLIPPER(inv(), clp.Params())
    for m in [int(x) for x in args.sizes.split(",")]:
        probs = problems(m, args.nprob, 9000 + m)
        for method, mname in ((clp.MCMethod.HEU, "HEU"), (clp.MCMethod.EXACT, "EXACT")):
            p = clp.MCParams()
            p.method, p.time_limit = method, args.time_limit
            b.max_clique_many(probs[:2], p)  # warm-up: module load, buffers
            t0 = time.perf_counter()
            got = b.max_clique_many(probs, p)
            t_batch = time.perf_counter() - t0
            t0 = time.perf_counter()
            single = []
            for q in probs:
                c.score_pairwise_consistency(q["D1"], q["D2"], q["A"])
                c.solve_as_maximum_clique(p)
                s = c.get_solution()
                single.append((s.nodes, s.mc_info))
            t_single = time.perf_counter() - t0
            both = 0
            for k, (s, (nodes1, info1)) in enumerate(zip(got, single)):
                for key in ("n_edges", "max_core", "upper_bound", "lower_bound"):
                    assert s.mc_info[key] == info1[key], (m, mname, k, key)
                if method == clp.MCMethod.HEU:
                    assert s.nodes == nodes1, (m, k)
                elif s.mc_info["proven"] and info1["proven"]:
                    assert s.nodes == nodes1, (m, k)
                    both += 1
            t_oracle = None
            if method == clp.MCMethod.HEU and args.oracle_nprob > 0:
                import clique_families as cf
                no = min(args.oracle_nprob, len(probs))
                adjs = []
                for q in probs[:no]:
                    c.score_pairwise_consistency(q["D1"], q["D2"], q["A"])
                    C_ = c.get_constraint_matrix()
                    adjs.append(cf.adjacency(dict(C=C_)))
                t0 = time.perf_counter()
                for adj in adjs:
                    co.heu(adj, co.core_numbers_level(adj))
                t_oracle = (time.perf_counter() - t0) / no
            i0 = got[0].mc_info
            row = dict(m=m, method=mname, nprob=len(probs), time_limit_s=args.time_limit, card=gpu,
                       batch_problems_per_s=len(probs) / t_batch, single_problems_per_s=len(probs) / t_single,
                       cpu_core_heu_problems_per_s=(1.0 / t_oracle) if t_oracle else None,
                       batch_s=t_batch, single_s=t_single,
                       batch_proven=sum(s.mc_info["proven"] for s in got),
                       batch_timed_out=sum(s.mc_info["timed_out"] for s in got),
                       single_proven=sum(i["proven"] for _, i in single), both_proven_identical=both,
                       batch_adjacency_ms=i0["adjacency_ms"], batch_peel_ms=i0["peel_ms"],
                       batch_heuristic_ms=i0["heuristic_ms"], batch_search_ms=i0["search_ms"],
                       mean_omega=float(np.mean([len(s.nodes) for s in got])))
            print(json.dumps(row), flush=True)
            rows.append(row)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
