"""Maximum clique of the constraint graph on the GPU: every method on the BASELINE configs.

    python scripts/bench_maxclique.py [--configs c1,c2,c3,c4] [--time-limit 60] [--oracle-max-m 20000] [--out file]

Per config: the phase times of clp_max_clique (adjacency build, k-core peel, heuristic, search), omega, proven, the
number of branch-and-bound nodes, the inlier precision of the clique (an inlier association is (p, p)) next to that
of solve(), and the time of the CPU restatement in tests/clique_oracle.py (core numbers + heuristic) for m up to
--oracle-max-m.  One JSON line per (config, method).
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def precision(A, nodes):
    if len(nodes) == 0:
        return 0.0
    sel = A[np.asarray(nodes, dtype=np.int64)]
    return float((sel[:, 0] == sel[:, 1]).mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c1,c2,c3,c4")
    ap.add_argument("--time-limit", type=float, default=60.0)
    ap.add_argument("--oracle-max-m", type=int, default=20000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import clipper_b200 as clp
    from clipper_b200 import datagen
    rows = []
    for name in args.configs.split(","):
        prob = datagen.config_problem(name)
        cfg = prob["cfg"]
        if cfg["kind"] == "euclidean":
            ip = clp.invariants.EuclideanDistanceParams()
            ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
            c = clp.CLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params())
        else:
            ip = clp.invariants.PointNormalDistanceParams()
            ip.sigp, ip.epsp, ip.sign, ip.epsn = cfg["sigp"], cfg["epsp"], cfg["sign"], cfg["epsn"]
            c = clp.CLIPPER(clp.invariants.PointNormalDistance(ip), clp.Params())
        c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
        A = c.get_initial_associations()
        c.solve(prob["u0"])
        p_solve = precision(A, c.get_solution().nodes)
        n_solve = len(c.get_solution().nodes)
        oracle_s = None
        if cfg["m"] <= args.oracle_max_m:
            import clique_families as cf
            import clique_oracle as co
            adj = cf.adjacency(dict(name=name, scored=prob))
            t0 = time.perf_counter()
            core = co.core_numbers_level(adj)
            co.heu(adj, core)
            oracle_s = time.perf_counter() - t0
            del adj
        for method, mname in ((clp.MCMethod.KCORE, "KCORE"), (clp.MCMethod.HEU, "HEU"), (clp.MCMethod.EXACT, "EXACT")):
            p = clp.MCParams()
            p.method, p.time_limit = method, args.time_limit
            try:
                c.solve_as_maximum_clique(p)
            except clp.ClipperError as e:
                row = dict(config=name, m=cfg["m"], method=mname, error=str(e))
                print(json.dumps(row), flush=True)
                rows.append(row)
                continue
            s = c.get_solution()
            info = s.mc_info
            row = dict(config=name, m=cfg["m"], method=mname, n_nodes=len(s.nodes), max_core=info["max_core"],
                       lb=info["lower_bound"], ub=info["upper_bound"], proven=info["proven"],
                       timed_out=info["timed_out"], n_edges=info["n_edges"], n_branches=info["n_branches"],
                       adjacency_ms=info["adjacency_ms"], peel_ms=info["peel_ms"], heuristic_ms=info["heuristic_ms"],
                       search_ms=info["search_ms"], kernel_ms=info["kernel_ms"], wall_s=info["t"],
                       precision=precision(A, s.nodes), solve_precision=p_solve, solve_nodes=n_solve,
                       oracle_core_heu_s=oracle_s)
            print(json.dumps(row), flush=True)
            rows.append(row)
        del c
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
