"""Putative associations for a batch of cloud pairs (distance_based_correspondences_many_dev, one batched call) against
a Python loop of distance_based_correspondences_dev over the same pairs; then the chain clouds -> A -> solve_many_dev,
batched against per pair.

  pairs: B in {64, 256, 1024}, n1 = n2 = n in {256, 1000, 2000}: pair p is n points of the bunny (the reference's
  bun10k, tests/golden/bun10k_points.npz; a seeded subset per pair) against a copy with bounded noise (sigma 0.01,
  beta 0.0554); d = 33 appends 30 seeded noise features to both.  knn in {1, 10}; radius inf and beta; with and
  without 1-to-1.
  kernel ms: the sum of the kernels of the batched call (knn_* and the staging kernel), or of all B single calls, from
  torch.profiler (a run of its own)
  event ms: CUDA events on torch's stream just before and just after the batched call, or the whole loop
  call ms: wall clock around the blocking batched call, or the whole loop, on torch's current (default) stream, clouds
  already on the device
  same_as_loop: every problem's rows of the batched A equal the looped call's, bit for bit (checked for every case)
  chain: knn = 1, radius beta, 1-to-1, d = 3: batched kNN -> solve_many_dev (problems without rows dropped) against B
  single calls, A padded by hand, then the same solve_many_dev; the wall clock of each chain

Prints one JSON line per measurement; --out also writes them to a JSON file.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

BETA = 0.0554


def pairs(B, n, d, seed=3):
    """B (D1, D2) pairs of F-order (d, n) float64 arrays: bunny subsets against noisy copies"""
    from clipper_b200 import datagen
    cloud = datagen.make_cloud(9992)
    rng = np.random.default_rng(seed + 7919 * n + 104729 * d)
    out = []
    for _ in range(B):
        P = cloud[:, rng.choice(cloud.shape[1], n, replace=False)]
        Q = P + datagen.bounded_normal_noise(rng, n, 0.01, BETA).T
        if d > 3:
            F = rng.standard_normal((d - 3, n))
            P = np.vstack([P, F])
            Q = np.vstack([Q, F + 0.01 * rng.standard_normal((d - 3, n))])
        out.append((np.asfortranarray(P), np.asfortranarray(Q)))
    return out


def kernel_ms(fn):
    import torch
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = 0.0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and ("knn_" in e.name or "stage_points" in e.name):
            tot += e.device_time if hasattr(e, "device_time") else e.cuda_time
    return tot / 1e3


def timed(fn, reps):
    """(wall ms per call, event ms of one call, kernel ms of one call)"""
    import torch
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    call = 1e3 * (time.perf_counter() - t0) / reps
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return call, e0.elapsed_time(e1), kernel_ms(fn)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batches", default="64,256,1024")
    ap.add_argument("--sizes", default="256,1000,2000")
    ap.add_argument("--dims", default="3,33")
    ap.add_argument("--knns", default="1,10")
    ap.add_argument("--modes", default="inf:0,inf:1,beta:0,beta:1", help="radius (inf or beta):1-to-1 (0 or 1) pairs")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_knn_batch needs a CUDA device"
    import clipper_b200 as clp
    from bench_knn import card
    dev = card()
    rows = []
    u = clp.utils

    def emit(r):
        r["card"] = dev
        print(json.dumps(r), flush=True)
        rows.append(r)

    modes = [(np.inf if r == "inf" else BETA, bool(int(o))) for r, o in (x.split(":") for x in args.modes.split(","))]
    for B in [int(x) for x in args.batches.split(",")]:
        for n in [int(x) for x in args.sizes.split(",")]:
            for d in [int(x) for x in args.dims.split(",")]:
                ps = pairs(B, n, d)
                singles = [(torch.from_numpy(P).cuda(), torch.from_numpy(Q).cuda()) for P, Q in ps]
                T1 = torch.stack([a for a, _ in singles])
                T2 = torch.stack([b for _, b in singles])
                for knn in [int(x) for x in args.knns.split(",")]:
                    for radius, one in modes:
                        batched = lambda: u.distance_based_correspondences_many_dev(T1, T2, knn, radius, one)  # noqa: E731
                        looped = lambda: [u.distance_based_correspondences_dev(a, b, knn, radius, one)  # noqa: E731
                                          for a, b in singles]
                        A, m = batched()
                        L = looped()
                        same = all(np.array_equal(A[p, :m[p]].cpu().numpy(), L[p].cpu().numpy()) for p in range(B))
                        bc, be, bk = timed(batched, args.reps)
                        lc, le, lk = timed(looped, args.reps)
                        emit(dict(case="knn_batch", B=B, n=n, d=d, knn=knn, radius=("inf" if radius == np.inf else radius),
                                  one_to_one=one, m_total=int(sum(m)), same_as_loop=bool(same),
                                  batched=dict(kernel_ms=round(bk, 3), event_ms=round(be, 3), call_ms=round(bc, 3)),
                                  loop=dict(kernel_ms=round(lk, 3), event_ms=round(le, 3), call_ms=round(lc, 3)),
                                  call_speedup=round(lc / bc, 2)))
                        if not same:
                            raise SystemExit("batched A differs from the looped A: B=%d n=%d d=%d knn=%d" % (B, n, d, knn))
                if d == 3:
                    chain(clp, B, n, T1, T2, singles, emit, args.reps)
                del T1, T2, singles
                torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


def chain(clp, B, n, T1, T2, singles, emit, reps):
    """batched kNN -> solve_many_dev against B single kNN calls, A padded by hand -> the same solve_many_dev"""
    import torch
    ip = clp.invariants.EuclideanDistanceParams()
    ip.sigma, ip.epsilon = 0.01, 0.02
    bc = clp.BatchCLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params())
    u = clp.utils

    def solve(A, m):
        keep = [p for p in range(B) if m[p] > 0]   # m = 0 would mean all-to-all to the solve
        idx = torch.tensor(keep, device=T1.device)
        mk = [m[p] for p in keep]
        u0 = torch.full((len(keep), max(mk)), 0.5, dtype=torch.float64, device=T1.device)
        return bc.solve_many_dev(T1[idx], T2[idx], A[idx], u0, m=mk)

    def batched():
        A, m = u.distance_based_correspondences_many_dev(T1, T2, 1, BETA, True)
        return solve(A, m)

    def looped():
        As = [u.distance_based_correspondences_dev(a, b, 1, BETA, True) for a, b in singles]
        m = [int(a.shape[0]) for a in As]
        A = torch.zeros((B, max(m), 2), dtype=torch.int32, device=T1.device)
        for p, a in enumerate(As):
            A[p, :m[p]] = a
        return solve(A, m)

    out = {}
    for name, fn in (("batched", batched), ("loop", looped)):
        s = fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            s = fn()
            torch.cuda.synchronize()
            ts.append(1e3 * (time.perf_counter() - t0))
        out[name] = (float(np.median(ts)), [(x.nodes, x.score) for x in s])
    emit(dict(case="chain", B=B, n=n, d=3, knn=1, radius=BETA, one_to_one=True,
              batched_ms=round(out["batched"][0], 3), loop_ms=round(out["loop"][0], 3),
              same_solutions=out["batched"][1] == out["loop"][1],
              speedup=round(out["loop"][0] / out["batched"][0], 2)))


if __name__ == "__main__":
    main()
