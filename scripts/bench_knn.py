"""Putative associations on the GPU (clp_correspondences_dev): kernel time, call time, achieved fp64 rate, and scipy's
cKDTree(workers=-1) on the same host and inputs; then the whole chain clouds -> A -> score -> solve on the device
against the host chain (cKDTree, numpy arrays, score_pairwise_consistency, solve).

  cases: n1 = n2 = n in {9 992 (the bunny against a noisy copy), 1e5, 1e6 (synthetic surfaces)}, d in {3, 33}
  (d = 33: the cloud's coordinates padded with seeded noise features), knn in {1, 10}, radius inf, no 1-to-1
  kernel ms: the sum of the knn_* kernels of one call, from torch.profiler (a run of its own); the call blocks to read
  m, so CUDA events around it cannot leave the host's part out
  event ms: CUDA events on torch's stream just before and just after the call (its kernels, the read of m and the gaps)
  call ms: wall clock around the blocking call on torch's current (default) stream, inputs already on the device
  fp64 rate: 3 d operations per (query, candidate) pair over the kernel time; the data sheet's 34 TFLOP/s FP64 counts a
  fused multiply-add as two operations, and this kernel never fuses (its bits are pinned), so it can reach half of it

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

PEAK_FP64 = 34e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def clouds(n, d, seed=3):
    from clipper_b200 import datagen
    rng = np.random.default_rng(seed)
    P = datagen.make_cloud(n)
    Q = P + datagen.bounded_normal_noise(rng, n, 0.01, 0.0554).T
    if d > 3:
        F = rng.standard_normal((d - 3, n))
        P = np.vstack([P, F])
        Q = np.vstack([Q, F + 0.01 * rng.standard_normal((d - 3, n))])
    return np.asfortranarray(P), np.asfortranarray(Q)


def kernel_ms(fn):
    import torch
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = 0.0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "knn_" in e.name:
            tot += e.device_time if hasattr(e, "device_time") else e.cuda_time
    return tot / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="9992,100000,1000000")
    ap.add_argument("--dims", default="3,33")
    ap.add_argument("--kdtree-max-pairs-d", type=float, default=5e10,
                    help="for d > 3, skip cKDTree where n * n * d exceeds this (a kd-tree in high d is a slow brute force)")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_knn needs a CUDA device"
    import clipper_b200 as clp
    from scipy.spatial import cKDTree
    dev = card()
    rows = []

    def emit(r):
        r["card"] = dev
        print(json.dumps(r), flush=True)
        rows.append(r)

    for n in [int(x) for x in args.sizes.split(",")]:
        for d in [int(x) for x in args.dims.split(",")]:
            D1, D2 = clouds(n, d)
            T1, T2 = torch.from_numpy(D1).cuda(), torch.from_numpy(D2).cuda()
            pairs = float(n) * n
            for knn in (1, 10):
                call = lambda: clp.utils.distance_based_correspondences_dev(T1, T2, knn, np.inf, False)  # noqa: E731
                A = call()                                   # warm-up (and the module loads)
                torch.cuda.synchronize()
                reps = args.reps if pairs * d < 1e12 else 1
                t0 = time.perf_counter()
                for _ in range(reps):
                    call()
                torch.cuda.synchronize()
                call_ms = 1e3 * (time.perf_counter() - t0) / reps
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                call()
                e1.record()
                e1.synchronize()
                kms = kernel_ms(call)
                r = dict(case="knn", n=n, d=d, knn=knn, m=int(A.shape[0]), call_ms=round(call_ms, 3),
                         event_ms=round(e0.elapsed_time(e1), 3),
                         kernel_ms=round(kms, 3), fp64_tflops=round(3 * d * pairs / (kms * 1e-3) / 1e12, 2),
                         share_of_34=round(3 * d * pairs / (kms * 1e-3) / PEAK_FP64, 3))
                if d <= 3 or pairs * d <= args.kdtree_max_pairs_d:
                    t0 = time.perf_counter()
                    tree = cKDTree(D2.T)
                    _, idx = tree.query(D1.T, k=knn, workers=-1)
                    r["kdtree_ms"] = round(1e3 * (time.perf_counter() - t0), 3)
                    idx = idx.reshape(n, knn)
                    r["same_as_kdtree"] = bool(np.array_equal(A[:, 1].cpu().numpy(), idx.reshape(-1)))
                else:
                    r["kdtree_ms"] = "not measured"
                emit(r)
            del T1, T2
            torch.cuda.empty_cache()

    # the whole chain on the bunny: device (A from the clouds on the GPU, scored without a copy) against host (cKDTree)
    D1, D2 = clouds(9992, 3)
    ip = clp.invariants.EuclideanDistanceParams()
    ip.sigma, ip.epsilon = 0.01, 0.02
    beta = 0.0554

    def device_chain():
        T1, T2 = torch.from_numpy(D1).cuda(), torch.from_numpy(D2).cuda()
        A = clp.utils.distance_based_correspondences_dev(T1, T2, 1, beta, True)
        c = clp.CLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params())
        c.score_pairwise_consistency_dev(T1, T2, A)
        c.solve(np.full(A.shape[0], 0.5))
        return c.get_solution(), A.shape[0]

    def host_chain():
        _, idx = cKDTree(D2.T).query(D1.T, k=1, workers=-1)   # bm_utils.cpp's steps with knn = 1
        sd = np.sum((D1 - D2[:, idx]) ** 2, axis=0)
        keep = np.nonzero(sd <= beta * beta)[0]
        best = {}
        for i in keep.tolist():
            j = int(idx[i])
            if j not in best or sd[i] < sd[best[j]]:
                best[j] = i
        A = np.asfortranarray(np.array([[best[j], j] for j in sorted(best)], dtype=np.int32))
        c = clp.CLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params())
        c.score_pairwise_consistency(D1, D2, A)
        c.solve(np.full(A.shape[0], 0.5))
        return c.get_solution(), A.shape[0]

    for name, fn in (("device_chain", device_chain), ("host_chain", host_chain)):
        fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            s, m = fn()
            torch.cuda.synchronize()
            ts.append(1e3 * (time.perf_counter() - t0))
        emit(dict(case=name, n=9992, m=m, nodes=len(s.nodes), ms_median=round(float(np.median(ts)), 3)))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
