"""The rigid transform of selected associations: the batched device call (estimate_rigid_transform_many_dev) against a
Python loop of single device calls (estimate_rigid_transform_dev) and against the numpy host loop (an SVD per
problem, the steps a caller without it takes), on the same problems; then single device calls at large k.

  problems: B in {1, 64, 1024, 4096}, k in {3, 100, 1000}: problem p is k points of the bunny (the reference's bun10k,
  tests/golden/bun10k_points.npz, a seeded subset) against a rotated and translated copy with noise 0.01; the rows
  are every row of A = (i, i).
  call ms: wall clock around the blocking call (median of --reps), clouds and A already on the device; the loops:
  the whole loop.  The numpy loop includes the copies of the rows' points to the host and of the transforms back.
  kernel ms: clp_tf_info.kernel_ms of the batched call (CUDA events around its kernels).
  single: k in {10^4, 10^5, 10^6}, one device call, call ms and kernel ms.
  same_as_loop: every batched T equals the looped single call's, bit for bit.

Prints the card's name and power limit, then one JSON line per measurement; --out also writes them to a JSON file.
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except OSError:
        return "unknown"


def problems(B, k, seed=5):
    """(D1, D2, A) CUDA tensors (B, 3, k), (B, 3, k), (B, k, 2)"""
    import torch
    from clipper_b200 import datagen
    cloud = datagen.make_cloud(9992)
    rng = np.random.default_rng(seed + 31 * k + 7 * B)
    n = min(k, 9992)
    P1 = np.empty((B, 3, k)); P2 = np.empty((B, 3, k))
    for p in range(B):
        X = cloud[:, rng.choice(9992, n, replace=False)]
        if k > n:
            X = np.tile(X, (1, (k + n - 1) // n))[:, :k] + 1e-3 * rng.standard_normal((3, k))
        Q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
        Q *= np.sign(np.linalg.det(Q))
        P1[p] = X
        P2[p] = Q @ X + rng.uniform(-1, 1, (3, 1)) + 0.01 * rng.standard_normal((3, k))
    A = np.repeat(np.arange(k, dtype=np.int32)[None, :, None], 2, 2).repeat(B, 0)
    return torch.from_numpy(P1).cuda(), torch.from_numpy(P2).cuda(), torch.from_numpy(np.ascontiguousarray(A)).cuda()


def timed(fn, reps):
    import torch
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts)), out


def numpy_loop(D1, D2, A):
    """the host loop a caller runs without the GPU estimate: copy the rows' points back, an SVD per problem, upload"""
    import torch
    a = D1.cpu().numpy(); b = D2.cpu().numpy(); idx = A.cpu().numpy()
    Ts = np.zeros((a.shape[0], 4, 4))
    for p in range(a.shape[0]):
        x = a[p][:, idx[p, :, 0]]; y = b[p][:, idx[p, :, 1]]
        mx, my = x.mean(1, keepdims=True), y.mean(1, keepdims=True)
        U, _, Vt = np.linalg.svd((y - my) @ (x - mx).T)
        S = np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt))])
        R = U @ S @ Vt
        Ts[p, :3, :3], Ts[p, :3, 3], Ts[p, 3, 3] = R, (my - R @ mx).ravel(), 1.0
    return torch.from_numpy(Ts).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, nargs="*", default=[1, 64, 1024, 4096])
    ap.add_argument("--k", type=int, nargs="*", default=[3, 100, 1000])
    ap.add_argument("--single-k", type=int, nargs="*", default=[10000, 100000, 1000000])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--loop-max", type=int, default=1024, help="largest B the Python loops are timed at")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import clipper_b200 as clp
    assert torch.cuda.is_available(), "bench_transform measures on the GPU"
    u = clp.utils
    rows = []

    def emit(r):
        r["card"] = dev_card
        print(json.dumps(r), flush=True)
        rows.append(r)

    dev_card = card()
    print("card:", dev_card, flush=True)
    for B in a.B:
        for k in a.k:
            D1, D2, A = problems(B, k)
            u.estimate_rigid_transform_many_dev(D1, D2, A)  # warm-up
            ms, (T, infos) = timed(lambda: u.estimate_rigid_transform_many_dev(D1, D2, A), a.reps)
            r = dict(case="batch", B=B, k=k, call_ms=ms, kernel_ms=infos[0].kernel_ms)
            if B <= a.loop_max:
                loop_ms, Ts = timed(lambda: [u.estimate_rigid_transform_dev(D1[p], D2[p], A[p])[0] for p in range(B)], 1)
                np_ms, Tn = timed(lambda: numpy_loop(D1, D2, A), 1)
                r.update(loop_ms=loop_ms, numpy_ms=np_ms,
                         same_as_loop=all(torch.equal(T[p], Ts[p]) for p in range(B)),
                         max_diff_numpy=float((T - Tn).abs().max()))
            emit(r)
    for k in a.single_k:
        D1, D2, A = problems(1, k)
        u.estimate_rigid_transform_dev(D1[0], D2[0], A[0])
        ms, (T, info) = timed(lambda: u.estimate_rigid_transform_dev(D1[0], D2[0], A[0]), a.reps)
        emit(dict(case="single", k=k, call_ms=ms, kernel_ms=info.kernel_ms, status=info.status))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
