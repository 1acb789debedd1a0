"""numpy restatement of the rigid transform of selected associations (include/clipper_b200.h, clp_estimate_transform).

estimate(D1, D2, A, rows) -> dict(T, status, k, rmse, sv, gap, R, t, mu_a) for D1 (d, n1), D2 (d, n2), A (m, 2) or None
(A None or m = 0: the all-to-all hypothesis, row r = (r // n2, r % n2)) and rows (k indices of A, or None: every row).
Two-pass fp64 means (shifted by the first pair, math.fsum), H = sum (b - mu_b)(a - mu_a)' on the centred points (math.fsum:
a BLAS product of 10^5 terms is off by more than the tolerances), np.linalg.svd, Umeyama's sign fix, the gap and status rules of the header.
"""
import math

import numpy as np

OK, EMPTY, DEGENERATE, NONFINITE = 0, 1, 2, 3
GAP_TOL = 1e-12


def pairs(D1, D2, A, rows):
    """the (d, k) arrays a and b of the used pairs"""
    n2 = D2.shape[1]
    if A is None or len(A) == 0:
        nrows = D1.shape[1] * n2
        idx = np.arange(nrows, dtype=np.int64) if rows is None else np.asarray(rows, dtype=np.int64)
        if idx.size and (idx.min() < 0 or idx.max() >= nrows):
            raise IndexError("row out of range")
        i1, i2 = idx // n2, idx % n2
    else:
        A = np.asarray(A)
        idx = np.arange(len(A), dtype=np.int64) if rows is None else np.asarray(rows, dtype=np.int64)
        if idx.size and (idx.min() < 0 or idx.max() >= len(A)):
            raise IndexError("row out of range")
        i1, i2 = A[idx, 0].astype(np.int64), A[idx, 1].astype(np.int64)
    return D1[:, i1], D2[:, i2]


def estimate(D1, D2, A=None, rows=None):
    D1 = np.asarray(D1, dtype=np.float64)
    D2 = np.asarray(D2, dtype=np.float64)
    d = D1.shape[0]
    a, b = pairs(D1, D2, A, rows)
    k = a.shape[1]
    T = np.eye(d + 1)
    if k == 0:
        return dict(T=T, status=EMPTY, k=0, rmse=0.0, sv=np.zeros(3), gap=0.0, R=np.eye(d), t=np.zeros(d),
                    mu_a=np.zeros(d))
    if not (np.isfinite(a).all() and np.isfinite(b).all()):
        T[:d, :] = np.nan
        return dict(T=T, status=NONFINITE, k=k, rmse=np.nan, sv=np.full(3, np.nan), gap=np.nan,
                    R=np.full((d, d), np.nan), t=np.full(d, np.nan), mu_a=np.full(d, np.nan))
    # the means as correctly rounded sums of x - x0, x0 the first pair (exact subtraction near x0: clouds far from the origin lose
    # nothing to the offset; all points equal gives the point itself)
    mu_a = a[:, 0] + np.array([math.fsum(r) for r in a - a[:, :1]]) / k
    mu_b = b[:, 0] + np.array([math.fsum(r) for r in b - b[:, :1]]) / k
    x, y = a - mu_a[:, None], b - mu_b[:, None]
    H = np.array([[math.fsum(y[r] * x[c]) for c in range(d)] for r in range(d)])  # correctly rounded sums
    U, s, Vt = np.linalg.svd(H)
    det = np.linalg.det(H)
    sign = -1.0 if det < 0 else 1.0
    sv = np.zeros(3)
    sv[:d] = s
    gap = s[d - 2] + sign * s[d - 1]
    if s[0] == 0:
        R = np.eye(d)
        status = DEGENERATE
    else:
        S = np.eye(d)
        S[d - 1, d - 1] = np.sign(np.linalg.det(U) * np.linalg.det(Vt))
        R = U @ S @ Vt
        status = OK if gap > GAP_TOL * s[0] else DEGENERATE
    t = mu_b - R @ mu_a
    T[:d, :d], T[:d, d] = R, t
    r = R @ x - y
    rmse = float(np.sqrt((r * r).sum() / k))
    return dict(T=T, status=status, k=k, rmse=rmse, sv=sv, gap=float(gap), R=R, t=t, mu_a=mu_a)


def rotation(d, rng):
    """a random proper rotation"""
    Q, Rr = np.linalg.qr(rng.standard_normal((d, d)))
    Q = Q * np.sign(np.diag(Rr))
    if np.linalg.det(Q) < 0:
        Q[:, 0] = -Q[:, 0]
    return Q
