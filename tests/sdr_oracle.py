"""fp64 numpy restatement of the semidefinite relaxation the library solves (clp_sdp_solve, DESIGN §3 "SDR").

    maximise <M, X>  subject to  X >= 0 (PSD), tr X = 1,  X_ij = 0 where C_ij = 0,  X_ij >= 0 where C_ij != 0

Two-block ADMM on X in the spectraplex and Z in P = {Z symmetric, 0 off the pattern of C, >= 0 on it}; the device
kernel runs the same steps with a warm-started Jacobi eigensolver, this restatement with numpy.linalg.eigh.  The
projection onto the spectraplex is unique even with repeated eigenvalues, so both compute the same iterates up to
rounding.  `certificate` checks an answer without reference to the algorithm.
"""
import time

import numpy as np


def project_simplex(lam):
    """Euclidean projection of lam onto {p >= 0, sum p = 1}: p_i = max(lam_i - tau, 0)."""
    lam = np.asarray(lam, dtype=np.float64)
    s = np.sort(lam)[::-1]
    cs = 0.0
    tau = 0.0
    for j in range(s.size):  # sequential prefix sums, the kernel's order
        cs += s[j]
        t = (cs - 1.0) / (j + 1)
        if s[j] - t > 0:
            tau = t
    return np.maximum(lam - tau, 0.0)


def _bound(M, Y, pat):
    Yt = np.where(pat, np.minimum(Y, 0.0), Y)
    return float(np.linalg.eigvalsh(M - Yt)[-1])


def solve(M, C, max_iters=2000, eps_abs=1e-3, eps_rel=1e-3, time_limit_s=0.0):
    """Returns a dict with X, lambdas (ascending), evec1, thr, nodes, iters, converged, timed_out, value, bound,
    res_pri, res_dual, rho and the number of rebalances."""
    t0 = time.perf_counter()
    M = np.asarray(M, dtype=np.float64)
    m = M.shape[0]
    pat = np.asarray(C) != 0
    np.fill_diagonal(pat, True)
    Z = np.eye(m) / m
    U = np.zeros((m, m))
    rho = 1.0
    converged = timed_out = 0
    rebalances = 0
    bound = None
    k = 0
    for k in range(1, max_iters + 1):
        W = (Z - U) + M / rho
        lam, V = np.linalg.eigh(W)
        p = project_simplex(lam)
        Vp = V[:, p > 0]
        X = (Vp * p[p > 0]) @ Vp.T
        Zn = np.where(pat, np.maximum(X + U, 0.0), 0.0)
        U = U + X - Zn
        r_p = float(np.abs(X - Zn).max())
        r_d = rho * float(np.abs(Zn - Z).max())
        Z = Zn
        value = float((M * X).sum())
        bound = None
        if (r_p <= eps_abs + eps_rel * max(np.abs(X).max(), np.abs(Z).max())
                and r_d <= eps_abs + eps_rel * np.abs(rho * U).max()):
            bound = _bound(M, rho * U, pat)
            if abs(value - bound) <= eps_abs + eps_rel * max(abs(value), abs(bound)):
                converged = 1
                break
        if k % 10 == 0:
            if r_p > 10 * r_d:
                rho *= 2; U = U / 2; rebalances += 1
            elif r_d > 10 * r_p:
                rho /= 2; U = U * 2; rebalances += 1
        if time_limit_s > 0 and time.perf_counter() - t0 >= time_limit_s:
            timed_out = 1
            break
    if bound is None:
        bound = _bound(M, rho * U, pat)
    top = int(np.argmax(p))  # lowest index among equal largest p
    evec1 = V[:, top].copy()
    big = int(np.argmax(np.abs(evec1)))
    if evec1[big] < 0:
        evec1 = -evec1
    thr = float(np.abs(evec1).max() / 2)
    nodes = [i for i in range(m) if abs(evec1[i]) > thr]
    return dict(X=X, lambdas=np.sort(p), evec1=evec1, thr=thr, nodes=nodes, iters=k, converged=converged,
                timed_out=timed_out, value=value, bound=bound, res_pri=r_p, res_dual=r_d, rho=rho,
                rebalances=rebalances)


def certificate(M, C, X, bound, tol=1e-6):
    """Algorithm-independent check of an answer: X is PSD with unit trace, meets the pattern constraints to tol, and
    the dual bound is within tol of its value.  Returns a list of failures (empty: certified)."""
    M = np.asarray(M, dtype=np.float64)
    X = np.asarray(X, dtype=np.float64)
    pat = np.asarray(C) != 0
    np.fill_diagonal(pat, True)
    bad = []
    ev = np.linalg.eigvalsh((X + X.T) / 2)
    if ev[0] < -tol:
        bad.append("X not PSD: min eigenvalue %g" % ev[0])
    if abs(np.trace(X) - 1) > tol:
        bad.append("trace %r" % np.trace(X))
    if (~pat).any() and np.abs(X[~pat]).max() > tol:
        bad.append("off-pattern entry %g" % np.abs(X[~pat]).max())
    if X[pat].min() < -tol:
        bad.append("negative on-pattern entry %g" % X[pat].min())
    value = float((M * X).sum())
    if bound - value > tol:
        bad.append("gap %g" % (bound - value))
    return bad
