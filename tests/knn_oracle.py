"""numpy restatement of the putative-association generator (clp_correspondences, clp_knn.cuh; the reference's
benchmarks/bm_utils.cpp:147-232 with its undefined cases defined).

    sd(i, j) = sum_k (D1[k,i] - D2[k,j])^2, k = 0 .. d-1 in order, each subtract, multiply and add rounded on its own
    neighbours of i: the min(knn, n2) candidates of least (sd, j), NaN sd never one
    kept: sd <= radius * radius; rows by i, then rank
    1-to-1: per c1 the c0 of least sd (smallest c0 on a tie), rows by c1

numpy evaluates every elementwise operation correctly rounded and never contracts a multiply and an add, so the squared
distances here carry the device's bits.
"""
import numpy as np


def squared_distances(D1, D2, rows=slice(None)):
    """(n1', n2) squared distances of the columns D1[:, rows] to every column of D2, accumulated in order k = 0 .. d-1"""
    Q = D1[:, rows]
    s = None
    for k in range(D1.shape[0]):
        t = Q[k][:, None] - D2[k][None, :]
        s = t * t if s is None else s + t * t
    return s


def neighbours(D1, D2, knn, chunk=512):
    """(idx, sd): (n1, kk) int64 and float64, kk = min(knn, n2); idx -1 (sd NaN) where a query has fewer than kk
    candidates of non-NaN sd"""
    n1, n2 = D1.shape[1], D2.shape[1]
    kk = min(int(knn), n2)
    idx = np.full((n1, kk), -1, dtype=np.int64)
    sd = np.full((n1, kk), np.nan)
    for r0 in range(0, n1, chunk):
        S = squared_distances(D1, D2, slice(r0, r0 + chunk))
        # a stable sort keeps equal sd in ascending j: the order (sd, j); numpy sorts NaN last
        o = np.argsort(S, axis=1, kind="stable")[:, :kk]
        v = np.take_along_axis(S, o, axis=1)
        ok = ~np.isnan(v)
        idx[r0:r0 + chunk] = np.where(ok, o, -1)
        sd[r0:r0 + chunk] = v
    return idx, sd


def correspondences(D1, D2, knn, radius, enforce_1to1):
    """(m, 2) int32 associations, as clp_correspondences returns them"""
    D1 = np.asarray(D1, dtype=np.float64)
    D2 = np.asarray(D2, dtype=np.float64)
    n1, n2 = D1.shape[1], D2.shape[1]
    if n1 == 0 or n2 == 0:
        return np.zeros((0, 2), dtype=np.int32)
    idx, sd = neighbours(D1, D2, knn)
    r2 = np.float64(radius) * np.float64(radius)
    with np.errstate(invalid="ignore"):
        keep = (idx >= 0) & (sd <= r2)
    ii, rr = np.nonzero(keep)            # row-major: i ascending, then rank
    c0, c1, s = ii, idx[ii, rr], sd[ii, rr]
    if not enforce_1to1:
        return np.stack([c0, c1], axis=1).astype(np.int32)
    # per c1: least sd, then least c0 (the first pushed among equal sd, pushes come in c0 order)
    o = np.lexsort((c0, s, c1))
    first = np.ones(o.size, dtype=bool)
    first[1:] = c1[o][1:] != c1[o][:-1]
    sel = o[first]
    return np.stack([c0[sel], c1[sel]], axis=1).astype(np.int32)


def correspondences_loop(D1, D2, knn, radius, enforce_1to1):
    """the reference's loop (bm_utils.cpp:186-229) in plain Python over an exhaustive neighbour search, for small inputs:
    an independent statement of the same semantics"""
    D1 = np.asarray(D1, dtype=np.float64)
    D2 = np.asarray(D2, dtype=np.float64)
    d, n1, n2 = D1.shape[0], D1.shape[1], D2.shape[1]
    radius_sq = float(radius) * float(radius)
    rows, corres = [], {}
    for i in range(n1):
        cand = []
        for j in range(n2):
            s = 0.0
            for k in range(d):
                t = float(D1[k, i]) - float(D2[k, j])
                s = t * t if k == 0 else s + t * t
            if s == s:
                cand.append((s, j))
        cand.sort()
        for s, j in cand[:min(int(knn), n2)]:
            if s <= radius_sq:
                rows.append((i, j))
                corres.setdefault(j, []).append((s, i))
    if enforce_1to1:
        rows = []
        for j in sorted(corres):
            best = corres[j][0]
            for e in corres[j][1:]:
                if e[0] < best[0]:
                    best = e
            rows.append((best[1], j))
    return np.array(rows, dtype=np.int32).reshape(-1, 2)
