"""Graph families for the maximum-clique tests.

Every family is a dict with
  name    short id
  M, C    dense m x m inputs of set_matrix_data (C may carry (M=0, C=1) edges and (M>0, C=0) non-edges) -- or
  scored  ("euclidean" | "pointnormal", problem dict of clipper_b200.datagen, invariant parameters) for scoring
  claim   what the family is built to contain: {"omega": w} and/or {"clique": nodes} (checked on the CPU)
The graph of a family is C without its diagonal (for a scored family: the oracle's C).
"""
import numpy as np


def _inputs(adj, rng, weird=False):
    """M, C for set_matrix_data with the graph `adj` in the strict upper triangle.  weird: some edges carry M = 0
    (C = 1) and some non-edges carry M > 0 (C = 0) -- M's values must not matter."""
    n = adj.shape[0]
    C = np.triu(adj, 1).astype(np.float64)
    W = rng.uniform(0.05, 1.0, size=(n, n))
    M = np.where(C > 0, W, 0.0)
    if weird and n > 1:
        up = np.triu(np.ones((n, n), dtype=bool), 1)
        M[(C > 0) & (rng.random((n, n)) < 0.3)] = 0.0
        nonedge = up & (C == 0) & (rng.random((n, n)) < 0.3)
        M[nonedge] = W[nonedge]
    C = C + C.T + np.eye(n)
    M = np.triu(M, 1)
    M = M + M.T + np.eye(n)
    return np.asfortranarray(M), np.asfortranarray(C)


def _sym(A):
    A = np.triu(np.asarray(A, dtype=bool), 1)
    return A | A.T


def gnp(n, p, seed):
    rng = np.random.default_rng(seed)
    return _sym(rng.random((n, n)) < p)


def planted(n, p, k, seed):
    rng = np.random.default_rng(seed)
    A = gnp(n, p, seed)
    S = np.sort(rng.choice(n, size=k, replace=False))
    A[np.ix_(S, S)] = True
    np.fill_diagonal(A, False)
    return A, S.tolist()


def moon_moser(parts):
    """complete multipartite graph with `parts` triangles: 3^parts maximum cliques of size `parts`"""
    n = 3 * parts
    grp = np.arange(n) // 3
    A = grp[:, None] != grp[None, :]
    return A


def disjoint_cliques(q, size):
    n = q * size
    grp = np.arange(n) // size
    A = grp[:, None] == grp[None, :]
    np.fill_diagonal(A, False)
    return A


def star(n):
    A = np.zeros((n, n), dtype=bool)
    A[0, 1:] = True
    A[1:, 0] = True
    return A


def complete(n):
    A = np.ones((n, n), dtype=bool)
    np.fill_diagonal(A, False)
    return A


def straddling(n, starts, size, p, seed):
    """cliques of `size` starting at the given indices (crossing 32-bit word boundaries) in a sparse G(n, p)"""
    A = gnp(n, p, seed)
    for s in starts:
        S = np.arange(s, s + size)
        A[np.ix_(S, S)] = True
    np.fill_diagonal(A, False)
    return A


def graph_families():
    """every family given by its inputs (no scoring)"""
    import fixtures as fx
    out = []
    rng = np.random.default_rng(20240)
    for n in (1, 2, 3, 31, 32, 33, 64, 65, 200, 500):
        for p in (0.0, 0.1, 0.5, 0.9):
            A = gnp(n, p, seed=1000 * n + int(100 * p))
            M, C = _inputs(A, rng)
            out.append(dict(name="gnp_n%d_p%g" % (n, p), M=M, C=C, claim={}))
    for n, p, k in ((200, 0.1, 20), (500, 0.1, 25), (500, 0.5, 30)):
        A, S = planted(n, p, k, seed=7 * n + k)
        M, C = _inputs(A, rng)
        out.append(dict(name="planted_n%d_p%g_k%d" % (n, p, k), M=M, C=C, claim={"clique": S}))
    for parts in (4, 7):
        M, C = _inputs(moon_moser(parts), rng)
        out.append(dict(name="moon_moser_%d" % parts, M=M, C=C, claim={"omega": parts}))
    for q, size in ((3, 5), (8, 12)):
        M, C = _inputs(disjoint_cliques(q, size), rng)
        out.append(dict(name="disjoint_%dx%d" % (q, size), M=M, C=C, claim={"omega": size}))
    for n in (2, 40):
        M, C = _inputs(star(n), rng)
        out.append(dict(name="star_%d" % n, M=M, C=C, claim={"omega": 2}))
    for n in (1, 33, 70):
        M, C = _inputs(complete(n), rng)
        out.append(dict(name="complete_%d" % n, M=M, C=C, claim={"omega": n}))
    for n in (50, 97):
        M, C = _inputs(np.zeros((n, n), dtype=bool), rng)
        out.append(dict(name="edgeless_%d" % n, M=M, C=C, claim={"omega": 1}))
    A = straddling(160, (28, 60, 95), 9, 0.05, seed=5)
    M, C = _inputs(A, rng)
    out.append(dict(name="straddle_160", M=M, C=C, claim={"clique": list(range(28, 37))}))
    A = straddling(130, (30,), 36, 0.1, seed=6)  # one clique over three words
    M, C = _inputs(A, rng)
    out.append(dict(name="straddle_wide_130", M=M, C=C, claim={"clique": list(range(30, 66))}))
    A, S = planted(120, 0.3, 14, seed=9)
    M, C = _inputs(A, rng, weird=True)
    out.append(dict(name="weird_entries_120", M=M, C=C, claim={"clique": S}))
    out.append(dict(name="mtrue_12", M=np.asfortranarray(fx.MTRUE_12.copy()), C=np.asfortranarray(fx.MTRUE_12.copy()),
                    claim={"omega": 3}))
    M20, _ = fx.m20()
    out.append(dict(name="m20", M=np.asfortranarray(M20), C=np.asfortranarray((M20 > 0).astype(np.float64)), claim={}))
    return out


def scored_families(full=False):
    """scored problems: c1 (m = 1000), c2's parameters at m = 5000, PointNormal (c3's parameters) at m = 2000"""
    from clipper_b200 import datagen
    out = []
    for name, m in (("c1", None), ("c2", 5000), ("c3", 2000)):
        prob = datagen.config_problem(name, m=m)
        out.append(dict(name="scored_%s_m%d" % (name, prob["m"]), scored=prob))
    if full:
        prob = datagen.config_problem("c2")
        out.append(dict(name="scored_c2_full", scored=prob))
    return out


def adjacency(fam):
    """the boolean graph of a family (scored: the oracle's C), symmetric, no diagonal"""
    if "C" in fam:
        A = np.triu(fam["C"] != 0, 1)
        return A | A.T
    from oracle import clipper_oracle as orc
    prob = fam["scored"]
    cfg = prob["cfg"]
    o = orc.Oracle()
    if cfg["kind"] == "euclidean":
        o.score_euclidean(prob["D1"], prob["D2"], prob["A"], sigma=cfg["sigma"], epsilon=cfg["epsilon"])
    else:
        o.score_pointnormal(prob["D1"], prob["D2"], prob["A"], sigp=cfg["sigp"], epsp=cfg["epsp"],
                            sign=cfg["sign"], epsn=cfg["epsn"])
    m = o.m
    cp, ri, _ = o.get_csc(1)
    A = np.zeros((m, m), dtype=bool)
    cols = np.repeat(np.arange(m), np.diff(cp))
    A[ri, cols] = True
    A |= A.T
    np.fill_diagonal(A, False)
    return A
