"""Sweeps over the support of the trial vector (clp_resident.cuh, res_support_kind): once the projected candidate has at
most m / 4 non-zeros, the resident packed solver (when its packed copy does not fit L2) copies every row's entries in
those columns into a restricted copy and sweeps only that copy while the support stays inside it.  The solves must still
match the oracle, and clp_last_solve_sweeps must show which sweeps ran."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def clp(built):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import clipper_b200 as clipperpy
    return clipperpy


@pytest.fixture(scope="module")
def orc():
    from oracle import clipper_oracle
    return clipper_oracle


def _scored(clp, orc, prob):
    cfg = prob["cfg"]
    ip = clp.invariants.EuclideanDistanceParams(); ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params())
    c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
    o = orc.Oracle()
    o.score_euclidean(prob["D1"], prob["D2"], prob["A"], sigma=cfg["sigma"], epsilon=cfg["epsilon"])
    return c, o


def _given(clp, orc, M, C, **prm):
    """the handle (fp32 storage) and the oracle fed the values the handle stores, both with the parameters prm"""
    p = clp.Params()
    for k, v in prm.items():
        setattr(p, k, v)
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()), p)
    c.set_sparse_matrix_data(M, C)
    M32 = M.copy(); M32.data = M32.data.astype(np.float32).astype(np.float64)
    o = orc.Oracle(orc.default_params(**prm)) if prm else orc.Oracle()
    o.set_sparse_upper(M.shape[0], M32.indptr, M32.indices, M32.data, C.indptr, C.indices, C.data)
    return c, o


def _solve_both(c, o, u0):
    so = o.solve(u0)
    c.solve(u0)
    sg = c.get_solution()
    sw = c.last_solve_sweeps()
    assert sw["full"] + sw["rebuild"] + sw["restricted"] == sg.n_evals
    assert sorted(sg.nodes) == sorted(so.nodes.tolist())
    assert abs(sg.score - so.score) <= 1e-5 * abs(so.score)
    return sg, sw


def _check_reads(c, sw, m):
    """a restricted sweep reads, per row, at most its kept entries and at most m / 4 of them, plus at most 3 padding
    entries up to a whole 4-entry chunk"""
    n = sw["rebuild"] + sw["restricted"]
    kept, _ = c.sparse_info()
    assert 0 < sw["entries"] <= n * min(kept, m * (m // 4)), sw
    assert sw["padding"] <= n * 3 * m, sw


def test_scored_problem_switches(clp, orc):
    """(a) config 2: the support falls below m / 4 and the solve switches to restricted sweeps; (b) the support then
    leaves S' again and S' is rebuilt.  Same node set and objective as the oracle."""
    from clipper_b200 import datagen
    prob = datagen.config_problem("c2")
    c, o = _scored(clp, orc, prob)
    assert c.dense_mode() == 6
    sg, sw = _solve_both(c, o, prob["u0"])
    assert sw["rebuild"] >= 2 and sw["restricted"] > 0, sw
    _check_reads(c, sw, prob["cfg"]["m"])


def test_copy_within_l2_sweeps_whole(clp, orc):
    """config 1's packed copy fits L2: every evaluation sweeps the whole copy"""
    from clipper_b200 import datagen
    prob = datagen.config_problem("c1")
    c, o = _scored(clp, orc, prob)
    assert c.dense_mode() == 6
    sg, sw = _solve_both(c, o, prob["u0"])
    assert sw == dict(full=sg.n_evals, rebuild=0, restricted=0, entries=0, padding=0, fallback=0)


def _second_cluster(m, density, seed, hub, whub):
    """datagen.weighted_matrix_problem plus a second group of `hub` vertices, each joined to every vertex of the planted
    cluster with weights U[0.9 whub, whub) (plain entries: M > 0 and C = 1 on every stored pair)"""
    import scipy.sparse as sp
    from clipper_b200 import datagen
    p = datagen.weighted_matrix_problem(m, density, seed)
    M = p["M"].tocoo()
    key = M.row.astype(np.int64) * m + M.col
    w = M.data.copy()
    strong = w >= 0.9  # only the planted cluster's pairs weigh 0.9 or more
    deg = np.bincount(np.concatenate([M.row[strong], M.col[strong]]), minlength=m)
    S1 = np.flatnonzero(deg >= max(3, m // 16) - 1)
    rng = np.random.default_rng(seed + 1)
    rest = np.setdiff1d(np.arange(m), S1)
    B = np.sort(rng.choice(rest, hub, replace=False))
    a, b = np.meshgrid(B, S1, indexing="ij")
    lo, hi = np.minimum(a, b).ravel().astype(np.int64), np.maximum(a, b).ravel()
    nk, nw = lo * m + hi, rng.uniform(0.9 * whub, whub, lo.size)
    keep = ~np.isin(key, nk)
    key, w = np.concatenate([key[keep], nk]), np.concatenate([w[keep], nw])
    M = sp.csc_matrix((w, (key // m, key % m)), shape=(m, m)); M.sort_indices()
    C = sp.csc_matrix((np.ones_like(w), (key // m, key % m)), shape=(m, m)); C.sort_indices()
    return M, C, p["u0"]


# m = 12 000 at density 0.08 plus 3 600 vertices joined to the first cluster: a packed copy larger than the 50 MB L2 of
# an H100.  Once the iterate sits on the first cluster, every joined vertex has a positive gradient, so the next trial
# point's support holds them all (more than m / 4).  maxiniters = 10 keeps the oracle's solve short (922 evaluations).
REGROW = (12000, 0.08, 41, 3600, 0.5)


def test_support_regrows(clp, orc):
    """(b) a second group of vertices: after the first rebuild the support leaves S' again, within m / 4 (another rebuild) and
    past it (full sweeps while a restricted copy exists, which keep S' and its copy as they are).  Same node set and
    objective as the oracle fed the stored values."""
    M, C, u0 = _second_cluster(*REGROW)
    c, o = _given(clp, orc, M, C, maxiniters=10)
    assert c.dense_mode() == 6
    _, sw = _solve_both(c, o, u0)
    assert sw["rebuild"] >= 2 and sw["fallback"] >= 1 and sw["restricted"] > 0, sw
    _check_reads(c, sw, M.shape[0])


def test_given_matrix(clp, orc):
    """a given weighted matrix (fp32 storage, packed): switches and matches the oracle fed the stored values"""
    from clipper_b200 import datagen
    p = datagen.weighted_matrix_problem(12000, 0.15, 31)
    c, o = _given(clp, orc, p["M"], p["C"])
    assert c.dense_mode() == 6
    _, sw = _solve_both(c, o, p["u0"])
    assert sw["rebuild"] >= 1 and sw["restricted"] > 0, sw


def test_dense_support_never_switches(clp, orc):
    """(c) half of the associations are inliers: the support never falls to m / 4, every evaluation sweeps the whole
    copy"""
    from clipper_b200 import datagen
    cfg = dict(datagen.CONFIGS["c2"], m=12000, rho=0.5)
    prob = dict(datagen.euclidean_problem(cfg["m"], cfg["rho"], cfg["seed"]), cfg=cfg)
    c, o = _scored(clp, orc, prob)
    sg, sw = _solve_both(c, o, prob["u0"])
    assert sw == dict(full=sg.n_evals, rebuild=0, restricted=0, entries=0, padding=0, fallback=0)


def test_largest_resident_m(clp, orc):
    """(d) m at the resident solver's cap: the largest restricted slots and bitmaps"""
    from clipper_b200 import datagen
    prob = datagen.config_problem("c2", 27648)
    c, o = _scored(clp, orc, prob)
    assert c.dense_mode() == 6
    _, sw = _solve_both(c, o, prob["u0"])
    assert sw["restricted"] > 0, sw


@pytest.mark.parametrize("odd", [0.1, 0.4])
def test_odd_entries(clp, orc, odd):
    """(e) entries with M = 0, C = 1 or M > 0, C = 0: the 6-byte copy, which sweeps the whole copy every time"""
    from clipper_b200 import datagen
    p = datagen.weighted_matrix_problem(4000, 0.01, 500 + int(100 * odd), odd=odd)
    c, o = _given(clp, orc, p["M"], p["C"])
    sg, sw = _solve_both(c, o, p["u0"])
    assert sw["full"] == sg.n_evals and sw["restricted"] == 0, sw
