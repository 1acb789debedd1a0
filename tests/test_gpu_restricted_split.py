"""The split of the restricted sweeps (clp_resident.cuh, res_restrict_split): after each rebuild of S', the resident
packed solver cuts the row slots into contiguous, cost-balanced ranges, one per warp of the grid, and hands every row's
(M w, C w) to the CTA that owns the row as two tagged LL cells.  Only who sweeps a row changes, not how it is summed, so the solves
must match the oracle and be byte-identical from one handle to the next; CLP_PROF_CTAS reports the restricted entries
every CTA swept."""
import re

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


def _scored(clp, prob):
    cfg = prob["cfg"]
    ip = clp.invariants.EuclideanDistanceParams(); ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params())
    c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
    return c


def _handle(clp, M, C, **prm):
    p = clp.Params()
    for k, v in prm.items():
        setattr(p, k, v)
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()), p)
    c.set_sparse_matrix_data(M, C)
    assert c.dense_mode() == 6
    return c


def _oracle(orc, M, C, **prm):
    """the oracle fed the fp32 values the handle stores"""
    M32 = M.copy(); M32.data = M32.data.astype(np.float32).astype(np.float64)
    o = orc.Oracle(orc.default_params(**prm)) if prm else orc.Oracle()
    o.set_sparse_upper(M.shape[0], M32.indptr, M32.indices, M32.data, C.indptr, C.indices, C.data)
    return o


def _solve(c, u0):
    c.solve(u0)
    s = c.get_solution()
    return s, c.last_solve_sweeps()


def _same_as_oracle(s, so):
    assert sorted(s.nodes) == sorted(so.nodes.tolist())
    assert abs(s.score - so.score) <= 1e-5 * abs(so.score)


def _same_bytes(s, t):
    assert s.u.tobytes() == t.u.tobytes()
    assert np.float64(s.score).tobytes() == np.float64(t.score).tobytes()
    assert s.n_evals == t.n_evals and sorted(s.nodes) == sorted(t.nodes)


def test_concentrated_support(clp, orc, monkeypatch, capfd):
    """the planted cluster's vertices hold the longest rows, so S' lies in the first CTAs' items and most restricted
    entries belong to them; the split hands those rows to every CTA, each warp within one slot of its share"""
    from clipper_b200 import datagen
    p = datagen.weighted_matrix_problem(20000, 0.06, 71)
    M, C = p["M"], p["C"]
    m = M.shape[0]
    deg = np.diff(M.indptr) + np.bincount(M.indices, minlength=m)
    cluster = max(3, m // 16)
    coo = M.tocoo(); strong = coo.data >= 0.9  # only the planted cluster's pairs weigh 0.9 or more
    S = np.unique(np.concatenate([coo.row[strong], coo.col[strong]]))
    assert S.size == cluster and set(np.argsort(-deg, kind="stable")[:cluster]) == set(S)
    monkeypatch.setenv("CLP_PROF_CTAS", "2")
    s, sw, entries, over, _ = _cta_profile(_handle(clp, M, C), p["u0"], capfd)
    _same_as_oracle(s, _oracle(orc, M, C).solve(p["u0"]))
    assert sw["rebuild"] >= 1 and sw["restricted"] > 0, sw
    _balanced(sw, entries, over)


def test_tiny_support_largest_m(clp, orc):
    """m at the resident solver's cap, a planted cluster of 16 vertices in a sparse random graph: the last S' holds few
    columns and the split cuts ranges of a few entries per warp"""
    import scipy.sparse as sp
    m, k = 27648, 16
    rng = np.random.default_rng(5)
    want = int(0.018 * m * (m - 1) / 2)
    a = rng.integers(0, m, want + 8); b = rng.integers(0, m, a.size)
    keep = a != b
    key = np.unique(np.minimum(a[keep], b[keep]).astype(np.int64) * m + np.maximum(a[keep], b[keep]))
    S = np.sort(rng.choice(m, k, replace=False))
    si, sj = np.triu_indices(k, 1)
    ckey = S[si].astype(np.int64) * m + S[sj]
    key = np.concatenate([key[~np.isin(key, ckey)], ckey])
    w = np.concatenate([rng.uniform(0.05, 0.5, key.size - ckey.size), rng.uniform(0.95, 1.0, ckey.size)])
    M = sp.csc_matrix((w, (key // m, key % m)), shape=(m, m)); M.sort_indices()
    C = sp.csc_matrix((np.ones_like(w), (key // m, key % m)), shape=(m, m)); C.sort_indices()
    u0 = rng.random(m)
    c = _handle(clp, M, C)
    s, sw = _solve(c, u0)
    _same_as_oracle(s, _oracle(orc, M, C).solve(u0))
    assert sw["restricted"] > 0, sw


def test_tags_across_launches(clp):
    """two solves from different u0 on one handle: the cells of the first launch never stand in for the second's"""
    from clipper_b200 import datagen
    prob = datagen.config_problem("c2")
    u0b = np.random.default_rng(3).random(prob["cfg"]["m"])
    c = _scored(clp, prob)
    s1, sw1 = _solve(c, prob["u0"])
    s2, sw2 = _solve(c, u0b)
    assert sw1["restricted"] > 0 and sw2["restricted"] > 0, (sw1, sw2)
    f1, _ = _solve(_scored(clp, prob), prob["u0"])
    f2, _ = _solve(_scored(clp, prob), u0b)
    _same_bytes(s1, f1)
    _same_bytes(s2, f2)


def _second_cluster(m, density, seed, hub, whub):
    """datagen.weighted_matrix_problem plus `hub` vertices joined to every vertex of the planted cluster"""
    import scipy.sparse as sp
    from clipper_b200 import datagen
    p = datagen.weighted_matrix_problem(m, density, seed)
    M = p["M"].tocoo()
    key = M.row.astype(np.int64) * m + M.col
    w = M.data.copy()
    strong = w >= 0.9
    deg = np.bincount(np.concatenate([M.row[strong], M.col[strong]]), minlength=m)
    S1 = np.flatnonzero(deg >= max(3, m // 16) - 1)
    rng = np.random.default_rng(seed + 1)
    B = np.sort(rng.choice(np.setdiff1d(np.arange(m), S1), hub, replace=False))
    a, b = np.meshgrid(B, S1, indexing="ij")
    lo, hi = np.minimum(a, b).ravel().astype(np.int64), np.maximum(a, b).ravel()
    nk, nw = lo * m + hi, rng.uniform(0.9 * whub, whub, lo.size)
    keep = ~np.isin(key, nk)
    key, w = np.concatenate([key[keep], nk]), np.concatenate([w[keep], nw])
    M = sp.csc_matrix((w, (key // m, key % m)), shape=(m, m)); M.sort_indices()
    C = sp.csc_matrix((np.ones_like(w), (key // m, key % m)), shape=(m, m)); C.sort_indices()
    return M, C, p["u0"]


def test_repeated_rebuilds(clp, orc):
    """the regrowth problem of test_support_regrows re-splits at every rebuild: oracle parity, and the same bytes from
    two handles"""
    M, C, u0 = _second_cluster(12000, 0.08, 41, 3600, 0.5)
    s, sw = _solve(_handle(clp, M, C, maxiniters=10), u0)
    assert sw["rebuild"] >= 2 and sw["restricted"] > 0, sw
    _same_as_oracle(s, _oracle(orc, M, C, maxiniters=10).solve(u0))
    t, tw = _solve(_handle(clp, M, C, maxiniters=10), u0)
    assert tw == sw
    _same_bytes(s, t)


def _cta_profile(c, u0, capfd):
    """one solve with CLP_PROF_CTAS=2: per CTA the restricted entries swept and how far its costliest warp range of the
    split lay above the share total / (G NW), in costliest slots; and the "[clp prof] restricted entries" line"""
    capfd.readouterr()
    s, sw = _solve(c, u0)
    err = capfd.readouterr().err
    rows = [ln.split()[2:] for ln in err.splitlines() if ln.startswith("[clp cta]")]
    assert rows, err
    line = [ln for ln in err.splitlines() if ln.startswith("[clp prof] restricted entries")]
    return s, sw, np.array([float(r[7]) for r in rows]), np.array([float(r[8]) for r in rows]), line


def _balanced(sw, entries, over):
    """the split covers every restricted row exactly once (the CTAs' entries add up to the sweep counters) and no warp's
    range costs a whole slot more than its share (a range ends at the first slot whose prefix reaches the next share)"""
    assert entries.sum() == sw["entries"], (entries.sum(), sw)
    assert over.max() < 1.0, over
    assert over.max() > -1.0, over  # -1: no CTA reported a split


def test_split_balance(clp, monkeypatch, capfd):
    """CLP_PROF_CTAS=2 on config 2: every warp's range of the split lies within one slot of its share of the cost the
    split balances (chunks + kRowCost per row slot), the CTAs' entries add up to what clp_last_solve_sweeps counts, and
    the split depends on the data alone (the same per-CTA figures from two handles)"""
    from clipper_b200 import datagen
    monkeypatch.setenv("CLP_PROF_CTAS", "2")
    prob = datagen.config_problem("c2")
    s, sw, e1, o1, line = _cta_profile(_scored(clp, prob), prob["u0"], capfd)
    assert sw["restricted"] > 0, sw
    _balanced(sw, e1, o1)
    assert len(line) == 1 and re.search(r"max %d " % e1.max(), line[0]), line
    t, _, e2, o2, _ = _cta_profile(_scored(clp, prob), prob["u0"], capfd)
    assert np.array_equal(e1, e2) and np.array_equal(o1, o2)
    _same_bytes(s, t)
