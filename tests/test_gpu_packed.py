"""The resident solver's packed compact copy (4-byte entries: column delta + exponent code + mantissa, DESIGN.md section 2)
against the 6-byte layout (CLP_PACK=0) on the same problems, and the cases that must fall back to 6 bytes."""
import os

import numpy as np
import pytest

from fixtures import bytes_per_pass as _bytes_per_pass

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


class _env:
    """sets environment variables for the handles created inside (they are read when a handle is created)"""
    def __init__(self, **kw):
        self.kw = {k: str(v) for k, v in kw.items()}

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.kw}
        os.environ.update(self.kw)

    def __exit__(self, *exc):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _euclid(clp, cfg):
    ip = clp.invariants.EuclideanDistanceParams()
    ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
    return clp.CLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params())


def _run(clp, prob, pack, v):
    with _env(CLP_PACK=pack):
        c = _euclid(clp, prob["cfg"])
    c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
    assert c.dense_mode() == 6
    y, Mv, Cv = c.matvec(v, 0.6)
    c.solve(prob["u0"])
    return c, (y, Mv, Cv), c.get_solution()


def _assert_same(a, b):
    (ya, Mva, Cva), sa = a
    (yb, Mvb, Cvb), sb = b
    for x, r in ((Mva, Mvb), (Cva, Cvb), (ya, yb)):
        assert np.abs(x - r).max() <= 1e-12 * max(1.0, np.abs(r).max())
    assert sa.nodes == sb.nodes and sa.n_evals == sb.n_evals and sa.ifinal == sb.ifinal
    assert abs(sa.score - sb.score) <= 1e-12 * abs(sb.score)


@pytest.mark.parametrize("m", [3000, 3001, 9000])
def test_packed_equals_6_byte_layout(clp, orc, m):
    """both layouts: same decisions, objective and mat-vec to 1e-12, both equal to the oracle; sparse_info counts the
    bytes a pass reads.  Odd m: the last entry of the trial vector takes the scalar path beside the 16-byte-granular
    bulk copies of the staging."""
    from clipper_b200 import datagen
    prob = datagen.config_problem("c2", m); cfg = prob["cfg"]
    o = orc.Oracle(); o.score_euclidean(prob["D1"], prob["D2"], prob["A"], sigma=cfg["sigma"], epsilon=cfg["epsilon"])
    so = o.solve(prob["u0"])
    v = np.random.default_rng(m).random(m)
    kept = None
    got = {}
    for pack in (1, 0):
        c, mv, s = _run(clp, prob, pack, v)
        if kept is None:
            A = c.get_affinity_matrix(); np.fill_diagonal(A, 0.0); kept = A != 0
        assert c.sparse_info() == (int(kept.sum()), _bytes_per_pass(kept, pack == 1))
        assert sorted(s.nodes) == sorted(so.nodes.tolist())
        assert abs(s.score - so.score) <= 1e-5 * abs(so.score)
        got[pack] = (mv, s)
    _assert_same(got[1], got[0])


def test_packed_equals_6_byte_layout_c2_full_size(clp):
    """c2 at full size (m = 20 000, density 12.8 %)"""
    from clipper_b200 import datagen
    prob = datagen.config_problem("c2")
    v = np.random.default_rng(7).random(prob["cfg"]["m"])
    got = {}
    for pack in (1, 0):
        c, mv, s = _run(clp, prob, pack, v)
        got[pack] = (mv, s, c.sparse_info())
        del c
    _assert_same(got[1][:2], got[0][:2])
    assert got[1][2][0] == got[0][2][0]                 # same kept entries
    assert got[1][2][1] < 0.75 * got[0][2][1]            # a pass reads a quarter fewer bytes or better


def test_packed_is_bit_reproducible(clp):
    from clipper_b200 import datagen
    prob = datagen.config_problem("c2", 6000)
    v = np.random.default_rng(3).random(6000)
    c1, mv1, s1 = _run(clp, prob, 1, v)
    c2, mv2, s2 = _run(clp, prob, 1, v)
    c1.solve(prob["u0"]); s3 = c1.get_solution()
    for s in (s2, s3):
        assert np.array_equal(s.u, s1.u) and s.score == s1.score and s.n_evals == s1.n_evals
    for a, b in zip(mv1, mv2):
        assert np.array_equal(a, b)


def _weighted(m, seed, tiny=None, plus_zero=False):
    rng = np.random.default_rng(seed)
    M = np.triu(rng.uniform(0.05, 1.0, (m, m)) * (rng.random((m, m)) < 0.1), 1)
    C = (M > 0).astype(np.float64)
    if tiny is not None:
        M[3, 7] = tiny; C[3, 7] = 1.0
    if plus_zero:
        M[5, 11] = 0.0; C[5, 11] = 1.0        # no affinity, no penalty: stored as +0.0 (not plain)
    M = M + M.T + np.eye(m); C = C + C.T + np.eye(m)
    return M, C


@pytest.mark.parametrize("case", ["in_window", "below_window", "plus_zero"])
def test_packing_gate_and_fallback_vs_oracle(clp, orc, case):
    """setMatrixData: a plain matrix whose exponents fit 15 binades is packed; a value 2^-40 below the largest, or a
    non-plain +0.0 entry, keeps the 6-byte layout.  Every case equals the oracle."""
    m = 700
    M, C = _weighted(m, 5, tiny=1e-12 if case == "below_window" else None, plus_zero=case == "plus_zero")
    kept = ((M != 0) | (C != 0)) & ~np.eye(m, dtype=bool)
    o = orc.Oracle(); o.set_matrix_data(M, C)
    ip = clp.invariants.EuclideanDistanceParams()
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params())
    c.set_matrix_data(M, C)
    assert c.dense_mode() == 6
    assert c.sparse_info() == (int(kept.sum()), _bytes_per_pass(kept, case == "in_window"))
    rng = np.random.default_rng(9)
    v = rng.random(m)
    y, Mv, Cv = c.matvec(v, 1.1); yo, _ = o.gradf(v, 1.1)
    assert np.abs(y - yo).max() <= 1e-5 * np.abs(yo).max()
    assert np.abs(Cv - o.matvec(v, 1)).max() <= 1e-12 * np.abs(Cv).max()
    u0 = rng.random(m)
    c.solve(u0); so = o.solve(u0)
    assert sorted(c.get_solution().nodes) == sorted(so.nodes.tolist())
