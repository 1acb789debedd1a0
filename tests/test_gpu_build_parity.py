"""The compact build (device-wide sort, item scan and persistent fill) gives the same copy whichever way its counts
arrive: a scored handle (counts and windows from the scoring kernel) and a handle loaded through setMatrixData with the
scored handle's own affinity and constraint matrices (counting pass of the build) must solve bit for bit alike.  The
bytes of a pass (sparse_info) are checked against a host restatement of the stable sort: which rows head an item, and so
every item's length, follows from the sorted order."""
import numpy as np
import pytest

import packed_families as pf
from fixtures import bytes_per_pass

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def clp(built):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import clipper_b200 as clipperpy
    return clipperpy


def _handle(clp, cfg=None, mode=None):
    ip = clp.invariants.EuclideanDistanceParams()
    if cfg:
        ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params())
    if mode is not None:
        c.set_dense_mode(mode)
    return c


def _kept(c):
    A = c.get_affinity_matrix(); np.fill_diagonal(A, 0.0)
    return A != 0


def _same_solution(a, b, u0):
    a.solve(u0); b.solve(u0)
    sa, sb = a.get_solution(), b.get_solution()
    assert np.array_equal(sa.u, sb.u)
    assert sa.score == sb.score and sa.nodes == sb.nodes and sa.n_evals == sb.n_evals


@pytest.mark.parametrize("m,mode", [(3001, None), (9000, None), (20000, None), (9000, 3)])
def test_scored_and_loaded_builds_agree(clp, m, mode):
    """mode None: the resident (packed) layout, 20 000 = config 2; mode 3: column segments (several per row)"""
    from clipper_b200 import datagen
    prob = datagen.config_problem("c2", m)
    scored = _handle(clp, prob["cfg"], mode)
    scored.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
    loaded = _handle(clp, prob["cfg"], mode)
    loaded.set_matrix_data(scored.get_affinity_matrix(), scored.get_constraint_matrix())
    assert scored.dense_mode() == loaded.dense_mode() == (6 if mode is None else 3)
    assert scored.sparse_info() == loaded.sparse_info()
    kept = _kept(scored)
    if mode is None:
        want = bytes_per_pass(kept, True)
    else:
        import scipy.sparse as sp
        want = pf.seg_bytes_per_pass(sp.csr_matrix(kept), 4)[0]
    assert scored.sparse_info() == (int(kept.sum()), want)
    _same_solution(scored, loaded, prob["u0"])


@pytest.mark.parametrize("m", [3000, pf.RES_MAX_M])
def test_loaded_twice_agree_on_imbalanced_rows(clp, m):
    """F3 (heavy, empty and short rows; ties across many sort tiles): a second handle loaded from the first one's
    matrices builds the same copy"""
    case, _, _ = pf.f3_imbalance(m)
    U, Cu = case.dense_upper()
    M = U + U.T + np.eye(m); C = Cu + Cu.T + np.eye(m)
    first = _handle(clp)
    first.set_matrix_data(M, C)
    second = _handle(clp)
    second.set_matrix_data(first.get_affinity_matrix(), first.get_constraint_matrix())
    assert first.dense_mode() == second.dense_mode() == 6
    assert first.sparse_info() == second.sparse_info()
    kept = _kept(first)
    assert first.sparse_info() == (int(kept.sum()), bytes_per_pass(kept, True))
    _same_solution(first, second, np.random.default_rng(m).random(m))
