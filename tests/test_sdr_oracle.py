"""The numpy restatement of the semidefinite relaxation (sdr_oracle.py) against the algorithm-independent certificate,
and the pinned answers of the reference's 20x20 matrix and the toy problem.  CPU only."""
import numpy as np
import pytest

import sdr_families as fam
import sdr_oracle as so


def _family(name):
    return fam.oracle_scored(name) if name in fam.SCORED else fam.given(name)


@pytest.mark.parametrize("name", fam.GIVEN + list(fam.SCORED))
def test_oracle_certified_at_tight_tolerance(name):
    M, C = _family(name)
    r = so.solve(M, C, eps_abs=1e-7, eps_rel=1e-7)
    assert r["converged"] == 1
    assert so.certificate(M, C, r["X"], r["bound"]) == []
    assert r["bound"] - r["value"] <= 1e-6


def test_simplex_projection():
    np.testing.assert_allclose(so.project_simplex([0.3, 0.3, -1.0]), [0.5, 0.5, 0.0])       # ties
    np.testing.assert_allclose(so.project_simplex([5.0, 0.1, -2.0]), [1.0, 0.0, 0.0])       # one positive entry
    np.testing.assert_allclose(so.project_simplex([2.0] * 4), [0.25] * 4)                   # all equal
    p = so.project_simplex(np.random.default_rng(3).normal(size=50))
    assert p.min() >= 0 and abs(p.sum() - 1) < 1e-14


def test_reference_matrix_answer():
    M, C = fam.given("m20")
    r = so.solve(M, C)
    assert r["nodes"] == [8, 9, 16] and r["converged"] == 1
    assert abs(np.trace(r["X"]) - 1) < 1e-12
    assert np.all(np.diff(r["lambdas"]) >= 0) and abs(r["lambdas"].sum() - 1) < 1e-12
    assert r["thr"] == pytest.approx(np.abs(r["evec1"]).max() / 2)


def test_toy_answer():
    M, C = fam.given("toy")
    assert so.solve(M, C)["nodes"] == [0, 4, 8]


def test_max_iters_and_rebalancing():
    M, C = fam.given("m20")
    r = so.solve(M, C, max_iters=5, eps_abs=1e-9, eps_rel=1e-9)
    assert r["iters"] == 5 and r["converged"] == 0 and r["rho"] == 1.0
    r = so.solve(M, C, max_iters=1)
    assert r["iters"] == 1 and r["converged"] == 0
    # W = I/m + M in the first iteration: X is the projection of its eigenvalues
    lam, V = np.linalg.eigh(np.eye(20) / 20 + M)
    p = so.project_simplex(lam)
    np.testing.assert_allclose(r["X"], (V * p) @ V.T, atol=1e-14)
    # rho is only rebalanced every 10 iterations, by a factor 2, while keeping rho U
    t = so.solve(M, C, eps_abs=1e-7, eps_rel=1e-7)
    assert t["rebalances"] >= 1 and np.log2(t["rho"]) == int(np.log2(t["rho"]))
    r9 = so.solve(M, C, max_iters=9, eps_abs=1e-12, eps_rel=1e-12)
    assert r9["rebalances"] == 0 and r9["rho"] == 1.0
