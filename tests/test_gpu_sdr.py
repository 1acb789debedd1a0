"""The semidefinite relaxation on the GPU (clp_sdp_solve, clp_batch_sdp_matrices, solveAsMSRCSDR) against the numpy
restatement in tests/sdr_oracle.py and the algorithm-independent certificate, on the families of tests/sdr_families.py.
Run with  pytest -m gpu  on an H100.

  max_iters = 1, 2: X equal to the oracle's to 1e-12 (the cold and the warm-started eigensolver)
  full solves at the default tolerance and at 1e-7: the same nodes, iterations within one, X to 1e-9 where the
  iteration counts are equal, value and bound to 1e-9 relative; at 1e-7 the certificate holds
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import fixtures as fx
import sdr_families as fam
import sdr_oracle as so

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def clp(built):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import clipper_b200 as clipperpy
    return clipperpy


def _make(clp, storage=0):
    return clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()), clp.Params(),
                       storage=storage)


def _params(clp, max_iters=2000, eps=1e-3, time_limit=0.0):
    p = clp.SDPParams()
    p.max_iters, p.eps_abs, p.eps_rel, p.time_limit_secs = max_iters, eps, eps, time_limit
    return p


def _sdr(c, p):
    c.solve_as_msrc_sdr(p)
    s = c.get_solution()
    return s, s.sdp_info


def _loaded(clp, name, storage):
    """a handle holding the family, and the M, C it holds (what the kernel reads)"""
    c = _make(clp, storage)
    if name in fam.SCORED:
        kind, p = fam.scored_problem(name)
        if kind == "euclidean":
            c.score_pairwise_consistency(p["D1"], p["D2"], p["A"])
        else:
            c = clp.CLIPPER(clp.invariants.PointNormalDistance(clp.invariants.PointNormalDistanceParams()), clp.Params(),
                            storage=storage)
            c.score_pairwise_consistency(p["D1"], p["D2"], p["A"])
    else:
        M, Cm = fam.given(name)
        c.set_matrix_data(M, Cm)
    return c, c.get_affinity_matrix(), c.get_constraint_matrix()


CASES = [("m20", 0), ("m20", 1)] + [(n, 0) for n in fam.GIVEN if n != "m20"] + [(n, 0) for n in fam.SCORED]


@pytest.mark.parametrize("name,storage", CASES)
def test_family_against_oracle(clp, name, storage):
    c, M, Cm = _loaded(clp, name, storage)
    m = M.shape[0]
    for k in (1, 2):  # the first iterations pin the cold and the warm-started eigensolver
        s, info = _sdr(c, _params(clp, max_iters=k))
        o = so.solve(M, Cm, max_iters=k)
        assert (info["iters"], info["converged"]) == (o["iters"], o["converged"]), (k, info, o["value"], o["bound"])
        np.testing.assert_allclose(info["X"], o["X"], rtol=0, atol=1e-12)
    for eps in (1e-3, 1e-7):
        s, info = _sdr(c, _params(clp, eps=eps))
        o = so.solve(M, Cm, eps_abs=eps, eps_rel=eps)
        X = info["X"]
        assert info["converged"] == 1 and abs(info["iters"] - o["iters"]) <= 1, (eps, info["iters"], o["iters"])
        if name != "two_cliques":  # a double top eigenvalue: any vector of its space is an answer
            assert s.nodes == o["nodes"], (s.nodes, o["nodes"])
        if info["iters"] == o["iters"]:
            np.testing.assert_allclose(X, o["X"], rtol=0, atol=1e-9)
            assert info["value"] == pytest.approx(o["value"], rel=1e-9, abs=1e-12), (eps, info["value"], o["value"])
            assert info["bound"] == pytest.approx(o["bound"], rel=1e-9, abs=1e-12), (eps, info["bound"], o["bound"])
        # the outputs read out of the last iterate
        assert abs(np.trace(X) - 1) < 1e-10 and np.linalg.eigvalsh((X + X.T) / 2)[0] > -1e-12
        assert np.all(np.diff(info["lambdas"]) >= 0) and abs(info["lambdas"].sum() - 1) < 1e-12
        ev = info["evec1"]
        big = int(np.argmax(np.abs(ev)))
        assert ev[big] > 0 and info["thr"] == np.abs(ev).max() / 2
        assert s.nodes == [i for i in range(m) if abs(ev[i]) > info["thr"]]
        assert info["value"] == pytest.approx(float((M * X).sum()), rel=1e-12, abs=1e-14)
        assert info["pobj"] == -info["value"] and info["dobj"] == -info["bound"]
        assert s.score == -1 and s.u.shape == (m,) and not s.u.any()
        if eps == 1e-7:
            assert so.certificate(M, Cm, X, info["bound"]) == []


def test_reference_answers(clp):
    c, _, _ = _loaded(clp, "m20", 0)
    s, info = _sdr(c, _params(clp))
    assert s.nodes == [8, 9, 16]
    model, data = fx.toy_problem()
    c = _make(clp)
    c.score_pairwise_consistency(model, data)
    s, info = _sdr(c, _params(clp))
    assert s.nodes == [0, 4, 8]
    assert sorted(map(tuple, c.get_selected_associations().tolist())) == [(0, 0), (1, 1), (2, 2)]
    s1, info1 = _sdr(c, _params(clp, eps=1e-7))
    assert s1.nodes == [0, 4, 8]
    c.solve_as_msrc_sdr()  # without params: a build without SCS, nothing selected
    assert c.get_solution().nodes == [] and c.get_solution().score == -1


def test_small_and_degenerate(clp):
    c, _, _ = _loaded(clp, "m1", 0)
    s, info = _sdr(c, _params(clp))
    assert s.nodes == [0] and info["X"].tolist() == [[1.0]] and info["converged"] == 1
    c, _, _ = _loaded(clp, "eye", 0)
    s, info = _sdr(c, _params(clp, max_iters=1))
    np.testing.assert_allclose(info["X"], np.eye(16) / 16, atol=1e-14)


def test_determinism_and_handle_untouched(clp):
    c, M, Cm = _loaded(clp, "euclid64", 0)
    u0 = np.random.default_rng(5).random(64)
    c.solve(u0)
    before = c.get_solution()
    s1, i1 = _sdr(c, _params(clp, eps=1e-6))
    s2, i2 = _sdr(c, _params(clp, eps=1e-6))
    for k in ("X", "lambdas", "evec1"):
        assert np.array_equal(i1[k], i2[k])
    for k in ("iters", "value", "bound", "res_pri", "res_dual", "rho", "n_sweeps"):
        assert i1[k] == i2[k]
    assert s1.nodes == s2.nodes
    assert np.array_equal(c.get_affinity_matrix(), M) and np.array_equal(c.get_constraint_matrix(), Cm)
    c.solve(u0)
    after = c.get_solution()
    assert np.array_equal(before.u, after.u) and before.nodes == after.nodes and before.score == after.score


def test_errors_and_flags(clp):
    from clipper_b200 import _capi
    L = _capi.load()
    c = _make(clp)
    with pytest.raises(clp.ClipperError) as e:  # no matrix
        _sdr(c, _params(clp))
    assert e.value.code == 1
    M = np.eye(129)
    c.set_matrix_data(M, M)
    with pytest.raises(clp.ClipperError) as e:
        _sdr(c, _params(clp))
    assert e.value.code == 4 and "128" in str(e.value)
    c, M, Cm = _loaded(clp, "m20", 0)
    for bad in (dict(max_iters=0), dict(eps=-1.0), dict(eps=float("nan")), dict(time_limit=-1.0),
                dict(time_limit=float("nan"))):
        with pytest.raises(clp.ClipperError) as e:
            _sdr(c, _params(clp, **bad))
        assert e.value.code == 1
    info = _capi.ClpSdpInfo()
    assert L.clp_sdp_solve(c._h, None, C.byref(info), None, None, None, None) == 1
    p = _capi.ClpSdpParams()
    L.clp_sdp_default_params(C.byref(p))
    assert (p.max_iters, p.eps_abs, p.eps_rel, p.time_limit_s) == (2000, 1e-3, 1e-3, 0.0)
    assert L.clp_sdp_solve(c._h, C.byref(p), None, None, None, None, None) == 1
    assert L.clp_sdp_solve(c._h, C.byref(p), C.byref(info), None, None, None, None) == 0  # NULL outputs are fine
    assert info.n_nodes == 3
    raw = info
    # max_iters reached
    s, info = _sdr(c, _params(clp, max_iters=5, eps=1e-12))
    assert info["iters"] == 5 and info["converged"] == 0 and info["timed_out"] == 0
    # a tiny time limit: the last iterate, PSD with trace 1
    c2, _, _ = _loaded(clp, "euclid128", 0)
    s, info = _sdr(c2, _params(clp, eps=0.0, time_limit=1e-4))
    X = info["X"]
    assert info["timed_out"] == 1 and info["converged"] == 0 and info["iters"] < 2000
    assert abs(np.trace(X) - 1) < 1e-10 and np.linalg.eigvalsh((X + X.T) / 2)[0] > -1e-12
    # a sharded handle
    h = C.c_void_p()
    assert L.clp_create(0, 0, C.byref(h)) == 0
    try:
        assert L.clp_shard_config(h, 0, 2) == 0
        Mf, Cf = np.asfortranarray(M), np.asfortranarray(Cm)
        dp = C.POINTER(C.c_double)
        assert L.clp_set_dense(h, Mf.ctypes.data_as(dp), Cf.ctypes.data_as(dp), 20) == 0
        assert L.clp_sdp_solve(h, C.byref(p), C.byref(raw), None, None, None, None) == 4
        assert b"sharded" in L.clp_last_error(h)
    finally:
        L.clp_destroy(h)


def _csc_problem(M, Cm):
    import scipy.sparse as sp
    return dict(M=sp.csc_matrix(np.triu(M, 1)), C=sp.csc_matrix(np.triu(Cm, 1)))


def test_batch_equals_single_handles(clp):
    """more problems than CTAs, m from 1 to 128; each equals an fp32 handle after set_sparse_matrix_data, bit for bit"""
    import scipy.sparse as sp
    from clipper_b200 import datagen
    rng = np.random.default_rng(7)
    ms = [1, 2, 3, 127, 128] + rng.integers(1, 129, 295).tolist()
    problems = []
    for k, m in enumerate(ms):
        p = datagen.weighted_matrix_problem(m, float(rng.uniform(0.05, 0.5)), 100 + k, odd=0.1 if k % 3 == 0 else 0.0)
        problems.append(dict(M=p["M"], C=p["C"]))
    b = clp.MatrixBatchCLIPPER()
    params = _params(clp, eps=1e-5)
    out = b.sdr_many(problems, params)
    assert b.info()[0] < len(problems)
    for k, (prob, s) in enumerate(zip(problems, out)):
        c = _make(clp, 0)
        c.set_sparse_matrix_data(prob["M"], prob["C"])
        r, ri = _sdr(c, params)
        assert s.nodes == r.nodes, k
        for key in ("X", "lambdas", "evec1"):
            assert np.array_equal(s.sdp_info[key], ri[key]), (k, key)
        for key in ("iters", "converged", "value", "bound", "res_pri", "res_dual", "rho", "n_sweeps", "thr"):
            assert s.sdp_info[key] == ri[key], (k, key)
    # bad inputs name the first bad problem; the handle stays usable
    big = dict(M=sp.csc_matrix((129, 129)), C=sp.csc_matrix((129, 129)))
    with pytest.raises(clp.ClipperError) as e:
        b.sdr_many(problems[:3] + [big] + problems[3:5], params)
    assert e.value.code == 4 and "problem 3" in str(e.value)
    neg = _csc_problem(-fx.MTRUE_12 + 2 * np.eye(12), fx.MTRUE_12)
    with pytest.raises(clp.ClipperError) as e:
        b.sdr_many(problems[:2] + [neg], params)
    assert e.value.code == 4 and "problem 2" in str(e.value)
    with pytest.raises(clp.ClipperError) as e:
        b.sdr_many(problems[:2], _params(clp, max_iters=0))
    assert e.value.code == 1
    again = b.sdr_many(problems[:4], params)
    for s, t in zip(again, out[:4]):
        assert np.array_equal(s.sdp_info["X"], t.sdp_info["X"]) and s.nodes == t.nodes


def test_batch_time_limit(clp):
    problems = [_csc_problem(*fam.given("m20")) for _ in range(400)]
    b = clp.MatrixBatchCLIPPER()
    out = b.sdr_many(problems, _params(clp, eps=0.0, time_limit=2e-3))
    assert all(s.sdp_info["timed_out"] == 1 for s in out)
    for s in out[:5]:
        X = s.sdp_info["X"]
        assert abs(np.trace(X) - 1) < 1e-10 and np.linalg.eigvalsh((X + X.T) / 2)[0] > -1e-12


def test_cpp_sdp_tests(built):
    out = subprocess.run([os.path.join(ROOT, "clipper_b200", "lib", "sdp_tests")], capture_output=True, text=True,
                         timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "3 tests" in out.stdout and "0 failures" in out.stdout


def test_clipperpy_agrees_with_capi(clp):
    import sys
    lib = os.path.join(ROOT, "clipper_b200", "lib")
    if lib not in sys.path:
        sys.path.insert(0, lib)
    import clipperpy as cp
    M, Cm = fam.given("m20")
    c = cp.CLIPPER(cp.invariants.EuclideanDistance(cp.invariants.EuclideanDistanceParams()), cp.Params())
    c.set_matrix_data(M, Cm)
    c.solve_as_msrc_sdr()  # without params: nothing selected
    assert list(c.get_solution().nodes) == []
    c.solve_as_msrc_sdr(cp.SDPParams())
    g = _make(clp, 0)
    g.set_matrix_data(M, Cm)
    s, _ = _sdr(g, clp.SDPParams())
    assert list(c.get_solution().nodes) == s.nodes == [8, 9, 16]
    assert c.get_solution().score == -1
