"""Maximum clique of the constraint graph on the GPU (clp_max_clique / solve_as_maximum_clique) against the CPU
restatement in tests/clique_oracle.py, on every family of tests/clique_families.py, through fp32 and fp64 storage and
through set_matrix_data, set_sparse_matrix_data and scoring.  Run with  pytest -m gpu  on an H100.

  core numbers and KCORE nodes: equal to the oracle (core numbers are unique)
  HEU nodes: equal to the oracle's statement of the heuristic
  EXACT: a clique of C, no smaller than HEU; when the oracle proves omega within its node budget, the size equals
         omega and the GPU reports proven = 1.  A family the oracle cannot prove (dense G(n, p) at n = 200, 500) is
         checked for validity and for a size at least the oracle's best.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import clique_families as cf
import clique_oracle as co
import fixtures as fx

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT_LIMIT = 20.0  # seconds per EXACT call of a family the oracle proved
HARD_LIMIT = 5.0    # seconds per EXACT call of a family the oracle could not prove
ORACLE_BUDGET = 300_000

_cache = {}


def _oracle(fam):
    if fam["name"] not in _cache:
        A = cf.adjacency(fam)
        core = co.core_numbers_level(A)
        h = co.heu(A, core)
        K, proven = co.exact(A, budget=ORACLE_BUDGET, lb_clique=h)
        _cache[fam["name"]] = dict(A=A, core=core, heu=h, K=K, proven=proven)
    return _cache[fam["name"]]


@pytest.fixture(scope="module")
def clp(built):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import clipper_b200 as clipperpy
    return clipperpy


def _mc(clp, method, time_limit=EXACT_LIMIT):
    p = clp.MCParams()
    p.method, p.time_limit = method, time_limit
    return p


def _solve(c, clp, method, time_limit=EXACT_LIMIT):
    c.solve_as_maximum_clique(_mc(clp, method, time_limit))
    s = c.get_solution()
    return s.nodes, s.mc_info


def _make(clp, storage):
    return clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()), clp.Params(),
                       storage=storage)


def _load(c, fam, path):
    import scipy.sparse as sp
    if path == "dense":
        c.set_matrix_data(fam["M"], fam["C"])
    else:
        c.set_sparse_matrix_data(sp.csc_matrix(np.triu(fam["M"], 1)), sp.csc_matrix(np.triu(fam["C"], 1)))


def _check_family(clp, c, o, name):
    A, m = o["A"], o["A"].shape[0]
    core = c.core_numbers()
    assert core.tolist() == o["core"].tolist(), name
    mc = int(o["core"].max())
    nodes, info = _solve(c, clp, clp.MCMethod.KCORE)
    assert nodes == np.flatnonzero(o["core"] >= mc).tolist(), name
    assert info["max_core"] == mc and info["upper_bound"] == mc + 1 and info["n_edges"] == int(A.sum()) // 2
    nodes, info = _solve(c, clp, clp.MCMethod.HEU)
    assert nodes == o["heu"], name
    assert info["lower_bound"] == len(o["heu"])
    lb_eq_ub = len(o["heu"]) == mc + 1
    nodes, info = _solve(c, clp, clp.MCMethod.EXACT, 0)
    assert nodes == o["heu"] and info["proven"] == int(lb_eq_ub) and info["n_branches"] == 0, name
    limit = EXACT_LIMIT if o["proven"] else HARD_LIMIT
    nodes, info = _solve(c, clp, clp.MCMethod.EXACT, limit)
    assert co.is_clique(A, nodes) and nodes == sorted(nodes), name
    assert len(nodes) >= len(o["heu"]) and info["n_nodes"] == len(nodes)
    if o["proven"]:
        assert len(nodes) == len(o["K"]) and info["proven"] == 1 and info["timed_out"] == 0, (name, info)
    else:
        assert len(nodes) >= len(o["K"]) or info["timed_out"] == 1, (name, len(nodes), len(o["K"]), info)
        if info["proven"]:
            assert len(nodes) >= len(o["K"])
    if info["proven"]:  # a proven answer does not depend on the schedule
        again, info2 = _solve(c, clp, clp.MCMethod.EXACT, limit)
        assert again == nodes and info2["proven"] == 1, name
    return info


FAMILIES = cf.graph_families()


@pytest.mark.parametrize("path", ["dense", "sparse"])
@pytest.mark.parametrize("storage", [0, 1])
@pytest.mark.parametrize("fam", FAMILIES, ids=[f["name"] for f in FAMILIES])
def test_graph_family(clp, fam, storage, path):
    o = _oracle(fam)
    c = _make(clp, storage)
    _load(c, fam, path)
    _check_family(clp, c, o, fam["name"])
    s = c.get_solution()
    assert s.score == -1 and s.ifinal == 0 and not s.u.any() and s.u.shape == (o["A"].shape[0],)


SCORED = cf.scored_families()


@pytest.mark.parametrize("storage", [0, 1])
@pytest.mark.parametrize("fam", SCORED, ids=[f["name"] for f in SCORED])
def test_scored_family(clp, fam, storage):
    o = _oracle(fam)
    prob = fam["scored"]
    cfg = prob["cfg"]
    if cfg["kind"] == "euclidean":
        ip = clp.invariants.EuclideanDistanceParams()
        ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
        c = clp.CLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params(), storage=storage)
    else:
        ip = clp.invariants.PointNormalDistanceParams()
        ip.sigp, ip.epsp, ip.sign, ip.epsn = cfg["sigp"], cfg["epsp"], cfg["sign"], cfg["epsn"]
        c = clp.CLIPPER(clp.invariants.PointNormalDistance(ip), clp.Params(), storage=storage)
    c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
    if not o["proven"]:
        print("%s: the CPU oracle did not prove omega within %d nodes; EXACT is checked for validity and size only"
              % (fam["name"], ORACLE_BUDGET))
    info = _check_family(clp, c, o, fam["name"])
    print(fam["name"], info)
    Ain = c.get_selected_associations()
    assert Ain.shape == (len(c.get_solution().nodes), 2)


def test_full_size_c2(clp):
    """c2 at m = 20000: KCORE and HEU equal the oracle; EXACT under a bounded time limit returns a valid clique no
    smaller than HEU (whether it proves optimality there is reported, not assumed)"""
    fam = cf.scored_families(full=True)[-1]
    prob = fam["scored"]
    cfg = prob["cfg"]
    A = cf.adjacency(fam)
    core = co.core_numbers_level(A)
    heu = co.heu(A, core)
    ip = clp.invariants.EuclideanDistanceParams()
    ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params())
    c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
    assert c.core_numbers().tolist() == core.tolist()
    nodes, info = _solve(c, clp, clp.MCMethod.KCORE)
    assert nodes == np.flatnonzero(core >= core.max()).tolist()
    nodes, info = _solve(c, clp, clp.MCMethod.HEU)
    assert nodes == heu
    nodes, info = _solve(c, clp, clp.MCMethod.EXACT, 30)
    print("c2 full:", info)
    assert co.is_clique(A, nodes) and len(nodes) >= len(heu)


def test_time_limit_zero_and_repeat(clp):
    fam = [f for f in FAMILIES if f["name"] == "planted_n500_p0.5_k30"][0]
    o = _oracle(fam)
    c = _make(clp, 0)
    _load(c, fam, "dense")
    nodes, info = _solve(c, clp, clp.MCMethod.EXACT, 0)
    assert nodes == o["heu"] and info["proven"] == 0 and info["timed_out"] == 0
    first, info = _solve(c, clp, clp.MCMethod.EXACT)
    assert sorted(first) == first and len(first) == 30 and info["proven"] == 1 and info["n_branches"] > 0
    for _ in range(3):
        assert _solve(c, clp, clp.MCMethod.EXACT)[0] == first
        assert _solve(c, clp, clp.MCMethod.HEU)[0] == o["heu"]


def test_errors(clp):
    from clipper_b200 import _capi
    L = _capi.load()
    c = _make(clp, 0)
    with pytest.raises(clp.ClipperError):  # no matrix
        c.solve_as_maximum_clique(_mc(clp, clp.MCMethod.EXACT))
    c.set_matrix_data(np.eye(1), np.eye(1))
    nodes, info = _solve(c, clp, clp.MCMethod.EXACT)
    assert nodes == [0] and info["proven"] == 1
    with pytest.raises(clp.ClipperError):
        c.solve_as_maximum_clique(_mc(clp, 7))
    # a sharded handle holds only its own rows
    h = C.c_void_p()
    assert L.clp_create(0, 0, C.byref(h)) == 0
    try:
        assert L.clp_shard_config(h, 0, 2) == 0
        M, Cm = fx.m20()
        M, Cm = np.asfortranarray(M), np.asfortranarray(Cm)
        dp = C.POINTER(C.c_double)
        assert L.clp_set_dense(h, M.ctypes.data_as(dp), Cm.ctypes.data_as(dp), 20) == 0
        out = np.zeros(20, np.int32)
        rc = L.clp_max_clique(h, 0, 10.0, out.ctypes.data_as(C.POINTER(C.c_int32)), None)
        assert rc == 4 and b"sharded" in L.clp_last_error(h)
        assert L.clp_core_numbers(h, out.ctypes.data_as(C.POINTER(C.c_int32))) == 4
    finally:
        L.clp_destroy(h)


@pytest.mark.parametrize("storage", [0, 1])
def test_toy_max_clique_all_inputs(clp, storage):
    # reference test/clipper_test.cpp:115-124,181-196: the toy scored, set dense and set sparse; its inliers (0, 4, 8)
    # are the unique maximum clique of C
    import scipy.sparse as sp
    model, data = fx.toy_problem()
    c = _make(clp, storage)
    c.score_pairwise_consistency(model, data)
    M, Cm = c.get_affinity_matrix(), c.get_constraint_matrix()
    c2 = _make(clp, storage)
    c2.set_matrix_data(M, Cm)
    c3 = _make(clp, storage)
    c3.set_sparse_matrix_data(sp.csc_matrix(np.triu(M, 1)), sp.csc_matrix(np.triu(Cm, 1)))
    u0 = np.full(12, 0.5)
    for cc in (c, c2, c3):
        cc.solve(u0)
        u0_used = cc.get_solution().u0
        for method in (clp.MCMethod.EXACT, clp.MCMethod.HEU):
            cc.solve_as_maximum_clique(_mc(clp, method))
            s = cc.get_solution()
            assert s.nodes == [0, 4, 8] and s.score == -1 and s.ifinal == 0 and not s.u.any()
            assert s.u0 is u0_used  # untouched, as in the reference
        # without MCParams the Python mirror keeps its earlier behaviour: nothing selected
        cc.solve_as_maximum_clique()
        assert cc.get_solution().nodes == [] and cc.get_solution().score == -1
    c.solve_as_maximum_clique(_mc(clp, clp.MCMethod.EXACT))
    assert sorted(map(tuple, c.get_selected_associations().tolist())) == [(0, 0), (1, 1), (2, 2)]


def test_clipperpy_flow(built):
    """the pybind11 module: solve_as_maximum_clique, then get_selected_associations"""
    import sys
    lib = os.path.join(ROOT, "clipper_b200", "lib")
    if lib not in sys.path:
        sys.path.insert(0, lib)
    import clipperpy as cp
    from clipper_b200 import datagen
    prob = datagen.config_problem("c1")
    cfg = prob["cfg"]
    ip = cp.invariants.EuclideanDistanceParams()
    ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
    c = cp.CLIPPER(cp.invariants.EuclideanDistance(ip), cp.Params())
    c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
    fam = [f for f in SCORED if f["name"] == "scored_c1_m1000"][0]
    o = _oracle(fam)
    for method, want in ((cp.MCMethod.KCORE, np.flatnonzero(o["core"] >= o["core"].max()).tolist()),
                         (cp.MCMethod.HEU, o["heu"])):
        p = cp.MCParams(); p.method = method
        c.solve_as_maximum_clique(p)
        assert list(c.get_solution().nodes) == want
    c.solve_as_maximum_clique()  # EXACT by default
    s = c.get_solution()
    assert co.is_clique(o["A"], list(s.nodes)) and s.score == -1 and not np.asarray(s.u).any()
    if o["proven"]:
        assert len(s.nodes) == len(o["K"])
    Ain = c.get_selected_associations()
    assert Ain.shape == (len(s.nodes), 2)
    assert (Ain[:, 0] == Ain[:, 1]).mean() > 0.9  # the clique is made of inliers


def test_cpp_maxclique_tests(built):
    out = subprocess.run([os.path.join(ROOT, "clipper_b200", "lib", "maxclique_tests")], capture_output=True,
                         text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "3 tests" in out.stdout and "0 failures" in out.stdout
