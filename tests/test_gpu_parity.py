"""GPU parity tests: the CUDA hot path (through the C-ABI) against the CPU oracle on the same
seeded inputs, against the reference's own fixtures, and -- at BASELINE.json's full size --
through size-independent properties.  Run with  pytest -m gpu  on an H100.

Tolerances (north_star: "matvec and objective within 1e-5 relative"):
  * CLP_STORE_F64 (strict-parity mode): affinities within 4 ulp(fp64) of the oracle (CUDA exp/acos
    vs glibc, each <= 1-2 ulp), identical sparsity pattern, mat-vec 1e-12, objective 1e-9,
    identical ifinal / evaluation count / inlier set.
  * CLP_STORE_F32 (default): affinities within 1 ulp(fp32) of the oracle's fp64 value rounded to
    fp32, identical pattern, mat-vec and objective 1e-5 relative, identical inlier set.
"""
import numpy as np
import pytest

import fixtures as fx

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


def make_euclid(clp, sigma=0.01, epsilon=0.06, mindist=0.0, storage=0, **pkw):
    ip = clp.invariants.EuclideanDistanceParams()
    ip.sigma, ip.epsilon, ip.mindist = sigma, epsilon, mindist
    p = clp.Params()
    for k, v in pkw.items():
        setattr(p, k, v)
    return clp.CLIPPER(clp.invariants.EuclideanDistance(ip), p, storage=storage)


def make_pn(clp, storage=0, **kw):
    ip = clp.invariants.PointNormalDistanceParams()
    for k, v in kw.items():
        setattr(ip, k, v)
    return clp.CLIPPER(clp.invariants.PointNormalDistance(ip), clp.Params(), storage=storage)


def assert_affinity_close(Mg, Mo, storage, ulps64=4):
    """pattern identical; values within the storage-type tolerance.
    EuclideanDistance: the distances and c=|l1-l2| are bit-identical to the oracle (IEEE sqrt, no
    FMA contraction), only exp() differs (CUDA vs glibc, each <= 1 ulp) -> 4 ulp(fp64).
    PointNormalDistance: acos() differs by <= 2 ulp and the score's condition number w.r.t. the
    angle difference is dn/sign^2 (up to ~35 at the defaults) -> callers pass ulps64=2048."""
    assert Mg.shape == Mo.shape
    pg, po = Mg != 0, Mo != 0
    assert np.array_equal(pg, po), "sparsity pattern differs in %d entries" % int((pg != po).sum())
    if storage == 1:
        err = np.abs(Mg - Mo)
        assert (err <= ulps64 * np.spacing(np.abs(Mo))).all(), err.max()
    else:
        Mo32 = Mo.astype(np.float32)
        err = np.abs(Mg.astype(np.float32) - Mo32)
        assert (err <= np.spacing(np.abs(Mo32))).all(), err.max()
        assert np.array_equal(Mg, Mg.astype(np.float32).astype(np.float64))


# ------------------------------------------------------------------------------------------
# the reference's own fixtures
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("storage", [0, 1])
def test_toy_affinity_and_inliers(clp, storage):
    # reference test/affinity_test.cpp:55-107 and test/clipper_test.cpp:56-66
    model, data = fx.toy_problem()
    c = make_euclid(clp, storage=storage)
    c.score_pairwise_consistency(model, data)
    A = c.get_initial_associations()
    assert A.shape == (12, 2)
    for i in range(4):
        for j in range(3):
            assert A[i * 3 + j, 0] == i and A[i * 3 + j, 1] == j
    M, C = c.get_affinity_matrix(), c.get_constraint_matrix()
    assert np.array_equal(np.diag(M), np.ones(12))
    assert np.array_equal(M, M.T) and np.array_equal(C, C.T)
    assert np.array_equal(M, C)
    assert np.array_equal(M, fx.MTRUE_12)
    for seed in [0, 2, 3, 4, 5, 6, 7, 8]:
        c.solve(np.random.default_rng(seed).random(12))
        Ain = c.get_selected_associations()
        assert sorted(map(tuple, Ain.tolist())) == [(0, 0), (1, 1), (2, 2)]
    c.solve()  # default: random u0 like the reference (utils.cpp:22-29); must run
    assert c.get_solution().u0.shape == (12,)


@pytest.mark.parametrize("storage", [0, 1])
def test_toy_get_set_roundtrip(clp, orc, storage):
    # reference test/clipper_test.cpp:115-124,181-196
    import scipy.sparse as sp
    model, data = fx.toy_problem()
    c = make_euclid(clp, storage=storage)
    c.score_pairwise_consistency(model, data)
    M, C = c.get_affinity_matrix(), c.get_constraint_matrix()
    c2 = make_euclid(clp, storage=storage)
    c2.set_matrix_data(M, C)
    assert np.array_equal(c2.get_affinity_matrix(), M) and np.array_equal(c2.get_constraint_matrix(), C)
    Mu = np.triu(M, 1); Cu = np.triu(C, 1)
    c3 = make_euclid(clp, storage=storage)
    c3.set_sparse_matrix_data(sp.csc_matrix(Mu), sp.csc_matrix(Cu))
    assert np.array_equal(c3.get_affinity_matrix(), M) and np.array_equal(c3.get_constraint_matrix(), C)
    u0 = np.full(12, 0.5)
    for cc in (c, c2, c3):
        cc.solve(u0)
    assert c.get_solution().nodes == c2.get_solution().nodes == c3.get_solution().nodes
    # SDR / max-clique entry points exist and behave like a build without SCS / PMC
    c2.solve_as_msrc_sdr(); assert c2.get_solution().nodes == [] and c2.get_solution().score == -1
    c2.solve_as_maximum_clique(); assert c2.get_solution().nodes == []


@pytest.mark.parametrize("storage", [0, 1])
def test_m20_weighted_vs_oracle(clp, orc, storage):
    # reference test/sdp_test.cpp:17-57 (the only bundled weighted problem)
    M, C = fx.m20()
    c = make_euclid(clp, storage=storage)
    c.set_matrix_data(M, C)
    o = orc.Oracle(); o.set_matrix_data(M, C)
    Mg = c.get_affinity_matrix()
    if storage == 1:
        assert np.array_equal(Mg, M)
    else:
        assert np.array_equal(Mg, M.astype(np.float32).astype(np.float64))
    assert np.array_equal(c.get_constraint_matrix(), C)
    for seed in range(4):
        u0 = np.random.default_rng(seed).random(20)
        c.solve(u0); sg = c.get_solution(); so = o.solve(u0)
        assert sg.nodes == so.nodes.tolist()
        tol = 1e-9 if storage == 1 else 1e-5
        assert abs(sg.score - so.score) <= tol * abs(so.score)
        assert np.allclose(sg.u, so.u, rtol=0, atol=1e-8 if storage == 1 else 1e-4)
        if storage == 1:
            assert sg.ifinal == so.ifinal and sg.n_evals == so.n_evals
    # Rounding::DSD on the solver output and the stand-alone DSD known answer (test/dsd_test.cpp)
    p = clp.Params(); p.rounding = clp.Rounding.DSD
    cd = clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()), p, storage=storage)
    cd.set_matrix_data(M, C); cd.solve(np.full(20, 1.0))
    assert set(cd.get_solution().nodes) <= set(fx.DSD_NODES_20) and len(cd.get_solution().nodes) >= 2
    p.rounding = clp.Rounding.NONZERO
    cn = clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()), p, storage=storage)
    cn.set_matrix_data(M, C); cn.solve(np.full(20, 1.0))
    o.params.rounding = 0
    assert cn.get_solution().nodes == o.solve(np.full(20, 1.0)).nodes.tolist()


@pytest.mark.parametrize("storage", [0, 1])
def test_planecloud_pointnormal_known_answer(clp, orc, storage):
    # reference examples/matlab/ex3_planecloud.m -- the only PointNormalDistance example with an answer
    D1, D2, Agt, pp = fx.planecloud()
    c = make_pn(clp, storage=storage, **pp)
    c.score_pairwise_consistency(D1, D2)
    o = orc.Oracle(); o.score_pointnormal(D1, D2, None, **pp)
    assert_affinity_close(c.get_affinity_matrix(), o.get_affinity_matrix(), storage, ulps64=2048)
    c.solve(np.full(16, 1.0))
    Ain = c.get_selected_associations()
    assert sorted(map(tuple, Ain.tolist())) == sorted(map(tuple, Agt.tolist()))


# ------------------------------------------------------------------------------------------
# seeded synthetic problems vs the oracle
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("storage", [0, 1])
@pytest.mark.parametrize("name,m", [("c1", None), ("c2", 256), ("c2", 2048), ("c2", 3001)])
def test_euclidean_score_matvec_solve_vs_oracle(clp, orc, name, m, storage):
    from clipper_b200 import datagen
    prob = datagen.config_problem(name, m); cfg = prob["cfg"]
    c = make_euclid(clp, sigma=cfg["sigma"], epsilon=cfg["epsilon"], storage=storage)
    c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
    o = orc.Oracle()
    o.score_euclidean(prob["D1"], prob["D2"], prob["A"], sigma=cfg["sigma"], epsilon=cfg["epsilon"])
    Mg, Mo = c.get_affinity_matrix(), o.get_affinity_matrix()
    assert_affinity_close(Mg, Mo, storage)
    assert np.array_equal(c.get_constraint_matrix(), o.get_constraint_matrix())
    assert np.array_equal(c.get_initial_associations(), prob["A"])
    nM, nC = c.count_nonzeros()
    assert nM == o.nnz(0) and nC == o.nnz(1)
    # K2: penalised mat-vec
    rng = np.random.default_rng(5)
    v = rng.random(cfg["m"]); d = 0.75
    y, Mv, Cv = c.matvec(v, d)
    yo, _ = o.gradf(v, d)
    tol = 1e-12 if storage == 1 else 1e-5
    assert np.abs(Mv - o.matvec(v, 0)).max() <= tol * np.abs(o.matvec(v, 0)).max()
    assert np.abs(Cv - o.matvec(v, 1)).max() <= 1e-12 * np.abs(o.matvec(v, 1)).max()
    assert np.abs(y - yo).max() <= tol * np.abs(yo).max()
    # K3-K6: solve
    c.solve(prob["u0"]); sg = c.get_solution(); so = o.solve(prob["u0"])
    assert sorted(sg.nodes) == sorted(so.nodes.tolist())
    assert sg.nodes == so.nodes.tolist() or storage == 0
    assert abs(sg.score - so.score) <= (1e-9 if storage == 1 else 1e-5) * abs(so.score)
    assert np.abs(sg.u - so.u).max() <= (1e-8 if storage == 1 else 1e-4)
    assert sg.ifinal == so.ifinal
    assert sg.n_matvec == sg.n_evals + 2
    if storage == 1:
        assert sg.n_evals == so.n_evals and sg.n_inner == so.n_inner
        assert abs(sg.d_final - so.d_final) <= 1e-9 * abs(so.d_final)
    assert np.array_equal(c.get_selected_associations(), prob["A"][np.asarray(sg.nodes), :])


@pytest.mark.parametrize("storage", [0, 1])
def test_pointnormal_vs_oracle(clp, orc, storage):
    from clipper_b200 import datagen
    prob = datagen.config_problem("c3", 700); cfg = prob["cfg"]
    kw = dict(sigp=cfg["sigp"], epsp=cfg["epsp"], sign=cfg["sign"], epsn=cfg["epsn"])
    c = make_pn(clp, storage=storage, **kw)
    c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
    o = orc.Oracle(); o.score_pointnormal(prob["D1"], prob["D2"], prob["A"], **kw)
    assert_affinity_close(c.get_affinity_matrix(), o.get_affinity_matrix(), storage, ulps64=2048)
    c.solve(prob["u0"]); sg = c.get_solution(); so = o.solve(prob["u0"])
    assert sorted(sg.nodes) == sorted(so.nodes.tolist())
    assert abs(sg.score - so.score) <= (1e-9 if storage == 1 else 1e-5) * abs(so.score)


def test_pointnormal_nan_is_zero(clp, orc):
    # SURVEY H3: unclamped acos; a normal slightly longer than 1 gives NaN -> score 0
    D1 = np.zeros((6, 3), order="F"); D2 = np.zeros((6, 3), order="F")
    D1[:3] = [[0, 1, 0], [0, 0, 1], [0, 0, 0]]; D2[:3] = D1[:3]
    D1[3:] = [[1 + 1e-12, 1, 0], [0, 0, 1], [0, 0, 0]]; D2[3:] = D1[3:]
    A = np.array([[0, 0], [1, 1], [2, 2]], dtype=np.int32)
    c = make_pn(clp, storage=1); c.score_pairwise_consistency(D1, D2, A)
    o = orc.Oracle(); o.score_pointnormal(D1, D2, A)
    assert np.array_equal(c.get_affinity_matrix() != 0, o.get_affinity_matrix() != 0)
    assert_affinity_close(c.get_affinity_matrix(), o.get_affinity_matrix(), 1, ulps64=2048)


@pytest.mark.parametrize("d", [1, 2, 3, 5])
def test_generic_dimension_and_mindist(clp, orc, d):
    rng = np.random.default_rng(d)
    n = 40
    D1 = np.asfortranarray(rng.random((d, n))); D2 = np.asfortranarray(D1 + 0.002 * rng.standard_normal((d, n)))
    m = 150
    A = np.stack([rng.integers(0, n, m), rng.integers(0, n, m)], axis=1).astype(np.int32)
    for mindist in (0.0, 0.2):
        c = make_euclid(clp, sigma=0.02, epsilon=0.05, mindist=mindist, storage=1)
        c.score_pairwise_consistency(D1, D2, A)
        o = orc.Oracle(); o.score_euclidean(D1, D2, A, sigma=0.02, epsilon=0.05, mindist=mindist)
        assert_affinity_close(c.get_affinity_matrix(), o.get_affinity_matrix(), 1)


@pytest.mark.parametrize("m", [1, 2, 3, 31, 32, 33, 127, 128, 129, 257])
def test_ragged_sizes(clp, orc, m):
    """edge sizes around the 32-row / 128-column tile boundaries; m=1 has no pairs at all.
    Distinct endpoints (no association shares a point): the first m//2 associations are true inliers and
    form the unique large clique, so the answer does not depend on rounding-level trajectory differences.
    (With many duplicated endpoints the landscape is degenerate: runs that differ only in summation order
    end in different -- equally valid -- cliques after thousands of evaluations.)"""
    rng = np.random.default_rng(m)
    n = max(64, 2 * m)
    D1 = np.asfortranarray(rng.random((3, n))); D2 = np.asfortranarray(D1 + 0.001 * rng.standard_normal((3, n)))
    A = np.stack([rng.permutation(n)[:m], rng.permutation(n)[:m]], axis=1).astype(np.int32)
    if m >= 3:
        A[: m // 2, 1] = A[: m // 2, 0]  # true inliers
        rest = np.setdiff1d(np.arange(n), A[: m // 2, 0])
        A[m // 2:, 1] = rng.permutation(rest)[: m - m // 2]
    for storage in (0, 1):
        c = make_euclid(clp, sigma=0.01, epsilon=0.05, storage=storage)
        c.score_pairwise_consistency(D1, D2, A)
        o = orc.Oracle(); o.score_euclidean(D1, D2, A, sigma=0.01, epsilon=0.05)
        assert_affinity_close(c.get_affinity_matrix(), o.get_affinity_matrix(), storage)
        u0 = rng.random(m) + 0.1
        c.solve(u0); sg = c.get_solution(); so = o.solve(u0)
        assert sorted(sg.nodes) == sorted(so.nodes.tolist())
        assert abs(sg.score - so.score) <= 1e-5 * max(1.0, abs(so.score))
        if m >= 31:  # DSD_HEU keeps round(F) nodes: the inlier clique up to a node or two
            assert len(set(range(m // 2)) & set(sg.nodes)) >= m // 2 - 2


def test_all_to_all_when_A_omitted(clp, orc):
    rng = np.random.default_rng(3)
    D1 = np.asfortranarray(rng.random((3, 9))); D2 = np.asfortranarray(D1[:, :7] + 0.0005)
    c = make_euclid(clp, storage=1); c.score_pairwise_consistency(D1, D2)
    o = orc.Oracle(); o.score_euclidean(D1, D2)
    assert np.array_equal(c.get_initial_associations(), o.get_initial_associations())
    assert np.array_equal(c.get_initial_associations(), clp.utils.create_all_to_all(9, 7))
    assert_affinity_close(c.get_affinity_matrix(), o.get_affinity_matrix(), 1)
    c.score_pairwise_consistency(D1, D2, np.zeros((0, 2), dtype=np.int32))  # empty A == all-to-all
    assert c.get_initial_associations().shape == (63, 2)


def test_no_affinity_no_penalty_entries(clp, orc):
    """SURVEY H6: setMatrixData allows C != pattern(M): (M=0,C=1) and (M>0,C=0) entries"""
    rng = np.random.default_rng(11)
    m = 60
    M = np.triu(rng.random((m, m)) * (rng.random((m, m)) < 0.3), 1)
    C = np.triu((rng.random((m, m)) < 0.5).astype(np.float64), 1)
    M = M + M.T + np.eye(m); C = C + C.T + np.eye(m)
    for storage in (0, 1):
        c = make_euclid(clp, storage=storage); c.set_matrix_data(M, C)
        o = orc.Oracle(); o.set_matrix_data(M, C)
        assert np.array_equal(c.get_constraint_matrix(), C)
        v = rng.random(m)
        y, Mv, Cv = c.matvec(v, 1.3); yo, _ = o.gradf(v, 1.3)
        assert np.abs(y - yo).max() <= (1e-12 if storage else 1e-5) * np.abs(yo).max()
        u0 = rng.random(m)
        c.solve(u0); so = o.solve(u0)
        assert sorted(c.get_solution().nodes) == sorted(so.nodes.tolist())


def test_params_are_honoured(clp, orc):
    from clipper_b200 import datagen
    prob = datagen.config_problem("c2", 400); cfg = prob["cfg"]
    for kw in (dict(rescale_u0=False), dict(maxiniters=3), dict(maxoliters=1), dict(maxlsiters=1),
               dict(beta=0.5, tol_u=1e-4, tol_F=1e-5), dict(affinityeps=0.3), dict(maxoliters=0)):
        c = make_euclid(clp, sigma=cfg["sigma"], epsilon=cfg["epsilon"], storage=1, **kw)
        c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
        p = orc.default_params(**{k: int(v) if isinstance(v, bool) else v for k, v in kw.items()})
        o = orc.Oracle(p)
        o.score_euclidean(prob["D1"], prob["D2"], prob["A"], sigma=cfg["sigma"], epsilon=cfg["epsilon"])
        c.solve(prob["u0"]); sg = c.get_solution(); so = o.solve(prob["u0"])
        assert sg.ifinal == so.ifinal, kw
        assert sg.n_evals == so.n_evals, kw
        assert abs(sg.score - so.score) <= 1e-9 * max(1.0, abs(so.score)), kw
        assert sorted(sg.nodes) == sorted(so.nodes.tolist()), kw


def test_custom_python_invariant_host_path(clp, orc):
    # reference examples/python/ex4_bunny.ipynb cells 13-15: a Python subclass of PairwiseInvariant
    class MyEuclid(clp.invariants.PairwiseInvariant):
        def __call__(self, ai, aj, bi, bj):
            c = abs(np.linalg.norm(ai - aj) - np.linalg.norm(bi - bj))
            return float(np.exp(-0.5 * c * c / 0.01 ** 2)) if c < 0.06 else 0.0
    model, data = fx.toy_problem()
    c = clp.CLIPPER(MyEuclid(), clp.Params())
    c.score_pairwise_consistency(model, data)
    assert np.array_equal(c.get_affinity_matrix(), fx.MTRUE_12)
    c.solve(np.full(12, 0.5))
    assert sorted(map(tuple, c.get_selected_associations().tolist())) == [(0, 0), (1, 1), (2, 2)]


def test_error_behaviour(clp):
    c = make_euclid(clp)
    with pytest.raises(clp.ClipperError):
        c.solve(np.ones(3))  # solve() before any matrix
    D = np.asfortranarray(np.random.default_rng(0).random((3, 5)))
    with pytest.raises(clp.ClipperError):
        c.score_pairwise_consistency(D, D, np.array([[0, 0], [7, 1]], dtype=np.int32))  # index out of range
    with pytest.raises(TypeError):
        c.score_pairwise_consistency(D.astype(np.float32), D)  # noconvert like clipperpy
    M = np.eye(4); M[0, 1] = M[1, 0] = -0.5
    with pytest.raises(clp.ClipperError):
        c.set_matrix_data(M, np.ones((4, 4)))  # negative affinity is outside the contract
    c.score_pairwise_consistency(D, D)
    with pytest.raises(ValueError):
        c.solve(np.ones(7))  # wrong u0 length


def test_deterministic_bitwise(clp):
    from clipper_b200 import datagen
    prob = datagen.config_problem("c2", 1500); cfg = prob["cfg"]
    outs = []
    for rep in range(3):
        c = make_euclid(clp, sigma=cfg["sigma"], epsilon=cfg["epsilon"])
        c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
        c.solve(prob["u0"]); s = c.get_solution()
        outs.append((s.u.tobytes(), s.score, tuple(s.nodes), s.n_evals))
    assert outs[0] == outs[1] == outs[2]


def test_device_pointer_entry_points(clp):
    """inputs resident in HBM (torch tensors), results identical to the host-pointer calls"""
    import ctypes as C
    import torch
    from clipper_b200 import datagen, _capi
    prob = datagen.config_problem("c2", 1024); cfg = prob["cfg"]
    c = make_euclid(clp, sigma=cfg["sigma"], epsilon=cfg["epsilon"])
    c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"]); c.solve(prob["u0"])
    ref = c.get_solution()
    dev = torch.device("cuda:0")
    D1 = torch.from_numpy(np.ascontiguousarray(prob["D1"].T)).to(dev)  # (n,3) row-major == (3,n) col-major
    D2 = torch.from_numpy(np.ascontiguousarray(prob["D2"].T)).to(dev)
    A = torch.from_numpy(np.ascontiguousarray(prob["A"].T)).to(dev)    # (2,m) row-major == (m,2) col-major
    u0 = torch.from_numpy(prob["u0"]).to(dev)
    uo = torch.empty_like(u0)
    g = make_euclid(clp, sigma=cfg["sigma"], epsilon=cfg["epsilon"])
    L = _capi.load()
    g.set_stream(torch.cuda.current_stream().cuda_stream)
    _capi.check(g.handle, L.clp_score_euclidean_dev(g.handle, D1.data_ptr(), 3, D1.shape[0], D2.data_ptr(), D2.shape[0],
                                                    A.data_ptr(), A.shape[1], cfg["sigma"], cfg["epsilon"], 0.0))
    s = _capi.ClpSolution(); nodes = np.zeros(1024, np.int32)
    _capi.check(g.handle, L.clp_solve_dev(g.handle, u0.data_ptr(), C.byref(s), uo.data_ptr(),
                                          nodes.ctypes.data_as(C.POINTER(C.c_int32))))
    torch.cuda.synchronize()
    assert nodes[: s.n_nodes].tolist() == ref.nodes and s.score == ref.score
    assert np.array_equal(uo.cpu().numpy(), ref.u)
    assert np.array_equal(g.get_initial_associations(), prob["A"])


# ------------------------------------------------------------------------------------------
# BASELINE.json full size (c2: m = 20000): size-independent properties
# ------------------------------------------------------------------------------------------
def test_full_size_c2_properties(clp):
    from clipper_b200 import datagen
    prob = datagen.config_problem("c2"); cfg = prob["cfg"]; m = cfg["m"]
    c = make_euclid(clp, sigma=cfg["sigma"], epsilon=cfg["epsilon"])
    c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
    nM, nC = c.count_nonzeros()
    assert nM == nC and 0.05 < nM / (m * (m - 1) / 2) < 0.30
    rng = np.random.default_rng(0)
    x, y = rng.random(m), rng.random(m)
    a, b, d = 0.3, -1.7, 0.9
    gx, Mx, Cx = c.matvec(x, d); gy, My, Cy = c.matvec(y, d); gz, Mz, Cz = c.matvec(a * x + b * y, d)
    # linearity of Mhat, Chat and Md
    for z, zx, zy in ((Mz, Mx, My), (Cz, Cx, Cy), (gz, gx, gy)):
        assert np.abs(z - (a * zx + b * zy)).max() <= 1e-9 * np.abs(z).max()
    # symmetry: x'(My) == y'(Mx)
    assert abs(x @ My - y @ Mx) <= 1e-10 * abs(x @ My)
    assert abs(x @ Cy - y @ Cx) <= 1e-10 * abs(x @ Cy)
    # C counts neighbours: Chat*1 are integers and sum to 2*nnz
    g1, M1, C1 = c.matvec(np.ones(m), 0.0)
    assert np.array_equal(C1, np.round(C1)) and C1.sum() == 2 * nC
    c.solve(prob["u0"]); s = c.get_solution()
    u = s.u
    assert (u >= 0).all() and abs(u @ u - 1) < 1e-12
    gu, _, _ = c.matvec(u, s.d_final)
    assert s.n_matvec == s.n_evals + 2 and s.ifinal >= 1
    # DSD_HEU: nodes are the round(F) largest entries of u, in descending order (utils.cpp:33-55)
    k = int(round(s.score))
    assert len(s.nodes) == k
    assert np.array_equal(np.asarray(s.nodes), clp.utils.find_indices_of_k_largest(u, k))
    assert (np.diff(u[np.asarray(s.nodes)]) <= 0).all()
    # the selected clique is (almost) entirely true inliers, which occupy rows [no, m)
    no = m - prob["ni"]
    prec = np.mean(np.asarray(s.nodes) >= no)
    assert prec > 0.95, prec
    # selected nodes are pairwise consistent: M restricted to them has no penalised pair on average
    assert s.kernel_ms > 0


# ------------------------------------------------------------------------------------------
# every sweep mode must agree with mode 0 (and each must match the oracle)
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("storage", [0, 1])
@pytest.mark.parametrize("m", [7, 100, 2047, 2049, 4500, 6200])
def test_sweep_modes_agree(clp, orc, m, storage):
    """mode 2 reads only the upper triangle (two-sided in-tile update); mode 0 reads the full matrix;
    mode 3 sweeps the segmented compact copy, mode 6 the full-row compact copy with the resident trial vector
    (another kernel: one synchronisation per evaluation); 4 picks automatically (= 6 at these sizes).  Sizes straddle
    the 2048-column stripe boundary, the diagonal-block logic and the 128-column segment steps."""
    from clipper_b200 import datagen
    prob = datagen.config_problem("c2", m); cfg = prob["cfg"]
    o = orc.Oracle()
    o.score_euclidean(prob["D1"], prob["D2"], prob["A"], sigma=cfg["sigma"], epsilon=cfg["epsilon"])
    so = o.solve(prob["u0"])
    rng = np.random.default_rng(m)
    v = rng.random(m)
    res = []
    modes = (0, 2, 3, 6, 4)
    effective = []
    for mode in modes:
        c = make_euclid(clp, sigma=cfg["sigma"], epsilon=cfg["epsilon"], storage=storage)
        c.set_dense_mode(mode)
        c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
        effective.append(c.dense_mode())
        y, Mv, Cv = c.matvec(v, 0.6)
        c.solve(prob["u0"]); s = c.get_solution()
        res.append((y, Mv, Cv, s))
    assert effective[:4] == [0, 2, 3, 6] and effective[4] in (2, 6)
    for k in range(1, len(modes)):
        assert np.abs(res[k][1] - res[0][1]).max() <= 1e-12 * max(1.0, np.abs(res[0][1]).max())
        assert np.abs(res[k][2] - res[0][2]).max() <= 1e-12 * max(1.0, np.abs(res[0][2]).max())
        assert np.abs(res[k][0] - res[0][0]).max() <= 1e-12 * max(1.0, np.abs(res[0][0]).max())
        s0, sk = res[0][3], res[k][3]
        assert sk.nodes == s0.nodes and sk.ifinal == s0.ifinal and sk.n_evals == s0.n_evals
        # the segmented kernels share every O(m) statement and differ only in how a row's products are grouped; the
        # resident kernel also groups the scalar reductions differently, so its trajectory agrees to rounding (1e-12 per
        # step) and its final objective to well below the solver's own stopping tolerance tol_F = 1e-9
        # (1e-12 held for every case on the round-1 synthetic cloud; on the bunny cloud the m = 4500 case reaches 4e-12
        # between two segmented sweeps: the differences are rounding noise amplified along ~70 evaluations)
        same_kernel = effective[k] in (0, 2, 3)
        assert abs(sk.score - s0.score) <= (1e-11 if same_kernel else 2e-11) * abs(s0.score)
        assert np.abs(sk.u - s0.u).max() <= (1e-11 if same_kernel else 1e-10)
    for _, _, _, s in res:
        assert sorted(s.nodes) == sorted(so.nodes.tolist())
        assert abs(s.score - so.score) <= (1e-9 if storage == 1 else 1e-5) * abs(so.score)


def test_full_matrix_stripe_sweep_is_rejected(clp):
    """there is no mode 1 (the stripe sweep reads the upper triangle only, as mode 2): asking for it is an error"""
    c = make_euclid(clp)
    with pytest.raises(clp.ClipperError):
        c.set_dense_mode(1)


@pytest.mark.parametrize("storage", [0, 1])
def test_compact_rows_keep_every_non_neutral_entry(clp, orc, storage):
    """mode 3 must keep (M=0,C=1) and (M>0,C=0) entries (SURVEY H6) -- only the -0.0 code is dropped"""
    rng = np.random.default_rng(21)
    m = 300
    M = np.triu(rng.random((m, m)) * (rng.random((m, m)) < 0.2), 1)
    C = np.triu((rng.random((m, m)) < 0.4).astype(np.float64), 1)
    M = M + M.T + np.eye(m); C = C + C.T + np.eye(m)
    o = orc.Oracle(); o.set_matrix_data(M, C)
    c = make_euclid(clp, storage=storage); c.set_dense_mode(3); c.set_matrix_data(M, C)
    assert c.dense_mode() == 3
    kept, nbytes = c.sparse_info()
    union = ((np.triu(M, 1) != 0) | (np.triu(C, 1) != 0)).sum() * 2
    assert kept == union
    v = rng.random(m)
    y, Mv, Cv = c.matvec(v, 1.1); yo, _ = o.gradf(v, 1.1)
    assert np.abs(y - yo).max() <= (1e-12 if storage else 1e-5) * np.abs(yo).max()
    assert np.abs(Cv - o.matvec(v, 1)).max() <= 1e-12 * np.abs(Cv).max()
    u0 = rng.random(m)
    c.solve(u0); so = o.solve(u0)
    assert sorted(c.get_solution().nodes) == sorted(so.nodes.tolist())
    # switching the sweep on an existing matrix re-finalises it
    c.set_dense_mode(0); y0, _, _ = c.matvec(v, 1.1)
    assert np.abs(y0 - y).max() <= 1e-12 * np.abs(y).max()


# ------------------------------------------------------------------------------------------
# committed golden files (tests/golden/*.npz: seeded inputs + the oracle's outputs, frozen by
# tests/test_oracle_golden.py::test_oracle_reproduces_golden_files)
# ------------------------------------------------------------------------------------------
def _golden_cases():
    import glob
    import os
    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    return sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(here, "*.npz")) if not os.path.basename(p).startswith("bun10k"))


@pytest.mark.parametrize("storage", [0, 1])
@pytest.mark.parametrize("name", _golden_cases())
def test_cuda_path_against_golden_files(clp, name, storage):
    import os
    import sys
    import scipy.sparse as sp
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import make_golden
    g = make_golden.load(name)
    m = g["A"].shape[0]
    if g["kind"] == "euclidean":
        c = make_euclid(clp, storage=storage, **g["params"]); ulps = 4
    else:
        c = make_pn(clp, storage=storage, **g["params"]); ulps = 2048
    c.score_pairwise_consistency(g["D1"], g["D2"], g["A"])
    U = sp.csc_matrix((g["M_val"], g["M_rowidx"], g["M_colptr"]), shape=(m, m)).toarray()
    Mo = U + U.T + np.eye(m)
    assert_affinity_close(c.get_affinity_matrix(), Mo, storage, ulps64=ulps)
    y, Mv, Cv = c.matvec(g["v"], float(g["d"]))
    tol = (1e-12 if g["kind"] == "euclidean" else 1e-9) if storage == 1 else 1e-5
    assert np.abs(Mv - g["Mv"]).max() <= tol * np.abs(g["Mv"]).max()
    assert np.abs(Cv - g["Cv"]).max() <= 1e-12 * np.abs(g["Cv"]).max()
    assert np.abs(y - g["gradf"]).max() <= tol * np.abs(g["gradf"]).max()
    c.solve(g["u0"]); s = c.get_solution()
    assert sorted(s.nodes) == sorted(g["nodes"].tolist())
    assert abs(s.score - float(g["score"])) <= (1e-9 if storage == 1 else 1e-5) * abs(float(g["score"]))
    assert np.abs(s.u - g["u"]).max() <= ((1e-8 if g["kind"] == "euclidean" else 1e-6) if storage == 1 else 1e-4)
    if storage == 1 and g["kind"] == "euclidean":  # strict-parity mode: the whole trajectory is the oracle's
        assert s.ifinal == int(g["ifinal"])       # (PointNormal values carry the acos difference, <= 2048 ulp)
        assert s.n_evals == int(g["n_evals"]) and s.n_inner == int(g["n_inner"])


@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("mindist", [0.0, 0.2])
@pytest.mark.parametrize("scale,shift", [(1.0, 0.0), (1e3, 0.0), (1e-3, 0.0), (1.0, 1e4)])
def test_screened_scoring_fp32_store(clp, orc, d, mindist, scale, shift):
    """default storage (fp32): the fp32-screened scoring kernel (compile-time d = 2, 3) must give the oracle's
    pattern exactly -- with mindist, at other coordinate scales and far from the origin (where the screening margin
    1024 * 2^-24 * R grows past epsilon and every pair takes the exact path)"""
    rng = np.random.default_rng(100 * d + int(mindist * 10) + int(np.log10(scale)) + int(shift > 0))
    n, m = 60, 333
    P = rng.random((d, n))
    D1 = np.asfortranarray(scale * P + shift); D2 = np.asfortranarray(scale * (P + 0.002 * rng.standard_normal((d, n))) + shift)
    A = np.stack([rng.integers(0, n, m), rng.integers(0, n, m)], axis=1).astype(np.int32)
    kw = dict(sigma=0.02 * scale, epsilon=0.05 * scale, mindist=mindist * scale)
    c = make_euclid(clp, storage=0, **kw)
    c.score_pairwise_consistency(D1, D2, A)
    o = orc.Oracle(); o.score_euclidean(D1, D2, A, **kw)
    assert_affinity_close(c.get_affinity_matrix(), o.get_affinity_matrix(), 0)
    nM, nC = c.count_nonzeros()
    assert nM == o.nnz(0) and nC == o.nnz(1)
    assert c.sparse_info()[0] in (0, 2 * o.nnz(0))  # kept entries of the compact copy (0: a dense sweep was chosen)


# ------------------------------------------------------------------------------------------
# resident-vector solver: the size limit (its two layouts: tests/test_gpu_packed.py)
# ------------------------------------------------------------------------------------------
def test_resident_at_its_size_limit(clp, orc):
    """m = 27 648: the fp64 trial vector takes 221 KB of the 227 KB of shared memory, the on-chip epilogue tables do
    not fit any more (HBM fallback); one column more and the segmented solver takes over."""
    from clipper_b200 import datagen
    for m, mode in ((27648, 6), (27649, 3)):
        prob = datagen.config_problem("c2", m); cfg = prob["cfg"]
        c = make_euclid(clp, sigma=cfg["sigma"], epsilon=cfg["epsilon"])
        c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
        assert c.dense_mode() == mode
        c.solve(prob["u0"]); s = c.get_solution()
        o = orc.Oracle(); o.score_euclidean(prob["D1"], prob["D2"], prob["A"], sigma=cfg["sigma"], epsilon=cfg["epsilon"])
        so = o.solve(prob["u0"])
        assert sorted(s.nodes) == sorted(so.nodes.tolist()) and abs(s.score - so.score) <= 1e-5 * abs(so.score)
