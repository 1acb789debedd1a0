"""Scored batches whose point clouds and associations are already on the GPU: BatchCLIPPER.solve_many_dev and
max_clique_many_dev (clp_batch_*_dev) against solve_many and max_clique_many on the same values, bit for bit, for the
built-in invariants and CudaInvariant; padded, strided, transposed, sliced and expanded tensors with poisoned padding;
the error codes and the first bad problem; a caller's stream; and CLIPPER.score_pairwise_consistency_dev against
score_pairwise_consistency."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_batch_custom import _all_to_all, _problems
from test_gpu_custom_invariant import EUCLID_SRC, NOTEBOOK_SRC

pytestmark = pytest.mark.gpu

SIZES = (1, 2, 127, 128, 129, 1000, 2048, 4096)
EXACT_LIMIT = 5.0


@pytest.fixture(scope="module")
def clp(built):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import clipper_b200 as clipperpy
    return clipperpy


def _with_d4(probs):
    """the problems with a fourth coordinate (a seeded function of the point) for the d = 4 invariant"""
    out = []
    for k, p in enumerate(probs):
        q = dict(p)
        for name in ("D1", "D2"):
            X = p[name]
            q[name] = np.asfortranarray(np.vstack([X, np.sin(7.0 * X[0] + k)[None, :] * 0.05]))
        out.append(q)
    return out


def _batch_problems(d, pointnormal=False, sizes=SIZES, seed=7100):
    """one batch mixing association lists of every size and all-to-all problems: 1 x 1, 64 x 64, and 64 x 64 inside
    the padding of the larger clouds"""
    dd = 6 if pointnormal else min(d, 3)
    probs = _problems(sizes, seed, d=dd, pointnormal=pointnormal)
    for n1, n2 in ((1, 1), (64, 64), (64, 64)):
        probs.append(_pn_all_to_all(seed + len(probs), n1, n2) if pointnormal
                     else _all_to_all(seed + len(probs), d=dd, n1=n1, n2=n2))
    return _with_d4(probs) if d == 4 else probs


def _pn_all_to_all(seed, n1, n2):
    """an all-to-all PointNormal problem: the first n1 and n2 points of a small seeded cloud and its perturbed copy"""
    from clipper_b200 import datagen
    prob = datagen.pointnormal_problem(64, 0.9, seed, n=200)
    return dict(D1=np.asfortranarray(prob["D1"][:, :n1]), D2=np.asfortranarray(prob["D2"][:, :n2]), A=None,
                u0=np.random.default_rng(seed).random(n1 * n2))


def _kinds(clp):
    ep = clp.invariants.EuclideanDistanceParams()
    pp = clp.invariants.PointNormalDistanceParams()
    return {
        "euclid2": (2, False, clp.invariants.EuclideanDistance(ep)),
        "euclid3": (3, False, clp.invariants.EuclideanDistance(ep)),
        "pointnormal": (6, True, clp.invariants.PointNormalDistance(pp)),
        "cuda_euclid3": (3, False, clp.invariants.CudaInvariant(EUCLID_SRC, (ep.sigma, ep.epsilon, ep.mindist))),
        "cuda_generic4": (4, False, clp.invariants.CudaInvariant(NOTEBOOK_SRC, (0.02, 0.08))),
    }


def _tensors(torch, probs, d_layout="contiguous", a_layout="contiguous", extra=(3, 5, 7)):
    """padded device tensors of a problem list: D1 (B, d, n1_max), D2 (B, d, n2_max) with NaN padding, A (B, m_max, 2)
    with -1 padding (all-to-all problems: m = 0), u0 (B, m_max) with NaN padding; and the sizes.  extra: padding added
    beyond the largest n1, n2 and m."""
    B = len(probs)
    d = probs[0]["D1"].shape[0]
    n1 = [p["D1"].shape[1] for p in probs]
    n2 = [p["D2"].shape[1] for p in probs]
    m = [0 if p["A"] is None else p["A"].shape[0] for p in probs]
    mu = [p["u0"].size for p in probs]
    N1, N2, MM = max(n1) + extra[0], max(n2) + extra[1], max(max(m), 1) + extra[2]
    D1 = np.full((B, d, N1), np.nan); D2 = np.full((B, d, N2), np.nan)
    A = np.full((B, MM, 2), -1, np.int32)
    U0 = np.full((B, max(max(mu), MM)), np.nan)
    for k, p in enumerate(probs):
        D1[k, :, :n1[k]] = p["D1"]; D2[k, :, :n2[k]] = p["D2"]
        if p["A"] is not None:
            A[k, :m[k]] = p["A"]
        U0[k, :mu[k]] = p["u0"]

    def dev(X, layout):
        t = torch.from_numpy(X).cuda()
        if layout == "contiguous":
            return t
        if layout == "transposed":  # (B, x, y) as a transposed view of a contiguous (B, y, x)
            return t.transpose(1, 2).contiguous().transpose(1, 2)
        assert layout == "slice"
        big = torch.full((X.shape[0] + 2, X.shape[1] + 3, X.shape[2] + 4), -7, dtype=t.dtype, device="cuda")
        big[1:X.shape[0] + 1, 2:X.shape[1] + 2, 3:X.shape[2] + 3] = t
        return big[1:X.shape[0] + 1, 2:X.shape[1] + 2, 3:X.shape[2] + 3]

    return (dev(D1, d_layout), dev(D2, d_layout), dev(A, a_layout), torch.from_numpy(U0).cuda(), n1, n2, m)


def _params(clp, rounding):
    p = clp.Params()
    p.rounding = rounding
    return p


def _same(host, dev, what):
    assert len(host) == len(dev), what
    for k, (s, t) in enumerate(zip(host, dev)):
        w = "%s, problem %d" % (what, k)
        assert s.u.tobytes() == t.u.cpu().numpy().tobytes(), w
        assert (s.score, s.d_final, s.ifinal, s.n_evals, s.n_inner) == (t.score, t.d_final, t.ifinal, t.n_evals, t.n_inner), w
        assert s.nodes == t.nodes, w


@pytest.mark.parametrize("rounding", ["NONZERO", "DSD_HEU"])
@pytest.mark.parametrize("kind", ["euclid2", "euclid3", "pointnormal", "cuda_euclid3", "cuda_generic4"])
def test_solve_matches_host(clp, kind, rounding):
    import torch
    d, pn, inv = _kinds(clp)[kind]
    probs = _batch_problems(d, pn)
    b = clp.BatchCLIPPER(inv, _params(clp, getattr(clp.Rounding, rounding)))
    host = b.solve_many(probs)
    kept = b.info()[2]
    D1, D2, A, U0, n1, n2, m = _tensors(torch, probs)
    dev = b.solve_many_dev(D1, D2, A, U0, n1, n2, m)
    _same(host, dev, kind)
    assert b.info()[2] == kept
    for k, (p, s) in enumerate(zip(probs, dev)):
        assert s.u0.cpu().numpy().tobytes() == p["u0"].tobytes()


@pytest.mark.parametrize("a_layout", ["contiguous", "transposed"])
@pytest.mark.parametrize("d_layout", ["contiguous", "transposed", "slice"])
def test_layouts(clp, d_layout, a_layout):
    import torch
    probs = _batch_problems(3, sizes=(1, 129, 1000, 2048), seed=7300)
    b = clp.BatchCLIPPER(_kinds(clp)["euclid3"][2], clp.Params())
    host = b.solve_many(probs)
    kept = b.info()[2]
    D1, D2, A, U0, n1, n2, m = _tensors(torch, probs, d_layout, a_layout)
    if d_layout != "contiguous":
        assert not D1.is_contiguous()
    if a_layout == "transposed":
        assert not A.is_contiguous()
    _same(host, b.solve_many_dev(D1, D2, A, U0, n1, n2, m), d_layout + "/" + a_layout)
    assert b.info()[2] == kept


def test_expanded_model_equals_copies(clp):
    """one model cloud against many scans: a batch-stride-0 D1 gives what explicit copies give"""
    import torch
    from clipper_b200 import datagen
    prob = datagen.euclidean_problem(2000, 0.8, 7400)
    B, n = 6, prob["D1"].shape[1]
    rng = np.random.default_rng(7400)
    model = torch.from_numpy(np.ascontiguousarray(prob["D1"])).cuda()
    scans = torch.from_numpy(np.stack([prob["D2"] + rng.normal(0, 0.002, prob["D2"].shape) for _ in range(B)])).cuda()
    A = torch.from_numpy(np.stack([prob["A"][rng.permutation(prob["A"].shape[0])[:1500]] for _ in range(B)])).cuda()
    U0 = torch.from_numpy(rng.random((B, 1500))).cuda()
    b = clp.BatchCLIPPER(_kinds(clp)["euclid3"][2], clp.Params())
    shared = model.unsqueeze(0).expand(B, 3, n)
    assert shared.stride(0) == 0
    a = b.solve_many_dev(shared, scans, A, U0)
    c = b.solve_many_dev(shared.contiguous(), scans, A, U0)
    for s, t in zip(a, c):
        assert s.u.cpu().numpy().tobytes() == t.u.cpu().numpy().tobytes()
        assert (s.score, s.nodes, s.n_evals) == (t.score, t.nodes, t.n_evals)
    host = b.solve_many([dict(D1=prob["D1"], D2=np.asfortranarray(scans[k].cpu().numpy()),
                              A=np.asfortranarray(A[k].cpu().numpy()), u0=U0[k].cpu().numpy()) for k in range(B)])
    _same(host, a, "expanded")


def _mc(clp, method, limit=EXACT_LIMIT):
    p = clp.MCParams()
    p.method, p.time_limit = method, limit
    return p


@pytest.mark.parametrize("kind", ["euclid3", "pointnormal", "cuda_euclid3"])
def test_max_clique_matches_host(clp, kind):
    import torch
    d, pn, inv = _kinds(clp)[kind]
    probs = _batch_problems(d, pn, sizes=(1, 2, 127, 128, 129, 1000), seed=7500)
    b = clp.BatchCLIPPER(inv, clp.Params())
    D1, D2, A, _, n1, n2, m = _tensors(torch, probs)
    for method in (clp.MCMethod.KCORE, clp.MCMethod.HEU, clp.MCMethod.EXACT):
        host = b.max_clique_many(probs, _mc(clp, method))
        dev = b.max_clique_many_dev(D1, D2, A, n1, n2, m, _mc(clp, method))
        for k, (s, t) in enumerate(zip(host, dev)):
            w = "%s %s problem %d" % (kind, method, k)
            assert s.core.tobytes() == t.core.tobytes(), w
            for f in ("max_core", "lower_bound", "upper_bound", "n_edges"):
                assert s.mc_info[f] == t.mc_info[f], w + " " + f
            if method != clp.MCMethod.EXACT:
                assert s.nodes == t.nodes and s.mc_info["proven"] == t.mc_info["proven"], w
            elif s.mc_info["proven"] and t.mc_info["proven"]:
                assert s.nodes == t.nodes, w


def _code(fn):
    import clipper_b200 as clipperpy
    with pytest.raises(clipperpy.ClipperError) as e:
        fn()
    return e.value.code, str(e.value)


def test_bad_indices_name_lowest_problem(clp):
    import torch
    probs = _problems((50, 60, 70, 80, 90, 100, 110), 7600)
    b = clp.BatchCLIPPER(_kinds(clp)["euclid3"][2], clp.Params())
    D1, D2, A, U0, n1, n2, m = _tensors(torch, probs)
    bad = A.clone()
    bad[5, 3, 1] = n2[5]        # one past the cloud (the padding holds NaN points)
    bad[3, 0, 0] = -1
    code, msg = _code(lambda: b.solve_many_dev(D1, D2, bad, U0, n1, n2, m))
    assert code == 1 and "problem 3:" in msg, msg
    code, msg = _code(lambda: b.max_clique_many_dev(D1, D2, bad, n1, n2, m, _mc(clp, clp.MCMethod.HEU)))
    assert code == 1 and "problem 3:" in msg, msg
    # the handle stays usable: the next call is correct
    _same(b.solve_many(probs), b.solve_many_dev(D1, D2, A, U0, n1, n2, m), "after the error")


def test_error_codes_match_host(clp):
    import torch
    from clipper_b200 import _capi
    ep = clp.invariants.EuclideanDistanceParams()
    probs = _problems((100, 200), 7700)
    b = clp.BatchCLIPPER(clp.invariants.EuclideanDistance(ep), clp.Params())
    D1, D2, A, U0, n1, n2, m = _tensors(torch, probs)
    # m[p] > 4096 and n1 n2 > 4096 for all-to-all: CLP_ERR_INVALID, as on the host
    big = _problems((4096,), 7701)[0]
    big["A"] = np.asfortranarray(np.vstack([big["A"], big["A"][:1]]))
    big["u0"] = np.concatenate([big["u0"], big["u0"][:1]])
    a2a = _all_to_all(7702, n1=65, n2=64)
    for p in (big, a2a):
        host = _code(lambda: b.solve_many([p]))[0]
        T = _tensors(torch, [p])
        assert _code(lambda: b.solve_many_dev(T[0], T[1], T[2] if p["A"] is not None else None, T[3], T[4], T[5],
                                              T[6] if p["A"] is not None else None))[0] == host == 1
    # a point stride of 0 (an expand along the points) and a NULL tensor: CLP_ERR_INVALID
    flat = D1[:, :, :1].expand(D1.shape[0], 3, D1.shape[2])
    assert _code(lambda: b.solve_many_dev(flat, D2, A, U0, n1, n2, m))[0] == 1
    pts = _capi.ClpPointsDev(None, (1, 1, 1), D2.data_ptr(), tuple(D2.stride()), A.data_ptr(), tuple(A.stride()),
                             (C.c_int64 * 2)(*n1), (C.c_int64 * 2)(*n2), (C.c_int64 * 2)(*m))
    sols = (_capi.ClpSolution * 2)()
    assert b._lib.clp_batch_solve_euclidean_dev(b._b, 2, 3, C.byref(pts), U0.data_ptr(), U0.stride(0), 0.01, 0.06, 0.0,
                                                sols, None, 0, None) == 1
    # Rounding::DSD: CLP_ERR_UNSUPPORTED on both paths
    p = clp.Params()
    p.rounding = clp.Rounding.DSD
    bd = clp.BatchCLIPPER(clp.invariants.EuclideanDistance(ep), p)
    assert _code(lambda: bd.solve_many(probs))[0] == _code(lambda: bd.solve_many_dev(D1, D2, A, U0, n1, n2, m))[0] == 4
    # Euclidean with d = 4: CLP_ERR_UNSUPPORTED on both paths
    p4 = _with_d4(probs)
    T = _tensors(torch, p4)
    assert _code(lambda: b.solve_many(p4))[0] == _code(lambda: b.solve_many_dev(*T[:4], *T[4:]))[0] == 4
    # PointNormalDistance with d != 6: ValueError on both paths
    bp = clp.BatchCLIPPER(clp.invariants.PointNormalDistance(clp.invariants.PointNormalDistanceParams()), clp.Params())
    with pytest.raises(ValueError):
        bp.solve_many(probs)
    with pytest.raises(ValueError):
        bp.solve_many_dev(D1, D2, A, U0, n1, n2, m)
    # the handle is still usable
    _same(b.solve_many(probs), b.solve_many_dev(D1, D2, A, U0, n1, n2, m), "after the errors")


def test_caller_stream(clp):
    import torch
    probs = _batch_problems(3, sizes=(128, 1000), seed=7800)
    b = clp.BatchCLIPPER(_kinds(clp)["euclid3"][2], clp.Params())
    D1, D2, A, U0, n1, n2, m = _tensors(torch, probs)
    ref = b.solve_many_dev(D1, D2, A, U0, n1, n2, m)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        b.set_stream(s.cuda_stream)
        D1s = D1.clone()      # written on the side stream just before the call
        got = b.solve_many_dev(D1s, D2, A, U0, n1, n2, m)
    b.set_stream(None)
    torch.cuda.synchronize()
    for x, y in zip(ref, got):
        assert x.u.cpu().numpy().tobytes() == y.u.cpu().numpy().tobytes()
        assert (x.score, x.nodes, x.n_evals) == (y.score, y.nodes, y.n_evals)


@pytest.mark.parametrize("all_to_all", [False, True])
@pytest.mark.parametrize("kind", ["euclid3", "pointnormal", "cuda_euclid3"])
def test_single_handle_score_dev(clp, kind, all_to_all):
    import torch
    d, pn, inv = _kinds(clp)[kind]
    if all_to_all:
        p = _pn_all_to_all(7900, 45, 40) if pn else _all_to_all(7900, n1=45, n2=40)
    else:
        p = _problems((1500,), 7900, d=d, pointnormal=pn)[0]
    a = clp.CLIPPER(inv, clp.Params())
    c = clp.CLIPPER(inv, clp.Params())
    a.score_pairwise_consistency(p["D1"], p["D2"], p["A"])
    # row-major device copies: the call lays them out column-major itself
    D1 = torch.from_numpy(np.ascontiguousarray(p["D1"])).cuda()
    D2 = torch.from_numpy(np.ascontiguousarray(p["D2"])).cuda()
    A = None if p["A"] is None else torch.from_numpy(np.ascontiguousarray(p["A"])).cuda()
    c.score_pairwise_consistency_dev(D1, D2, A)
    assert a.get_affinity_matrix().tobytes() == c.get_affinity_matrix().tobytes()
    assert a.get_constraint_matrix().tobytes() == c.get_constraint_matrix().tobytes()
    assert a.count_nonzeros() == c.count_nonzeros()
    assert np.array_equal(a.get_initial_associations(), c.get_initial_associations())
    a.solve(p["u0"]); c.solve(p["u0"])
    s, t = a.get_solution(), c.get_solution()
    assert s.u.tobytes() == t.u.tobytes() and s.nodes == t.nodes and (s.score, s.n_evals) == (t.score, t.n_evals)


def test_single_handle_score_dev_rejects_host_invariant(clp):
    import torch

    class HostInvariant(clp.invariants.PairwiseInvariant):
        def __call__(self, ai, aj, bi, bj):
            return 1.0

    c = clp.CLIPPER(HostInvariant(), clp.Params())
    X = torch.zeros((3, 4), dtype=torch.float64, device="cuda")
    with pytest.raises(TypeError):
        c.score_pairwise_consistency_dev(X, X)
