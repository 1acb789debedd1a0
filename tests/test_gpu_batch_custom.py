"""Batches scored with a CUDA-source invariant (BatchCLIPPER with a CudaInvariant, clp_batch_*_custom).

Problem p must get exactly what an fp32 CLIPPER with the same invariant gives.  Restatements of the built-in invariants
are held to the built-in batch bit for bit (u, every scalar, nodes, the kept-entry count, and the clique answers); an
asymmetric invariant is held to a single handle's matrices solved by MatrixBatchCLIPPER, which pins the i < j argument
order and the stored bits.  Also covered: more problems than one round of scratch slots, the compile cache, the error
order and the parameters.
"""
import numpy as np
import pytest

from test_gpu_custom_invariant import ASYM_SRC, EUCLID_SRC, PN_SRC

pytestmark = pytest.mark.gpu

SIZES = (1, 4, 12, 127, 128, 129, 333, 1024, 2048, 4096)
AFFINITY_EPS = (1e-4, 0.0, -1.0)
EXACT_LIMIT = 5.0


@pytest.fixture(scope="module")
def clp(built):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import clipper_b200 as clipperpy
    return clipperpy


def _problems(sizes, seed0, d=3, pointnormal=False):
    """seeded problems on the benchmark cloud (associations shuffled, so small ones hold inliers too); only the points
    the associations touch travel"""
    from clipper_b200 import datagen
    out = []
    for k, m in enumerate(sizes):
        make = datagen.pointnormal_problem if pointnormal else datagen.euclidean_problem
        prob = make(max(m, 64), 0.9, seed0 + k)
        rows = np.random.default_rng(seed0 + k).permutation(prob["A"].shape[0])[:m]
        A = prob["A"][rows]
        used1, inv1 = np.unique(A[:, 0], return_inverse=True)
        used2, inv2 = np.unique(A[:, 1], return_inverse=True)
        out.append(dict(D1=np.asfortranarray(prob["D1"][:d, used1]), D2=np.asfortranarray(prob["D2"][:d, used2]),
                        A=np.asfortranarray(np.stack([inv1, inv2], axis=1).astype(np.int32)), u0=prob["u0"][rows].copy()))
    return out


def _all_to_all(seed, d=3, n1=12, n2=10):
    rng = np.random.default_rng(seed)
    D1 = rng.random((d, n1)) * 0.2
    D2 = D1[:, rng.permutation(n1)[:n2]] + rng.normal(0.0, 0.002, (d, n2))
    return dict(D1=np.asfortranarray(D1), D2=np.asfortranarray(D2), A=None, u0=rng.random(n1 * n2))


def _params(clp, ae, rounding=None):
    p = clp.Params()
    p.affinityeps = ae
    if rounding is not None:
        p.rounding = rounding
    return p


def _euclid(clp, sigma, epsilon, mindist):
    ip = clp.invariants.EuclideanDistanceParams()
    ip.sigma, ip.epsilon, ip.mindist = sigma, epsilon, mindist
    return clp.invariants.EuclideanDistance(ip), clp.invariants.CudaInvariant(EUCLID_SRC, (sigma, epsilon, mindist))


def _pointnormal(clp):
    ip = clp.invariants.PointNormalDistanceParams()
    return (clp.invariants.PointNormalDistance(ip),
            clp.invariants.CudaInvariant(PN_SRC, (ip.sigp, ip.epsp, ip.sign, ip.epsn)))


def _same_solutions(a, b, what):
    assert len(a) == len(b), what
    for k, (s, t) in enumerate(zip(a, b)):
        w = "%s, problem %d" % (what, k)
        assert s.u.tobytes() == t.u.tobytes(), w
        assert (s.score, s.d_final, s.ifinal, s.n_evals, s.n_inner) == (t.score, t.d_final, t.ifinal, t.n_evals, t.n_inner), w
        assert s.nodes == t.nodes, w


def _same_cliques(a, b, what, exact=False):
    for k, (s, t) in enumerate(zip(a, b)):
        w = "%s, problem %d" % (what, k)
        i, j = s.mc_info, t.mc_info
        assert s.core.tolist() == t.core.tolist(), w
        for f in ("max_core", "lower_bound", "upper_bound", "n_edges"):
            assert i[f] == j[f], (w, f)
        if not exact or (i["proven"] and j["proven"]):
            assert s.nodes == t.nodes, w


def _mc(clp, method, time_limit=EXACT_LIMIT):
    p = clp.MCParams()
    p.method, p.time_limit = method, time_limit
    return p


def _configs(clp):
    """(name, built-in invariant, its restatement, problems)"""
    e2 = _problems(SIZES, 900, d=2) + [_all_to_all(1, d=2)]
    e3 = _problems(SIZES, 920, d=3) + [_all_to_all(2, d=3)]
    pn = _problems(SIZES, 940, d=6, pointnormal=True)
    return [("euclid d2",) + _euclid(clp, 0.015, 0.05, 0.0) + (e2,),
            ("euclid d3",) + _euclid(clp, 0.015, 0.05, 0.0) + (e3,),
            ("euclid d3 mindist",) + _euclid(clp, 0.015, 0.05, 0.02) + (e3,),
            ("pointnormal",) + _pointnormal(clp) + (pn,)]


# ---- 1. restated built-ins, bit for bit ---------------------------------------------------------------------------
def test_restated_builtins_solve(clp):
    for name, builtin, restated, probs in _configs(clp):
        for ae in AFFINITY_EPS:
            for rounding in (clp.Rounding.DSD_HEU, clp.Rounding.NONZERO):
                what = "%s ae %g rounding %s" % (name, ae, rounding)
                b = clp.BatchCLIPPER(builtin, _params(clp, ae, rounding))
                c = clp.BatchCLIPPER(restated, _params(clp, ae, rounding))
                sb, sc = b.solve_many(probs), c.solve_many(probs)
                _same_solutions(sb, sc, what)
                assert b.info()[2] == c.info()[2] > 0, what


def test_restated_builtins_max_clique(clp):
    for name, builtin, restated, probs in _configs(clp):
        for ae in (1e-4, -1.0):
            b = clp.BatchCLIPPER(builtin, _params(clp, ae))
            c = clp.BatchCLIPPER(restated, _params(clp, ae))
            for method in (clp.MCMethod.KCORE, clp.MCMethod.HEU, clp.MCMethod.EXACT):
                what = "%s ae %g method %s" % (name, ae, method)
                mp = _mc(clp, method)
                _same_cliques(b.max_clique_many(probs, mp), c.max_clique_many(probs, mp), what,
                              exact=method == clp.MCMethod.EXACT)


# ---- 2. asymmetric invariant against the single handle ------------------------------------------------------------
def _asym_problems():
    out = []
    for k, (n, m) in enumerate(((40, 150), (60, 400), (90, 1000), (25, 129))):
        rng = np.random.default_rng(30 + k)
        D1 = rng.integers(-3, 4, (2, n)).astype(np.float64)
        D2 = rng.integers(-3, 4, (2, n)).astype(np.float64)
        A = np.asfortranarray(np.stack([rng.integers(0, n, m), rng.integers(0, n, m)], 1).astype(np.int32))
        out.append(dict(D1=np.asfortranarray(D1), D2=np.asfortranarray(D2), A=A, u0=rng.random(m)))
    return out


def test_asymmetric_invariant_matches_single_handle(clp):
    probs = _asym_problems()
    for offset in (0.25, 1.5, -0.5):
        inv = clp.invariants.CudaInvariant(ASYM_SRC, (offset,))
        mats, single_mc = [], []
        for p in probs:
            h = clp.CLIPPER(inv, clp.Params())   # fp32 storage
            h.score_pairwise_consistency(p["D1"], p["D2"], p["A"])
            mats.append(dict(M=h.get_affinity_matrix(), C=h.get_constraint_matrix(), u0=p["u0"]))
            nodes = []
            for method in (clp.MCMethod.KCORE, clp.MCMethod.HEU):
                h.solve_as_maximum_clique(_mc(clp, method))
                nodes.append(h.get_solution().nodes)
            single_mc.append(nodes)
        assert sum(np.count_nonzero(np.triu(x["C"], 1)) for x in mats) > 1000
        ref = clp.MatrixBatchCLIPPER(clp.Params()).solve_many(mats)
        c = clp.BatchCLIPPER(inv, clp.Params())
        _same_solutions(ref, c.solve_many(probs), "asym offset %g" % offset)
        for k, method in enumerate((clp.MCMethod.KCORE, clp.MCMethod.HEU)):
            got = c.max_clique_many(probs, _mc(clp, method))
            for q, s in enumerate(got):
                assert s.nodes == sorted(single_mc[q][k]), ("asym offset %g method %s problem %d" % (offset, method, q))


# ---- 3. more problems than one round ------------------------------------------------------------------------------
def test_many_rounds(clp):
    rng = np.random.default_rng(77)
    sizes = rng.integers(4, 601, 1000).tolist()
    probs = _problems(sizes, 3000)
    builtin, restated = _euclid(clp, 0.015, 0.05, 0.0)
    c = clp.BatchCLIPPER(restated, clp.Params())
    first = c.solve_many(probs)
    ctas = c.info()[0]
    assert ctas < len(probs), "one round held every problem: %d slots" % ctas
    _same_solutions(first, c.solve_many(probs), "second call")
    one = clp.BatchCLIPPER(restated, clp.Params())
    for k in range(0, len(probs), 7):
        _same_solutions([first[k]], one.solve_many([probs[k]]), "problem %d alone" % k)
    _same_solutions(clp.BatchCLIPPER(builtin, clp.Params()).solve_many(probs), first, "built-in batch")
    b = clp.BatchCLIPPER(builtin, clp.Params())
    for method in (clp.MCMethod.KCORE, clp.MCMethod.HEU):
        mp = _mc(clp, method)
        got = c.max_clique_many(probs, mp)
        assert c.info()[0] < len(probs)
        _same_cliques(b.max_clique_many(probs, mp), got, "max clique %s" % method)


# ---- 4. compile and cache -----------------------------------------------------------------------------------------
def test_broken_source_then_valid_batch(clp):
    probs = _problems((50, 300, 129), 60)
    broken = clp.invariants.CudaInvariant(EUCLID_SRC.replace("return 0.0;", "return 0.0", 1), (0.015, 0.05, 0.0))
    c = clp.BatchCLIPPER(broken, clp.Params())
    for call in (lambda: c.solve_many(probs), lambda: c.max_clique_many(probs, _mc(clp, clp.MCMethod.HEU))):
        with pytest.raises(clp.ClipperError) as e:
            call()
        assert e.value.code == 1 and "invariant.cu(" in str(e.value), str(e.value)
    good = clp.invariants.CudaInvariant(EUCLID_SRC, (0.015, 0.05, 0.0))
    c._invariant = good
    _same_solutions(clp.BatchCLIPPER(good, clp.Params()).solve_many(probs), c.solve_many(probs), "after a failed compile")


def test_compile_cache(clp):
    from clipper_b200.api import jit_stats
    src = EUCLID_SRC + "\n// test_gpu_batch_custom.test_compile_cache\n"
    probs = _problems((100, 200), 70)
    a = clp.BatchCLIPPER(clp.invariants.CudaInvariant(src, (0.015, 0.05, 0.0)), clp.Params())
    n0 = jit_stats()[0]
    a.solve_many(probs)
    n1 = jit_stats()[0]
    assert n1 == n0 + 1
    a.solve_many(probs)
    a.max_clique_many(probs, _mc(clp, clp.MCMethod.HEU))
    b = clp.BatchCLIPPER(clp.invariants.CudaInvariant(src, (0.03, 0.05, 0.0)), clp.Params())
    b.solve_many(probs)
    assert jit_stats()[0] == n1
    b.solve_many(_problems((100, 200), 70, d=2))   # a new d
    assert jit_stats()[0] == n1 + 1
    b.solve_many(_problems((100,), 71, d=2))
    assert jit_stats()[0] == n1 + 1


# ---- 5. errors ----------------------------------------------------------------------------------------------------
def test_errors_keep_the_handle_usable(clp):
    probs = _problems((50, 300), 80)
    inv = clp.invariants.CudaInvariant(EUCLID_SRC, (0.015, 0.05, 0.0))
    ref = clp.BatchCLIPPER(inv, clp.Params()).solve_many(probs)
    c = clp.BatchCLIPPER(inv, clp.Params())

    def usable(what):
        _same_solutions(ref, c.solve_many(probs), what)

    c._params = _params(clp, 1e-4, clp.Rounding.DSD)
    with pytest.raises(clp.ClipperError) as e:
        c.solve_many(probs)
    assert e.value.code == 4
    c._params = clp.Params()
    usable("after DSD")

    c._invariant = clp.invariants.CudaInvariant(EUCLID_SRC, (0.015, 0.05, 0.0) + (1.0,) * 14)
    for call in (lambda: c.solve_many(probs), lambda: c.max_clique_many(probs, _mc(clp, clp.MCMethod.HEU))):
        with pytest.raises(clp.ClipperError) as e:
            call()
        assert e.value.code == 1
    c._invariant = inv
    usable("after 17 parameters")

    D1 = np.asfortranarray(np.random.default_rng(1).random((3, 4097)))
    big = dict(D1=D1, D2=D1.copy(), A=np.asfortranarray(np.stack([np.arange(4097)] * 2, 1).astype(np.int32)),
               u0=np.ones(4097))
    with pytest.raises(clp.ClipperError) as e:
        c.solve_many(probs + [big])
    assert e.value.code == 1
    usable("after m = 4097")

    bad = dict(probs[1])
    bad["A"] = probs[1]["A"].copy(order="F")
    bad["A"][7, 1] = probs[1]["D2"].shape[1]
    for call in (lambda: c.solve_many([probs[0], bad]), lambda: c.max_clique_many([probs[0], bad], _mc(clp, clp.MCMethod.KCORE))):
        with pytest.raises(clp.ClipperError) as e:
            call()
        assert e.value.code == 1 and "out of range" in str(e.value)
    usable("after an association out of range")

    mixed = [probs[0], _problems((50,), 82, d=2)[0]]
    with pytest.raises(ValueError):
        c.solve_many(mixed)
    usable("after mixed d")


# ---- 6. parameters ------------------------------------------------------------------------------------------------
def test_parameter_sets(clp):
    probs = _problems((129, 500, 1024), 90) + _problems((333,), 95)
    for sigma, epsilon, mindist in ((0.02, 0.04, 0.0), (0.05, 0.1, 0.01)):
        builtin, restated = _euclid(clp, sigma, epsilon, mindist)
        b, c = clp.BatchCLIPPER(builtin, clp.Params()), clp.BatchCLIPPER(restated, clp.Params())
        what = "sigma %g epsilon %g mindist %g" % (sigma, epsilon, mindist)
        _same_solutions(b.solve_many(probs), c.solve_many(probs), what)
        assert b.info()[2] == c.info()[2], what
