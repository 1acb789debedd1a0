"""Putative associations on the GPU (clp_correspondences, clp_correspondences_dev, utils::distanceBasedCorrespondences)
against the numpy restatement in tests/knn_oracle.py, bit for bit: m and every row of A.  Run with  pytest -m gpu  on an
H100.

  sizes around the tile and slice edges, d from 1 to the cap, knn from 1 to the cap, with and without 1-to-1, on
  Gaussian clouds and on small-integer clouds full of exact ties; the benchmark's bunny call; n1 = n2 = 2e5 against
  scipy's kd-tree; host against device pointers; repeated calls; a caller's stream; every error code; the chain
  clouds -> A -> score -> solve on the device against the host chain; the C++ shell and the clipperpy module
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import knn_oracle as ko

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KMAX, DMAX = 32, 64


@pytest.fixture(scope="module")
def clp(built):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import clipper_b200 as clipperpy
    return clipperpy


def _clouds(d, n1, n2, seed, ties=False):
    rng = np.random.default_rng(seed)
    if ties:  # small integers: many exactly equal squared distances, within and across candidate slices
        return (np.asfortranarray(rng.integers(0, 3, (d, n1)).astype(np.float64)),
                np.asfortranarray(rng.integers(0, 3, (d, n2)).astype(np.float64)))
    return np.asfortranarray(rng.standard_normal((d, n1))), np.asfortranarray(rng.standard_normal((d, n2)))


def _check(clp, D1, D2, knn, radius, one):
    got = clp.utils.distance_based_correspondences(D1, D2, knn, radius, one)
    want = ko.correspondences(D1, D2, knn, radius, one)
    assert got.dtype == np.int32 and got.shape == want.shape, (got.shape, want.shape)
    assert np.array_equal(got, want)
    return got


def _radii(D1, D2, knn):
    """inf, and a radius that keeps about half of the neighbour pairs"""
    _, sd = ko.neighbours(D1, D2, knn)
    med = np.nanmedian(sd) if np.isfinite(sd).any() else 1.0
    return [np.inf, float(np.sqrt(med))]


SIZES = [1, 31, 32, 33, 127, 128, 129, 1000, 4097]


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("one", [False, True])
def test_sizes(clp, n, one):
    for n1, n2, seed in ((n, n, 1), (n, 1000, 2), (33, n, 3)):
        D1, D2 = _clouds(3, n1, n2, 100 * n + seed)
        for knn in (1, 5):
            for r in _radii(D1, D2, knn):
                _check(clp, D1, D2, knn, r, one)


@pytest.mark.parametrize("d", [1, 2, 3, 8, 33, DMAX])
@pytest.mark.parametrize("knn", [1, 2, 5, KMAX])
@pytest.mark.parametrize("one", [False, True])
def test_dims_and_k(clp, d, knn, one):
    D1, D2 = _clouds(d, 129, 1000, 7 * d + knn)
    for r in _radii(D1, D2, knn):
        _check(clp, D1, D2, knn, r, one)


@pytest.mark.parametrize("d", [1, 3, 8])
@pytest.mark.parametrize("shape", [(1, 4097), (129, 4097), (1000, 1000), (4097, 33)])
def test_exact_ties(clp, d, shape):
    D1, D2 = _clouds(d, shape[0], shape[1], d + shape[0], ties=True)
    for knn in (1, 5, KMAX):
        for one in (False, True):
            _check(clp, D1, D2, knn, np.inf, one)
            _check(clp, D1, D2, knn, 1.0, one)


def test_slices_of_one_query(clp):
    # one query against many candidates: the candidate range is cut into slices whose lists are merged
    for n2 in (1025, 20000, 100003):
        D1, D2 = _clouds(3, 1, n2, n2, ties=True)
        for knn in (1, 7, KMAX):
            _check(clp, D1, D2, knn, np.inf, False)


def test_special_values(clp):
    D1, D2 = _clouds(3, 300, 500, 11)
    D1[1, 5] = np.nan
    D2[0, 7] = np.nan
    D2[2, 9] = np.inf
    D1[0, 10] = -np.inf
    for knn in (1, 3, KMAX):
        for r in (0.0, 0.5, np.inf, np.nan, -0.5):
            for one in (False, True):
                _check(clp, D1, D2, knn, r, one)
    # knn > n2: n2 neighbours; duplicates of a candidate: the lower index first
    E2 = np.asfortranarray(np.repeat(_clouds(3, 1, 4, 12)[1], 3, axis=1))
    A = _check(clp, D1[:, 20:40], E2, 20, np.inf, False)
    assert A.shape == (20 * 12, 2)
    # an empty cloud and single points
    assert clp.utils.distance_based_correspondences(D1, np.zeros((3, 0)), 3, np.inf, False).shape == (0, 2)
    assert clp.utils.distance_based_correspondences(np.zeros((3, 0)), D2, 3, np.inf, True).shape == (0, 2)
    _check(clp, D1[:, :1], D2[:, :1], 4, np.inf, True)


def test_bunny_benchmark_call(clp):
    """the reference benchmark's ground-truth call: the bunny against a noisy copy, knn 1, radius = the noise bound"""
    from clipper_b200 import datagen
    D1 = datagen.make_cloud(9992)
    beta = 0.0554
    eta = datagen.bounded_normal_noise(np.random.default_rng(5), 9992, 0.01, beta)
    D2 = np.asfortranarray(D1 + eta.T)
    A = _check(clp, D1, D2, 1, beta, True)
    assert A.shape[0] > 5000 and np.all(np.diff(A[:, 1]) > 0)


def test_large_against_kdtree(clp):
    from scipy.spatial import cKDTree
    n, knn = 200000, 4
    D1, D2 = _clouds(3, n, n, 99)
    A = clp.utils.distance_based_correspondences(D1, D2, knn, np.inf, False)
    dist, idx = cKDTree(D2.T).query(D1.T, k=knn + 1, workers=-1)
    # no near-ties: consecutive distances (the k-th against the (k+1)-th included) apart by far more than rounding
    assert np.all(np.diff(dist, axis=1) > 1e-9 * dist[:, 1:])
    assert A.shape == (n * knn, 2)
    assert np.array_equal(A[:, 0], np.repeat(np.arange(n), knn))
    assert np.array_equal(A[:, 1], idx[:, :knn].reshape(-1))


def test_host_and_device_agree_and_repeat(clp):
    import torch
    for d, n1, n2, knn, one in ((3, 5000, 7000, 5, False), (3, 5000, 7000, 1, True), (33, 700, 2000, KMAX, True)):
        D1, D2 = _clouds(d, n1, n2, n1 + d)
        r = _radii(D1, D2, knn)[1]
        host = clp.utils.distance_based_correspondences(D1, D2, knn, r, one)
        T1, T2 = torch.from_numpy(D1).cuda(), torch.from_numpy(D2).cuda()
        dev = clp.utils.distance_based_correspondences_dev(T1, T2, knn, r, one)
        assert dev.is_cuda and dev.dtype == torch.int32 and dev.stride() == (1, dev.shape[0])
        assert np.array_equal(dev.cpu().numpy(), host)
        again = clp.utils.distance_based_correspondences_dev(T1, T2, knn, r, one)
        assert torch.equal(again, dev)
        assert np.array_equal(clp.utils.distance_based_correspondences(D1, D2, knn, r, one), host)
        # a row-major (d, n) copy of the same clouds (the wrapper copies it on the device) reads the same values
        Tr = torch.from_numpy(np.ascontiguousarray(D1)).cuda()
        assert Tr.stride() == (n1, 1)
        assert torch.equal(clp.utils.distance_based_correspondences_dev(Tr, T2, knn, r, one), dev)


def test_caller_stream(clp):
    import torch
    D1, D2 = _clouds(3, 4000, 6000, 77)
    want = ko.correspondences(D1, D2, 3, np.inf, False)
    T1, T2 = torch.from_numpy(D1).cuda(), torch.from_numpy(D2).cuda()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        X = torch.zeros_like(T1)
        torch.cuda._sleep(50_000_000)   # the copy below lands long after the call is made
        X.copy_(T1)
        got = clp.utils.distance_based_correspondences_dev(X, T2, 3, np.inf, False)
    assert np.array_equal(got.cpu().numpy(), want)


def test_default_stream_orders_after_torch(clp):
    """on torch's default stream, inputs written on the device just before the call are read after they are written"""
    import torch
    assert torch.cuda.current_stream().cuda_stream == 0
    g = torch.Generator(device="cuda").manual_seed(4)
    base1 = torch.randn(3, 4000, dtype=torch.float64, device="cuda", generator=g)   # row-major (d, n): copied
    base2 = torch.randn(3, 6000, dtype=torch.float64, device="cuda", generator=g)
    want = {one: ko.correspondences(base1.cpu().numpy(), base2.cpu().numpy(), 3, 0.2, one) for one in (False, True)}
    for one in (False, True, False):
        torch.cuda._sleep(50_000_000)   # the products below land long after the call is made
        X1, X2 = base1 * 1.0, base2 * 1.0
        got = clp.utils.distance_based_correspondences_dev(X1, X2, 3, 0.2, one)
        assert np.array_equal(got.cpu().numpy(), want[one])


def test_knn_above_the_cap_fails_before_allocating(clp):
    import torch
    from clipper_b200 import _capi
    D1, D2 = _clouds(3, 200000, 200000, 8)
    with pytest.raises(_capi.ClipperError) as e:
        clp.utils.distance_based_correspondences(D1, D2, 10 ** 6, 1.0, False)
    assert e.value.code == 4 and "CLP_KNN_MAX_K" in str(e.value)
    T1, T2 = torch.from_numpy(D1).cuda(), torch.from_numpy(D2).cuda()
    with pytest.raises(_capi.ClipperError) as e:
        clp.utils.distance_based_correspondences_dev(T1, T2, 10 ** 6, 1.0, False)
    assert e.value.code == 4 and "CLP_KNN_MAX_K" in str(e.value)


def test_errors_leave_the_matrix(clp):
    from clipper_b200 import _capi
    lib = _capi.load()
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()), clp.Params())
    P = np.asfortranarray(np.random.default_rng(1).standard_normal((3, 50)))
    c.score_pairwise_consistency(P, P, np.asfortranarray(np.stack([np.arange(50), np.arange(50)], 1).astype(np.int32)))
    M0 = c.get_affinity_matrix()
    h = c.handle
    dp = C.POINTER(C.c_double)
    D = np.asfortranarray(np.zeros((DMAX + 1, 10)))
    A = np.zeros(2 * 10 * KMAX, dtype=np.int32)
    Ap = A.ctypes.data_as(C.POINTER(C.c_int32))
    m = C.c_int64(-1)

    def call(d=3, n1=10, n2=10, knn=2, cap=20, mp=True):
        return lib.clp_correspondences(h, D.ctypes.data_as(dp), d, n1, D.ctypes.data_as(dp), n2, knn, 1.0, 0, Ap, cap,
                                       C.byref(m) if mp else None)

    assert call(knn=0) == 1 and call(knn=-3) == 1
    assert call(d=0) == 1
    assert call(n1=-1) == 1
    assert call(cap=19) == 1
    assert call(mp=False) == 1
    assert call(knn=KMAX + 1, cap=10 * KMAX) == 4 and b"CLP_KNN_MAX_K" in lib.clp_last_error(h)
    assert call(d=DMAX + 1) == 4 and b"CLP_KNN_MAX_D" in lib.clp_last_error(h)
    assert call(knn=KMAX, cap=100) == 0 and m.value == 100   # knn > n2 is clamped: capacity n1 * n2
    assert call() == 0 and m.value >= 10
    assert np.array_equal(c.get_affinity_matrix(), M0)
    c.solve(np.full(50, 0.5))
    assert len(c.get_solution().nodes) == 50


def test_device_chain_matches_host_chain(clp):
    import torch
    from clipper_b200 import datagen
    D1 = datagen.make_cloud(9992)
    rng = np.random.default_rng(21)
    eta = datagen.bounded_normal_noise(rng, 9992, 0.01, 0.0554)
    D2 = np.asfortranarray(D1 + eta.T)
    D2[:, :2000] = rng.random((3, 2000))            # outliers
    T1, T2 = torch.from_numpy(D1).cuda(), torch.from_numpy(D2).cuda()
    A_dev = clp.utils.distance_based_correspondences_dev(T1, T2, 1, 0.0554, True)
    assert A_dev.t().is_contiguous()                # scored without a copy
    A = clp.utils.distance_based_correspondences(D1, D2, 1, 0.0554, True)
    assert np.array_equal(A_dev.cpu().numpy(), A)
    ip = clp.invariants.EuclideanDistanceParams()
    ip.sigma, ip.epsilon = 0.01, 0.02
    u0 = np.random.default_rng(3).random(A.shape[0])
    g = clp.CLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params())
    g.score_pairwise_consistency_dev(T1, T2, A_dev)
    g.solve(u0)
    h = clp.CLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params())
    h.score_pairwise_consistency(D1, D2, np.asfortranarray(A))
    h.solve(u0)
    assert np.array_equal(g.get_initial_associations(), A)
    assert sorted(g.get_solution().nodes) == sorted(h.get_solution().nodes)
    assert len(g.get_solution().nodes) > 0


def test_cpp_knn_tests(built):
    out = subprocess.run([os.path.join(ROOT, "clipper_b200", "lib", "knn_tests")], capture_output=True, text=True,
                         timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "4 tests" in out.stdout and "0 failures" in out.stdout


def test_clipperpy_agrees(clp):
    import sys
    lib = os.path.join(ROOT, "clipper_b200", "lib")
    if lib not in sys.path:
        sys.path.insert(0, lib)
    import clipperpy as cp
    D1, D2 = _clouds(3, 800, 900, 5)
    for knn, r, one in ((1, np.inf, False), (5, 0.3, True), (KMAX, 0.5, False)):
        want = ko.correspondences(D1, D2, knn, r, one)
        got = cp.utils.distance_based_correspondences(D1, D2, knn, r, one)
        assert got.dtype == np.int32 and np.array_equal(got, want)
