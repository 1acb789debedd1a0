"""Putative associations for a batch of cloud pairs (clp_batch_correspondences(_dev),
utils.distance_based_correspondences_many(_dev), utils::distanceBasedCorrespondencesBatch): every problem's m and rows
against the numpy restatement in tests/knn_oracle.py and against a single distance_based_correspondences_dev call on
the same problem, bit for bit.  Run with  pytest -m gpu  on an H100.

  mixed sizes (0 to above 4097, the 128-query and slice edges) in one batch; d from 1 to the cap and knn from 1 to the
  cap; radius 0, finite, inf and NaN with and without 1-to-1; exact ties and NaN coordinates; NaN and garbage padding;
  expanded and transposed clouds; a batch that slices against one that does not; 4096 tiny problems; repeated calls; a
  caller's stream and torch's default stream; every error code with the batch usable afterwards; host against device
  calls; the chain into BatchCLIPPER.solve_many_dev against the host chain; the C++ shell and the clipperpy module
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


def _cloud(rng, d, n, ties=False):
    if ties:  # small integers: many exactly equal squared distances, within and across candidate slices
        return np.asfortranarray(rng.integers(0, 3, (d, n)).astype(np.float64))
    return np.asfortranarray(rng.standard_normal((d, n)))


def _pad(clouds, fill=np.nan, extra=3):
    """(B, d, n_max + extra) float64 CUDA tensor of the clouds, the padding set to fill"""
    import torch
    d = clouds[0].shape[0]
    nmax = max(X.shape[1] for X in clouds) + extra
    T = np.full((len(clouds), d, nmax), fill)
    for p, X in enumerate(clouds):
        T[p, :, :X.shape[1]] = X
    return torch.from_numpy(T).cuda()


def _rows(A, m):
    """the rows of every problem as numpy (m[p], 2) int32 arrays"""
    H = A.cpu().numpy()
    return [H[p, :mp] for p, mp in enumerate(m)]


def _run(clp, P1, P2, knn, r, one, fill=np.nan):
    import torch
    T1, T2 = _pad(P1, fill), _pad(P2, fill)
    A, m = clp.utils.distance_based_correspondences_many_dev(T1, T2, knn, r, one, n1=[X.shape[1] for X in P1],
                                                             n2=[X.shape[1] for X in P2])
    cap = max(X.shape[1] * min(knn, Y.shape[1]) for X, Y in zip(P1, P2))
    assert A.dtype == torch.int32 and A.is_cuda and A.shape == (len(P1), cap, 2) and A.stride() == (2 * cap, 1, cap)
    return _rows(A, m), m


def _check(clp, P1, P2, knn, r, one, single=True, fill=np.nan):
    """the batched device call against the oracle and (single=True) against one single device call per problem"""
    import torch
    got, m = _run(clp, P1, P2, knn, r, one, fill)
    for p, (X, Y) in enumerate(zip(P1, P2)):
        want = ko.correspondences(X, Y, knn, r, one)
        assert m[p] == want.shape[0], (p, X.shape, Y.shape, m[p], want.shape)
        assert np.array_equal(got[p], want), (p, X.shape, Y.shape)
        if single:
            s = clp.utils.distance_based_correspondences_dev(torch.from_numpy(X).cuda(), torch.from_numpy(Y).cuda(), knn,
                                                             r, one)
            assert np.array_equal(s.cpu().numpy(), got[p]), p
    return got, m


def _nsplit(n1s, n2s, knn):
    """the candidate slices the library cuts for a batch (clp_capi.cu batch_correspondences): enough CTAs for every SM
    four times over, each slice at least 1024 candidates; problems without rows take no part"""
    import torch
    live = [(a, b) for a, b in zip(n1s, n2s) if a * min(knn, b) > 0]
    ctas = sum((a + 127) // 128 for a, _ in live)
    want = (4 * torch.cuda.get_device_properties(0).multi_processor_count + ctas - 1) // ctas
    return max(1, min(want, (max(b for _, b in live) + 1023) // 1024, 1024))


EDGE = [0, 1, 31, 32, 33, 127, 128, 129, 1000, 1023, 1024, 1025, 4097, 5000]


@pytest.mark.parametrize("d", [3, 8])
@pytest.mark.parametrize("one", [False, True])
def test_mixed_sizes(clp, d, one):
    rng = np.random.default_rng(10 + d + one)
    n1s = [1, 0, 129, 33, 4097, 128, 5, 0, 1000, 127, 1] + list(rng.choice(EDGE, 5))
    n2s = [1, 7, 0, 1025, 5000, 1024, 4097, 0, 1023, 129, 4097] + list(rng.choice(EDGE, 5))
    P1 = [_cloud(rng, d, n) for n in n1s]
    P2 = [_cloud(rng, d, n) for n in n2s]
    assert _nsplit(n1s, n2s, 5) > 1   # the batch slices its candidates
    for knn in (1, 5):
        for r in (np.inf, 1.0 if d == 3 else 3.0):
            got, m = _check(clp, P1, P2, knn, r, one, single=(knn == 5))
            assert m[1] == m[2] == m[7] == 0


@pytest.mark.parametrize("d", [1, 2, 3, 8, 33, DMAX])
@pytest.mark.parametrize("knn", [1, 2, 5, KMAX])
def test_dims_and_k(clp, d, knn):
    rng = np.random.default_rng(7 * d + knn)
    sizes = [(129, 1000), (1, 3), (40, 1), (300, 2100), (0, 5)]
    P1 = [_cloud(rng, d, a) for a, _ in sizes]
    P2 = [_cloud(rng, d, b) for _, b in sizes]
    _, sd = ko.neighbours(P1[0], P2[0], knn)
    for r in (np.inf, float(np.sqrt(np.nanmedian(sd)))):
        for one in (False, True):
            _check(clp, P1, P2, knn, r, one, single=(r == np.inf))


def test_radius_and_special_values(clp):
    rng = np.random.default_rng(11)
    P1 = [_cloud(rng, 3, n) for n in (300, 50, 1, 200)]
    P2 = [_cloud(rng, 3, n) for n in (500, 60, 9, 2000)]
    P1[0][1, 5] = np.nan
    P2[0][0, 7] = np.nan
    P2[0][2, 9] = np.inf
    P1[3][0, 10] = -np.inf
    P2[3][:, 100:140] = np.nan     # a run of NaN candidates inside a slice
    for knn in (1, 3, KMAX):
        for r in (0.0, 0.5, np.inf, np.nan):
            for one in (False, True):
                _check(clp, P1, P2, knn, r, one, single=(knn == 3))


@pytest.mark.parametrize("d", [1, 3, 8])
def test_exact_ties(clp, d):
    rng = np.random.default_rng(d)
    sizes = [(1, 4097), (129, 4097), (1000, 1000), (4097, 33), (2, 2)]
    P1 = [_cloud(rng, d, a, ties=True) for a, _ in sizes]
    P2 = [_cloud(rng, d, b, ties=True) for _, b in sizes]
    P2[4][:] = 1.0                 # duplicates of one candidate
    for knn in (1, 5, KMAX):
        for one in (False, True):
            _check(clp, P1, P2, knn, np.inf, one, single=False)
            _check(clp, P1, P2, knn, 1.0, one, single=(knn == 5))


def test_padding_changes_nothing(clp):
    rng = np.random.default_rng(3)
    P1 = [_cloud(rng, 3, n) for n in (100, 7, 0, 1500)]
    P2 = [_cloud(rng, 3, n) for n in (80, 2000, 4, 9)]
    for one in (False, True):
        base, m = _run(clp, P1, P2, 4, 0.8, one, fill=np.nan)
        for fill in (0.0, -np.inf, 1e300, -1e-300):   # points that would be neighbours if they were read
            got, m2 = _run(clp, P1, P2, 4, 0.8, one, fill=fill)
            assert m2 == m and all(np.array_equal(a, b) for a, b in zip(got, base))


def test_expanded_and_transposed_clouds(clp):
    import torch
    rng = np.random.default_rng(4)
    model = _cloud(rng, 3, 700)
    scans = [np.asfortranarray(model + 0.01 * rng.standard_normal(model.shape)) for _ in range(6)]
    for one in (False, True):
        want = [ko.correspondences(model, S, 2, 0.05, one) for S in scans]
        T1 = torch.from_numpy(model).cuda()[None].expand(6, 3, 700)       # one model for every scan: batch stride 0
        assert T1.stride()[0] == 0
        T2 = torch.from_numpy(np.stack([S.T for S in scans])).cuda().transpose(1, 2)   # (B, n, d) seen as (B, d, n)
        assert T2.stride() == (2100, 1, 3)
        A, m = clp.utils.distance_based_correspondences_many_dev(T1, T2, 2, 0.05, one)
        assert all(np.array_equal(a, w) for a, w in zip(_rows(A, m), want))
        # scans against the model, the batch dimension last in memory
        T3 = torch.from_numpy(np.ascontiguousarray(np.stack(scans).transpose(1, 2, 0))).cuda().permute(2, 0, 1)
        A, m = clp.utils.distance_based_correspondences_many_dev(T3, T1, 2, 0.05, one)
        assert all(np.array_equal(a, ko.correspondences(S, model, 2, 0.05, one)) for a, S in zip(_rows(A, m), scans))


def test_slicing_does_not_change_a_result(clp):
    """the same problems in a batch that slices its candidates and in one whose queries fill the device alone"""
    rng = np.random.default_rng(6)
    P1 = [_cloud(rng, 3, n, ties=True) for n in (1, 64, 129)]
    P2 = [_cloud(rng, 3, n, ties=True) for n in (100003, 20000, 4097)]
    F1 = [_cloud(rng, 3, 2000) for _ in range(40)]
    F2 = [_cloud(rng, 3, 300) for _ in range(40)]
    assert _nsplit([1, 64, 129], [100003, 20000, 4097], KMAX) > 1
    assert _nsplit([1, 64, 129] + [2000] * 40, [100003, 20000, 4097] + [300] * 40, KMAX) == 1
    for knn in (1, 7, KMAX):
        for one in (False, True):
            alone, m1 = _run(clp, P1, P2, knn, np.inf, one)
            mixed, m2 = _run(clp, F1[:20] + P1 + F1[20:], F2[:20] + P2 + F2[20:], knn, np.inf, one)
            assert m2[20:23] == m1 and all(np.array_equal(a, b) for a, b in zip(mixed[20:23], alone))
            for p in range(3):
                assert np.array_equal(alone[p], ko.correspondences(P1[p], P2[p], knn, np.inf, one))


def test_many_tiny_problems(clp):
    import torch
    rng = np.random.default_rng(8)
    B = 4096
    n1s, n2s = rng.integers(0, 9, B), rng.integers(0, 9, B)
    P1 = [_cloud(rng, 3, n, ties=True) for n in n1s]
    P2 = [_cloud(rng, 3, n, ties=True) for n in n2s]
    for one in (False, True):
        got, m = _run(clp, P1, P2, 2, 1.5, one)
        for p in range(B):
            assert np.array_equal(got[p], ko.correspondences(P1[p], P2[p], 2, 1.5, one)), p
        for p in range(0, B, 97):
            s = clp.utils.distance_based_correspondences_dev(torch.from_numpy(P1[p]).cuda(), torch.from_numpy(P2[p]).cuda(),
                                                             2, 1.5, one)
            assert np.array_equal(s.cpu().numpy(), got[p])


def test_repeated_calls_and_host_call(clp):
    rng = np.random.default_rng(9)
    for d, knn in ((3, 5), (33, KMAX)):
        P1 = [_cloud(rng, d, n) for n in (5000, 0, 700, 3)]
        P2 = [_cloud(rng, d, n) for n in (7000, 10, 2000, 0)]
        for one in (False, True):
            first, m = _run(clp, P1, P2, knn, np.inf, one)
            again, m2 = _run(clp, P1, P2, knn, np.inf, one)
            assert m2 == m and all(np.array_equal(a, b) for a, b in zip(first, again))
            host = clp.utils.distance_based_correspondences_many(P1, P2, knn, np.inf, one)
            assert [h.shape[0] for h in host] == m
            assert all(h.dtype == np.int32 and np.array_equal(h, a) for h, a in zip(host, first))
            assert all(np.array_equal(h, clp.utils.distance_based_correspondences(X, Y, knn, np.inf, one))
                       for h, X, Y in zip(host, P1, P2))


def test_caller_stream(clp):
    import torch
    rng = np.random.default_rng(77)
    P1 = [_cloud(rng, 3, n) for n in (4000, 300)]
    P2 = [_cloud(rng, 3, n) for n in (6000, 900)]
    want = [ko.correspondences(X, Y, 3, np.inf, False) for X, Y in zip(P1, P2)]
    T1, T2 = _pad(P1), _pad(P2)
    n1, n2 = [4000, 300], [6000, 900]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        X = torch.zeros_like(T1)
        torch.cuda._sleep(50_000_000)   # the copy below lands long after the call is made
        X.copy_(T1)
        A, m = clp.utils.distance_based_correspondences_many_dev(X, T2, 3, np.inf, False, n1=n1, n2=n2)
    assert all(np.array_equal(a, w) for a, w in zip(_rows(A, m), want))


def test_default_stream_orders_after_torch(clp):
    """on torch's default stream, clouds written on the device just before the call are read after they are written"""
    import torch
    assert torch.cuda.current_stream().cuda_stream == 0
    g = torch.Generator(device="cuda").manual_seed(4)
    base1 = torch.randn(3, 3, 4000, dtype=torch.float64, device="cuda", generator=g)
    base2 = torch.randn(3, 3, 6000, dtype=torch.float64, device="cuda", generator=g)
    want = {one: [ko.correspondences(base1[p].cpu().numpy(), base2[p].cpu().numpy(), 3, 0.2, one) for p in range(3)]
            for one in (False, True)}
    for one in (False, True, False):
        torch.cuda._sleep(50_000_000)   # the products below land long after the call is made
        X1, X2 = base1 * 1.0, base2 * 1.0
        A, m = clp.utils.distance_based_correspondences_many_dev(X1, X2, 3, 0.2, one)
        assert all(np.array_equal(a, w) for a, w in zip(_rows(A, m), want[one]))


def test_errors_leave_the_batch_usable(clp):
    """every error code, the first failing problem named, m all zero; then the same batch generates and solves"""
    from clipper_b200 import _capi
    lib = _capi.load()
    ip = clp.invariants.EuclideanDistanceParams()
    bc = clp.BatchCLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params())
    b = bc._b
    rng = np.random.default_rng(12)
    P = [_cloud(rng, 3, 50) for _ in range(3)]
    prob = [dict(D1=P[k], D2=P[k], A=np.asfortranarray(np.stack([np.arange(50), np.arange(50)], 1).astype(np.int32)),
                 u0=np.full(50, 0.5)) for k in range(3)]
    before = [(s.nodes, s.score, s.ifinal) for s in bc.solve_many(prob)]
    vp, i64 = C.c_void_p, C.c_int64
    big = np.zeros((DMAX + 1) * 50)
    outs = [np.zeros(2 * 50 * KMAX, np.int32) for _ in range(3)]
    m = (i64 * 3)()

    def call(nprob=3, d=3, n1=(50, 50, 50), n2=(50, 50, 50), knn=2, cap=100, mp=True, D1=True, Aout=True, last=None):
        m[:] = [7, 7, 7]
        rc = lib.clp_batch_correspondences(
            b, nprob, d, (vp * 3)(*[big.ctypes.data] * 3) if D1 else None, (i64 * 3)(*n1),
            (vp * 3)(*[big.ctypes.data] * 3), (i64 * 3)(*n2), knn, 1.0, 0,
            (vp * 3)(*[o.ctypes.data for o in outs]) if Aout else None, cap, m if mp else None)
        if mp and nprob >= 1:
            assert list(m) == [0, 0, 0] or rc == 0
        return rc

    def err():
        return lib.clp_batch_last_error(b).decode()

    assert call(mp=False) == 1
    assert call(nprob=0) == 1
    assert call(D1=False) == 1 and call(Aout=False) == 1
    assert call(knn=0) == 1 and call(d=0) == 1
    assert call(n2=(50, -1, 50)) == 1 and "problem 1" in err()
    assert call(knn=KMAX + 1, cap=50 * KMAX) == 4 and "CLP_KNN_MAX_K" in err()
    assert call(d=DMAX + 1) == 4 and "CLP_KNN_MAX_D" in err()
    assert call(n1=(50, 50, 2 ** 31 - 1), cap=2 ** 32) == 4 and "problem 2" in err()
    assert call(n1=(50, 51, 50), cap=100) == 1 and "problem 1" in err()
    assert call(knn=-1, d=DMAX + 1) == 1               # the checks come in their order
    assert call(knn=KMAX + 1, cap=0) == 4
    # scratch far beyond the device's memory: refused on the host, before anything is read
    assert call(d=DMAX, n1=(50, 2 ** 31 - 2, 50), n2=(50, 1, 50), knn=1, cap=2 ** 31) == 3 and "problem" not in err()
    assert "free device memory" in err()
    # the device call's checks
    sd = (i64 * 3)(150, 1, 3)
    bad = (i64 * 3)(150, 0, 3)
    dev = lambda s1=sd, s2=sd, sa=sd, cap=100: lib.clp_batch_correspondences_dev(
        b, 3, 3, 16, s1, (i64 * 3)(50, 50, 50), 16, s2, (i64 * 3)(50, 50, 50), 2, 1.0, 0, 16, sa, cap, m)
    assert dev(s1=bad) == 1 and dev(sa=bad) == 1 and dev(cap=99) == 1
    assert dev(s2=(i64 * 3)(-1, 1, 3)) == 1
    # the batch still works: a call that succeeds, then the solve it held before
    assert call() == 0 and all(mk >= 50 for mk in m)
    after = [(s.nodes, s.score, s.ifinal) for s in bc.solve_many(prob)]
    assert after == before


def test_device_chain_matches_host_chain(clp):
    """bunny subsets against noisy copies with outliers: batched kNN -> solve_many_dev, empty problems dropped, against
    solve_many on host associations from per-problem distance_based_correspondences"""
    import torch
    from clipper_b200 import datagen
    cloud = datagen.make_cloud(9992)
    rng = np.random.default_rng(21)
    beta = 0.0554
    P1, P2 = [], []
    for p in range(12):
        n = int(rng.integers(300, 1200))
        X = np.asfortranarray(cloud[:, rng.choice(9992, n, replace=False)])
        Y = np.asfortranarray(X + datagen.bounded_normal_noise(rng, n, 0.01, beta).T)
        Y[:, :n // 5] = rng.random((3, n // 5))                 # outliers
        if p in (3, 8):
            Y = Y + 10.0                                         # nothing within the radius: m = 0
        P1.append(X); P2.append(Y)
    T1, T2 = _pad(P1), _pad(P2)
    n1, n2 = [X.shape[1] for X in P1], [Y.shape[1] for Y in P2]
    A, m = clp.utils.distance_based_correspondences_many_dev(T1, T2, 1, beta, True, n1=n1, n2=n2)
    assert m[3] == m[8] == 0 and all(m[p] > 100 for p in range(12) if p not in (3, 8))
    keep = [p for p in range(12) if m[p] > 0]                    # m = 0 would mean all-to-all to the solve
    idx = torch.tensor(keep, device=A.device)
    ip = clp.invariants.EuclideanDistanceParams()
    ip.sigma, ip.epsilon = 0.01, 0.02
    mk = [m[p] for p in keep]
    u0 = torch.from_numpy(np.random.default_rng(3).random((len(keep), max(mk)))).cuda()
    dev = clp.BatchCLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params()).solve_many_dev(
        T1[idx], T2[idx], A[idx], u0, n1=[n1[p] for p in keep], n2=[n2[p] for p in keep], m=mk)
    probs = []
    for k, p in enumerate(keep):
        Ah = clp.utils.distance_based_correspondences(P1[p], P2[p], 1, beta, True)
        assert np.array_equal(Ah, A[p, :m[p]].cpu().numpy())
        probs.append(dict(D1=P1[p], D2=P2[p], A=Ah, u0=u0[k, :mk[k]].cpu().numpy()))
    host = clp.BatchCLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params()).solve_many(probs)
    for s, h in zip(dev, host):
        assert s.nodes == h.nodes and s.score == h.score and s.ifinal == h.ifinal
    assert all(len(s.nodes) > 0 for s in dev)


def test_cpp_knn_batch_tests(built):
    out = subprocess.run([os.path.join(ROOT, "clipper_b200", "lib", "knn_batch_tests")], capture_output=True, text=True,
                         timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "3 tests" in out.stdout and "0 failures" in out.stdout


def test_clipperpy_agrees(clp):
    import sys
    lib = os.path.join(ROOT, "clipper_b200", "lib")
    if lib not in sys.path:
        sys.path.insert(0, lib)
    import clipperpy as cp
    rng = np.random.default_rng(5)
    P1 = [_cloud(rng, 3, n) for n in (800, 0, 31)]
    P2 = [_cloud(rng, 3, n) for n in (900, 4, 1000)]
    for knn, r, one in ((1, np.inf, False), (5, 0.3, True), (KMAX, 0.5, False)):
        got = cp.utils.distance_based_correspondences_many(P1, P2, knn, r, one)
        assert len(got) == 3
        for g, X, Y in zip(got, P1, P2):
            assert g.dtype == np.int32 and np.array_equal(g, ko.correspondences(X, Y, knn, r, one))
    assert cp.utils.distance_based_correspondences_many([], [], 1, 1.0, False) == []
