"""The rigid transform of selected associations (clp_*estimate_transform*, utils.estimate_rigid_transform(_many)(_dev),
utils::estimateRigidTransform(Batch)) against the numpy restatement in tests/transform_oracle.py, and bit for bit
between its entries.  Run with  pytest -m gpu  on an H100.

Tolerances, where the status is OK and gap / sv[0] >= 1e-6 (u = 2^-52):
  T     max |T - T_oracle| <= 64 u sv[0] / gap (1 + |mu_a|)     (R's sensitivity, carried into t by mu_a)
  sv    within 64 u sv[0]
  rmse  within 1e-12 relative, plus 64 u (1 + |mu_a| + |mu_b|): centred coordinates carry a rounding of u |mu| each,
        which is all there is of a noise-free residual
and where it is DEGENERATE: R orthonormal to 1e-14 with det within 1e-14 of +1, and rmse no worse than the oracle's by
more than 1e-10 relative plus 1e-14 of the data's scale.  Statuses are compared away from the 1e-12 threshold only.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import transform_oracle as to

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -52
KS = (0, 1, 2, 3, 31, 32, 33, 127, 128, 129, 4096, 100000)


@pytest.fixture(scope="module")
def clp(built):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import clipper_b200 as clipperpy
    return clipperpy


def _problem(rng, d, k, kind="noise", offset=0.0, noise=0.0):
    """clouds D1 (d, k + 3), D2 (d, k + 5) and A (k, 2) pairing a random k of them, the pairs related by a random
    rotation; kind: noise, reflect (D2 mirrored), coplanar, collinear, identical, nonfinite (a NaN in a used pair) or
    unused_nan (a NaN in a point no row names)"""
    n1, n2 = k + 3, k + 5
    D1 = rng.standard_normal((d, n1)) + offset
    if kind == "coplanar" and d == 3:
        D1[2] = offset
    if kind == "collinear":
        D1 = np.outer(rng.standard_normal(d), rng.standard_normal(n1)) + offset
    if kind == "identical":
        D1[:] = rng.standard_normal((d, 1)) + offset
    R0 = to.rotation(d, rng)
    if kind == "reflect":
        R0[:, 0] = -R0[:, 0]
    i1, i2 = rng.permutation(n1)[:k], rng.permutation(n2)[:k]
    D2 = rng.standard_normal((d, n2)) + offset
    D2[:, i2] = R0 @ D1[:, i1] + rng.standard_normal(d)[:, None] * 3 + noise * rng.standard_normal((d, k))
    if kind == "nonfinite" and k > 0:
        D1[d - 1, i1[k // 2]] = np.nan
    if kind == "unused_nan":
        D1[0, [j for j in range(n1) if j not in set(i1.tolist())][0]] = np.nan
    A = np.ascontiguousarray(np.stack([i1, i2], 1).astype(np.int32))
    return np.asfortranarray(D1), np.asfortranarray(D2), A


def _check(T, info, o, d, scale=1.0):
    """one result (T row-major, TransformInfo) against the oracle's dict o, within the module's tolerances"""
    T = np.asarray(T)
    assert info.k == o["k"]
    assert np.array_equal(T[d], np.r_[np.zeros(d), 1.0])
    if o["status"] in (to.EMPTY, to.NONFINITE):
        assert info.status == o["status"]
        if o["status"] == to.EMPTY:
            assert np.array_equal(T, np.eye(d + 1)) and info.rmse == 0.0
        else:
            assert np.isnan(T[:d]).all() and np.isnan(info.rmse)
        return
    sv0 = o["sv"][0]
    rel = o["gap"] / sv0 if sv0 > 0 else 0.0
    if not 1e-14 <= rel <= 1e-10:
        assert info.status == o["status"], (info, o["status"], rel)
    if info.status == to.OK and rel >= 1e-6:
        bound = 64 * U * sv0 / o["gap"] * (1 + np.linalg.norm(o["mu_a"]))
        assert np.abs(T - o["T"]).max() <= bound, (np.abs(T - o["T"]).max(), bound)
        assert np.abs(info.sv - o["sv"]).max() <= 64 * U * sv0
        mu_b = o["t"] + o["R"] @ o["mu_a"]
        floor = 64 * U * (1 + np.linalg.norm(o["mu_a"]) + np.linalg.norm(mu_b))
        assert abs(info.rmse - o["rmse"]) <= 1e-12 * o["rmse"] + floor, (info.rmse, o["rmse"])
    elif info.status == to.DEGENERATE:
        R = T[:d, :d]
        assert np.abs(R @ R.T - np.eye(d)).max() <= 1e-14
        assert abs(np.linalg.det(R) - 1) <= 1e-14
        assert info.rmse <= o["rmse"] * (1 + 1e-10) + 1e-14 * scale


def _oracle(D1, D2, A, rows=None):
    """the oracle as the utils read their arguments: an A without rows and no rows is no pairs"""
    return to.estimate(D1, D2, A, [] if (A is not None and len(A) == 0 and rows is None) else rows)


def _tensors(D1, D2, A):
    import torch
    return (torch.from_numpy(np.ascontiguousarray(D1)).cuda(), torch.from_numpy(np.ascontiguousarray(D2)).cuda(),
            torch.from_numpy(A).cuda() if A is not None else None)


@pytest.mark.parametrize("d", [2, 3])
def test_families_against_oracle(clp, d):
    rng = np.random.default_rng(100 + d)
    u = clp.utils
    for k in KS:
        for offset in (0.0, 1e3):
            for noise in (0.0, 1e-3, 0.1):
                D1, D2, A = _problem(rng, d, k, "noise", offset, noise)
                T, info = u.estimate_rigid_transform(D1, D2, A)
                _check(T, info, _oracle(D1, D2, A), d, 1 + offset)
    for kind in ("reflect", "coplanar", "collinear", "identical", "nonfinite", "unused_nan"):
        for k in (1, 2, 3, 33, 4096):
            for offset in (0.0, 1e3):
                D1, D2, A = _problem(rng, d, k, kind, offset, 0.01)
                T, info = u.estimate_rigid_transform(D1, D2, A)
                _check(T, info, _oracle(D1, D2, A), d, 1 + offset)
                if kind == "collinear" and d == 3 and k >= 3:
                    assert info.status == to.DEGENERATE
                if kind == "coplanar" and k >= 3 and d == 3:
                    assert info.status == to.OK


def test_rows_and_all_to_all(clp):
    rng = np.random.default_rng(7)
    u = clp.utils
    for d in (2, 3):
        D1, D2, A = _problem(rng, d, 500, "noise", 5.0, 0.05)
        T0, i0 = u.estimate_rigid_transform(D1, D2, A)
        T1, i1 = u.estimate_rigid_transform(D1, D2, A, rows=np.arange(500))
        assert np.array_equal(T0, T1) and i0.rmse == i1.rmse
        rows = rng.integers(0, 500, 300)   # duplicates: each listing counts
        T2, i2 = u.estimate_rigid_transform(D1, D2, A, rows=rows)
        _check(T2, i2, to.estimate(D1, D2, A, rows), d)
        # all-to-all: row r is (r // n2, r % n2), the same pairs as the explicit rows of A
        n2 = D2.shape[1]
        a2a = [int(a) * n2 + int(b) for a, b in A[rows]]
        T3, i3 = u.estimate_rigid_transform(D1, D2, None, rows=a2a)
        assert np.array_equal(T2, T3) and i2.rmse == i3.rmse
        # every row of all-to-all: the pairs of clp_create_all_to_all's A, in its order (H vanishes there in exact
        # arithmetic, so only bit equality says something)
        T4, i4 = u.estimate_rigid_transform(D1[:, :7], D2[:, :9], None)
        T4a, i4a = u.estimate_rigid_transform(D1[:, :7], D2[:, :9], np.ascontiguousarray(u.create_all_to_all(7, 9)))
        assert i4.k == i4a.k == 63 and np.array_equal(T4, T4a) and i4.rmse == i4a.rmse
        T5, i5 = u.estimate_rigid_transform(D1, D2, A[:0])
        assert i5.status == to.EMPTY and np.array_equal(T5, np.eye(d + 1))


def test_bit_for_bit_between_entries(clp):
    """batch = single calls, host = device calls, repeated calls, a problem alone = inside a mixed batch"""
    import torch
    u = clp.utils
    rng = np.random.default_rng(11)
    for d in (2, 3):
        probs = [_problem(rng, d, k, kind, off, 0.05) for k, kind, off in
                 ((0, "noise", 0.0), (1, "noise", 1.0), (129, "reflect", 1e3), (3000, "noise", 10.0),
                  (33, "collinear", 0.0), (40, "nonfinite", 0.0), (17, "identical", 2.0))]
        rows = [None, None, np.arange(0, 129, 2), None, None, None, np.array([3, 3, 3, 5])]
        singles = [u.estimate_rigid_transform(D1, D2, A, rows=r) for (D1, D2, A), r in zip(probs, rows)]
        Ts, infos = u.estimate_rigid_transform_many([p[0] for p in probs], [p[1] for p in probs], [p[2] for p in probs],
                                                    rows=rows)
        again = u.estimate_rigid_transform_many([p[0] for p in probs], [p[1] for p in probs], [p[2] for p in probs],
                                                rows=rows)
        for (Ts1, i1), T2, i2, T3, i3 in zip(singles, Ts, infos, again[0], again[1]):
            for X, Y in ((Ts1, T2), (T2, T3)):
                assert np.array_equal(X.view(np.int64), Y.view(np.int64))
            assert i1.status == i2.status == i3.status and i1.k == i2.k
            assert np.array_equal(np.float64(i1.rmse).view(np.int64), np.float64(i2.rmse).view(np.int64))
            assert np.array_equal(i1.sv.view(np.int64), i2.sv.view(np.int64))
        # device calls: single and batched, with padding and NaN in it
        for p, ((D1, D2, A), r) in enumerate(zip(probs, rows)):
            X1, X2, XA = _tensors(D1, D2, A)
            Td, idv = u.estimate_rigid_transform_dev(X1, X2, XA, rows=r)
            assert np.array_equal(Td.cpu().numpy().view(np.int64), singles[p][0].view(np.int64))
            assert idv.status == singles[p][1].status
        n1 = [D1.shape[1] for D1, _, _ in probs]
        n2 = [D2.shape[1] for _, D2, _ in probs]
        m = [A.shape[0] for _, _, A in probs]
        keep = [p for p in range(len(probs)) if m[p] > 0]   # m = 0 would mean all-to-all
        B = len(keep)
        P1 = np.full((B, d, max(n1) + 2), np.nan)
        P2 = np.full((B, d, max(n2) + 2), np.nan)
        PA = np.full((B, max(m) + 1, 2), -7, np.int32)
        for j, p in enumerate(keep):
            P1[j, :, :n1[p]], P2[j, :, :n2[p]], PA[j, :m[p]] = probs[p][0], probs[p][1], probs[p][2]
        Tb, ib = u.estimate_rigid_transform_many_dev(
            torch.from_numpy(P1).cuda(), torch.from_numpy(P2).cuda(), torch.from_numpy(PA).cuda(),
            rows=[rows[p] for p in keep], n1=[n1[p] for p in keep], n2=[n2[p] for p in keep], m=[m[p] for p in keep])
        for j, p in enumerate(keep):
            assert np.array_equal(Tb[j].cpu().numpy().view(np.int64), singles[p][0].view(np.int64))
            assert ib[j].status == singles[p][1].status
            assert np.float64(ib[j].rmse).view(np.int64) == np.float64(singles[p][1].rmse).view(np.int64)
        # problem 3 alone against the same problem inside the mixed batch
        j = keep.index(3)
        Ta, _ = u.estimate_rigid_transform_many_dev(
            torch.from_numpy(P1[j:j + 1]).cuda(), torch.from_numpy(P2[j:j + 1]).cuda(), torch.from_numpy(PA[j:j + 1]).cuda(),
            n1=[n1[3]], n2=[n2[3]], m=[m[3]])
        assert torch.equal(Ta[0], Tb[j])


def test_layouts(clp):
    """padded, strided, expanded (batch stride 0) and 6 x n point-normal tensors sliced to their first 3 rows"""
    import torch
    u = clp.utils
    rng = np.random.default_rng(12)
    D1, D2, A = _problem(rng, 3, 200, "noise", 3.0, 0.02)
    want, _ = u.estimate_rigid_transform(D1, D2, A)
    B = 4
    N1 = torch.from_numpy(np.concatenate([D1, rng.standard_normal((3, D1.shape[1]))], 0)).cuda()  # 6 x n point-normals
    N2 = torch.from_numpy(np.concatenate([D2, rng.standard_normal((3, D2.shape[1]))], 0)).cuda()
    X1 = N1.unsqueeze(0).expand(B, 6, -1)[:, :3]                    # batch stride 0, sliced rows
    big2 = torch.zeros((B, 3, 2 * D2.shape[1]), dtype=torch.float64, device="cuda")
    big2[:, :, ::2] = N2[:3]
    X2 = big2[:, :, ::2]                                             # point stride 2
    At = torch.from_numpy(A).cuda()
    XA = torch.zeros((B, 2, 200), dtype=torch.int32, device="cuda")
    XA[:] = At.t()
    XA = XA.transpose(1, 2)                                          # (B, 200, 2) with strides (400, 1, 200)
    T, infos = u.estimate_rigid_transform_many_dev(X1, X2, XA)
    for p in range(B):
        assert np.array_equal(T[p].cpu().numpy(), want)
    Td, _ = u.estimate_rigid_transform_dev(N1[:3], X2[1], At)
    assert np.array_equal(Td.cpu().numpy(), want)


def test_streams(clp):
    import torch
    u = clp.utils
    rng = np.random.default_rng(13)
    D1, D2, A = _problem(rng, 3, 50000, "noise", 1.0, 0.01)
    want, _ = u.estimate_rigid_transform(D1, D2, A)
    T1, T2, TA = _tensors(D1, D2, A)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        Z1, Z2 = torch.zeros_like(T1), torch.zeros_like(T2)
        Z1.copy_(T1); Z2.copy_(T2)                                   # written on the caller's stream just before
        Td, _ = u.estimate_rigid_transform_dev(Z1, Z2, TA)
        Tb, _ = u.estimate_rigid_transform_many_dev(Z1[None], Z2[None], TA[None])
    s.synchronize()
    assert np.array_equal(Td.cpu().numpy(), want) and np.array_equal(Tb[0].cpu().numpy(), want)
    Y1 = torch.full_like(T1, np.nan)
    Y1.copy_(T1)                                                     # on torch's default stream, just before
    Td2, _ = u.estimate_rigid_transform_dev(Y1, T2, TA)
    Tb2, _ = u.estimate_rigid_transform_many_dev(Y1[None], T2[None], TA[None])
    assert np.array_equal(Td2.cpu().numpy(), want) and np.array_equal(Tb2[0].cpu().numpy(), want)


def test_errors_in_order(clp):
    """every error code in the header's order, the handle and batch usable afterwards and the handle's matrix kept"""
    import ctypes as C
    import torch
    from clipper_b200 import _capi
    lib = _capi.load()
    rng = np.random.default_rng(14)
    D1, D2, A = _problem(rng, 3, 20, "noise", 0.0, 0.01)
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()), clp.Params())
    c.score_pairwise_consistency(D1, D2, A)
    M0 = c.get_affinity_matrix()
    h = c.handle
    info = _capi.ClpTfInfo()
    T = np.zeros(16)
    A_f = np.asfortranarray(A)
    rows = np.arange(20, dtype=np.int32)

    def call(d=3, Ap=A_f, m=20, r=rows, k=20, Tp=T):
        return lib.clp_estimate_transform(h, D1.ctypes.data, d, D1.shape[1], D2.ctypes.data, D2.shape[1],
                                          Ap.ctypes.data if Ap is not None else None, m,
                                          r.ctypes.data if r is not None else None, k, Tp.ctypes.data if Tp is not None
                                          else None, C.byref(info))
    INVALID, UNSUPPORTED, ALLOC = 1, 4, 3
    bad_row = rows.copy(); bad_row[5] = 20
    bad_a = A_f.copy(); bad_a[3, 1] = D2.shape[1]
    assert call(Tp=None) == INVALID
    assert call(d=0) == INVALID
    assert call(k=-1) == INVALID
    assert call(r=bad_row) == INVALID and "row 20" in lib.clp_last_error(h).decode()
    assert call(Ap=bad_a) == INVALID
    assert call(d=4, r=bad_row) == INVALID       # INVALID comes before UNSUPPORTED
    assert call(d=4) == UNSUPPORTED
    assert call() == 0 and info.status == to.OK
    # CLP_ERR_ALLOC: every row of the all-to-all hypothesis over two clouds of 2^20 points is 2^40 pairs
    big = np.zeros((3, 1 << 20))
    rc = lib.clp_estimate_transform(h, big.ctypes.data, 3, big.shape[1], big.ctypes.data, big.shape[1], None, 0, None, 0,
                                    T.ctypes.data, C.byref(info))
    assert rc == ALLOC, lib.clp_last_error(h)
    assert call() == 0 and info.status == to.OK
    assert np.array_equal(c.get_affinity_matrix(), M0)
    # the batch: a device association index out of range names the lowest bad problem
    u = clp.utils
    X1 = torch.from_numpy(np.stack([D1] * 3)).cuda()
    X2 = torch.from_numpy(np.stack([D2] * 3)).cuda()
    XA = torch.from_numpy(np.stack([A] * 3)).cuda()
    XA[2, 4, 0] = -1
    XA[1, 7, 1] = 10 ** 6
    with pytest.raises(clp.ClipperError) as e:
        u.estimate_rigid_transform_many_dev(X1, X2, XA)
    assert e.value.code == INVALID and "problem 1" in str(e.value)
    with pytest.raises(clp.ClipperError) as e:
        u.estimate_rigid_transform_many_dev(X1, X2, XA, rows=[None, np.arange(5), None])
    assert e.value.code == INVALID and "problem 2" in str(e.value)
    T3, _ = u.estimate_rigid_transform_many_dev(X1, X2, XA, rows=[None, np.arange(5), np.arange(3)])
    want, _ = u.estimate_rigid_transform(D1, D2, A)
    assert np.array_equal(T3[0].cpu().numpy(), want)
    with pytest.raises(clp.ClipperError) as e:
        u.estimate_rigid_transform_many(list(X1.cpu().numpy()), list(X2.cpu().numpy()), [A, A, np.ascontiguousarray(XA[2].cpu().numpy())])
    assert e.value.code == INVALID and "problem 2" in str(e.value)
    with pytest.raises(clp.ClipperError) as e:
        u.estimate_rigid_transform_many([np.zeros((4, 3))], [np.zeros((4, 3))], [np.zeros((3, 2), np.int32)])
    assert e.value.code == UNSUPPORTED
    T4, _ = u.estimate_rigid_transform_many([D1], [D2], [A])
    assert np.array_equal(T4[0], want)


def test_bunny_chain(clp):
    """the notebook's registration on the bunny for a batch: B random rotations and translations with noise and outlier
    associations, BatchCLIPPER.solve_many_dev, then estimate_rigid_transform_many_dev on the solutions' nodes"""
    import torch
    from clipper_b200 import datagen
    cloud = datagen.make_cloud(9992)
    rng = np.random.default_rng(31)
    B, n, n_out, sigma, beta = 16, 600, 400, 0.005, 0.015
    P1, P2, As, truth, inl = [], [], [], [], []
    for p in range(B):
        X = cloud[:, rng.choice(9992, n, replace=False)]
        R0 = to.rotation(3, rng)
        t0 = rng.uniform(-5, 5, 3)
        Y = R0 @ X + t0[:, None] + datagen.bounded_normal_noise(rng, n, sigma, beta).T
        m_in = n - n_out
        A = np.stack([np.arange(n), np.arange(n)], 1).astype(np.int32)
        A[m_in:, 1] = rng.integers(0, n, n_out)         # outlier associations
        perm = rng.permutation(n)
        P1.append(np.asfortranarray(X)); P2.append(np.asfortranarray(Y)); As.append(A[perm])
        truth.append((R0, t0)); inl.append(np.sort(np.argsort(perm)[:m_in]))
    ip = clp.invariants.EuclideanDistanceParams()
    ip.sigma, ip.epsilon = 0.015, 0.04      # 2 beta < epsilon: every inlier pair is consistent
    T1 = torch.from_numpy(np.stack(P1)).cuda()
    T2 = torch.from_numpy(np.stack(P2)).cuda()
    TA = torch.from_numpy(np.stack(As)).cuda()
    u0 = torch.from_numpy(rng.random((B, n))).cuda()
    sols = clp.BatchCLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params()).solve_many_dev(T1, T2, TA, u0)
    T, infos = clp.utils.estimate_rigid_transform_many_dev(T1, T2, TA, rows=[s.nodes for s in sols])
    # the ground-truth bound, fixed on the CPU from the oracle on the true inliers: five times its rotation and
    # translation errors, plus 1e-3 (a margin for the few inliers a solve may miss or outliers it may keep)
    for p in range(B):
        o = to.estimate(P1[p], P2[p], As[p], sols[p].nodes)
        _check(T[p].cpu().numpy(), infos[p], o, 3)
        ot = to.estimate(P1[p], P2[p], As[p], inl[p])
        R0, t0 = truth[p]
        eR = np.abs(ot["R"] - R0).max()
        et = np.abs(ot["t"] - t0).max()
        got = T[p].cpu().numpy()
        assert np.abs(got[:3, :3] - R0).max() <= 5 * eR + 1e-3
        assert np.abs(got[:3, 3] - t0).max() <= 5 * et + 1e-3
        assert len(set(sols[p].nodes) & set(inl[p].tolist())) >= 0.9 * (n - n_out)


def test_cpp_transform_tests(built):
    out = subprocess.run([os.path.join(ROOT, "clipper_b200", "lib", "transform_tests")], capture_output=True, text=True,
                         timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "3 tests" in out.stdout and "0 failures" in out.stdout


def test_clipperpy_agrees(clp):
    lib = os.path.join(ROOT, "clipper_b200", "lib")
    if lib not in sys.path:
        sys.path.insert(0, lib)
    import clipperpy as cp
    import fixtures as fx
    model, data = fx.toy_problem()
    A = np.array([[0, 0], [1, 1], [2, 2]], dtype=np.int32)
    T, info = cp.utils.estimate_rigid_transform(model, data, A)
    Tm, im = clp.utils.estimate_rigid_transform(model, data, A)
    assert np.array_equal(T, Tm) and info["status"] == im.status == to.OK and info["k"] == 3
    o = to.estimate(model, data, A)
    assert np.abs(T - o["T"]).max() <= 1e-14
    Te, ie = cp.utils.estimate_rigid_transform(model, data, np.zeros((0, 2), np.int32))
    assert ie["status"] == to.EMPTY and np.array_equal(Te, np.eye(4))
    rng = np.random.default_rng(15)
    probs = [_problem(rng, 3, k, "noise", 1.0, 0.05) for k in (0, 5, 300)]
    Ts, infos = cp.utils.estimate_rigid_transform_many([p[0] for p in probs], [p[1] for p in probs], [p[2] for p in probs])
    for (D1, D2, A), Tp, ip in zip(probs, Ts, infos):
        Tq, iq = clp.utils.estimate_rigid_transform(D1, D2, A)
        assert np.array_equal(Tp, Tq) and ip["status"] == iq.status
