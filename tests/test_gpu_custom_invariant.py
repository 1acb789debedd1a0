"""CUDA-source invariants (CudaInvariant, clp_score_custom): compiled at run time into the unscreened scoring kernel.

Restatements of the two built-in invariants must give the built-in handles' matrices bit for bit on every
single-problem family of scoring_families (both storages): the built-ins store what their exact fp64 path computes,
and the restatements run the same operations (the same _rn intrinsics, the same libdevice exp and acos, compiled by
NVRTC and nvcc of one toolkit).  An asymmetric invariant pins the argument order (i < j) against the two host custom
paths; the notebook's Custom invariant is checked against the Python host path within its libm differences.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import scoring_families as sf

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "clipper_b200", "lib")
AFFINITY_EPS = (1e-4, 0.0, -1.0)

# EuclideanDistance with the kernel's operation order (point_dist, euclid_score); prm = (sigma, epsilon, mindist)
EUCLID_SRC = r"""
__device__ double clp_invariant(const double* ai, const double* aj, const double* bi, const double* bj, int d,
                                const double* prm) {
  double s1 = 0.0, s2 = 0.0;
  for (int q = 0; q < d; ++q) { const double t = __dsub_rn(ai[q], aj[q]); s1 = __dadd_rn(s1, __dmul_rn(t, t)); }
  for (int q = 0; q < d; ++q) { const double t = __dsub_rn(bi[q], bj[q]); s2 = __dadd_rn(s2, __dmul_rn(t, t)); }
  const double l1 = __dsqrt_rn(s1), l2 = __dsqrt_rn(s2);
  if (prm[2] > 0 && (l1 < prm[2] || l2 < prm[2])) return 0.0;
  const double c = fabs(__dsub_rn(l1, l2));
  if (!(c < prm[1])) return 0.0;
  return exp(__ddiv_rn(__dmul_rn(__dmul_rn(-0.5, c), c), __dmul_rn(prm[0], prm[0])));
}
"""

# PointNormalDistance (unclamped acos); prm = (sigp, epsp, sign, epsn)
PN_SRC = r"""
__device__ double len3(const double* a, const double* b) {
  double s = 0.0;
  for (int q = 0; q < 3; ++q) { const double t = __dsub_rn(a[q], b[q]); s = __dadd_rn(s, __dmul_rn(t, t)); }
  return __dsqrt_rn(s);
}
__device__ double dot3(const double* a, const double* b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a[3], b[3]), __dmul_rn(a[4], b[4])), __dmul_rn(a[5], b[5]));
}
__device__ double clp_invariant(const double* ai, const double* aj, const double* bi, const double* bj, int d,
                                const double* prm) {
  const double l1 = len3(ai, aj), l2 = len3(bi, bj);
  const double alpha1 = acos(dot3(ai, aj)), alpha2 = acos(dot3(bi, bj));
  const double dp = fabs(__dsub_rn(l1, l2)), dn = fabs(__dsub_rn(alpha1, alpha2));
  if (dp < prm[1] && dn < prm[3]) {
    const double sp = exp(__ddiv_rn(__dmul_rn(__dmul_rn(-0.5, dp), dp), __dmul_rn(prm[0], prm[0])));
    const double sn = exp(__ddiv_rn(__dmul_rn(__dmul_rn(-0.5, dn), dn), __dmul_rn(prm[2], prm[2])));
    return __dmul_rn(sp, sn);
  }
  return 0.0;
}
"""

# the Custom invariant of the reference's notebook (examples/python/ex4_bunny.ipynb); prm = (sigma, epsilon)
NOTEBOOK_SRC = r"""
__device__ double clp_invariant(const double* ai, const double* aj, const double* bi, const double* bj, int d,
                                const double* prm) {
  double s1 = 0.0, s2 = 0.0;
  for (int q = 0; q < d; ++q) { s1 += (ai[q] - aj[q]) * (ai[q] - aj[q]); s2 += (bi[q] - bj[q]) * (bi[q] - bj[q]); }
  const double c = fabs(sqrt(s1) - sqrt(s2));
  return c < prm[1] ? exp(-0.5 * c * c / (prm[0] * prm[0])) : 0.0;
}
"""

# exact on small integers, no libm, f(i, j) != f(j, i); prm = (offset,)
ASYM_SRC = r"""
__device__ double clp_invariant(const double* ai, const double* aj, const double* bi, const double* bj, int d,
                                const double* prm) {
  return (ai[0] - 2.0 * aj[0]) + 0.5 * (bi[1] - bj[0]) + prm[0];
}
"""


def _asym(ai, aj, bi, bj, offset):
    return (ai[0] - 2.0 * aj[0]) + 0.5 * (bi[1] - bj[0]) + offset


@pytest.fixture(scope="module")
def clp(built):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import clipper_b200 as clipperpy
    return clipperpy


def _families():
    F = [sf.s1_eps_ties(d) for d in (1, 2, 3, 4, 5)] + [sf.s2_mindist_ties(d) for d in (1, 2, 3, 4)]
    for scale in sf.S3_SCALES:
        F += [sf.s3_screen_band(scale, 2), sf.s3_screen_band(scale, 3), sf.s3_screen_band(scale, 3, "pn")]
    F += [sf.s4_pointnormal_angles(), sf.s7_nonfinite()] + sf.s6_distinctness()
    F += [sf.s8_tiles(m) for m in sf.S8_SIZES] + [sf.s8_tiles(m, "pn") for m in (31, 128, 4097)]
    for ae in AFFINITY_EPS:
        F += [sf.s5_underflow().with_affinityeps(ae), sf.s1_eps_ties(3).with_affinityeps(ae),
              sf.s4_pointnormal_angles().with_affinityeps(ae), sf.s3_screen_band(1e19, 3).with_affinityeps(ae)]
    out, seen = {}, set()
    for f in F:
        if f.name not in seen:
            seen.add(f.name); out[f.name] = f
    return out


FAMILIES = _families()


def _params(clp, ae):
    p = clp.Params()
    p.affinityeps = ae
    return p


def _builtin(clp, fam):
    q = fam.params
    if fam.kind == "euclid":
        ip = clp.invariants.EuclideanDistanceParams()
        ip.sigma, ip.epsilon, ip.mindist = q["sigma"], q["epsilon"], q["mindist"]
        return clp.invariants.EuclideanDistance(ip)
    ip = clp.invariants.PointNormalDistanceParams()
    ip.sigp, ip.epsp, ip.sign, ip.epsn = q["sigp"], q["epsp"], q["sign"], q["epsn"]
    return clp.invariants.PointNormalDistance(ip)


def _restated(clp, fam):
    q = fam.params
    if fam.kind == "euclid":
        return clp.invariants.CudaInvariant(EUCLID_SRC, (q["sigma"], q["epsilon"], q["mindist"]))
    return clp.invariants.CudaInvariant(PN_SRC, (q["sigp"], q["epsp"], q["sign"], q["epsn"]))


def _bits(x):
    return np.ascontiguousarray(x).view(np.int64)


def _same_matrices(a, b, what):
    for get in ("get_affinity_matrix", "get_constraint_matrix"):
        x, y = getattr(a, get)(), getattr(b, get)()
        assert np.array_equal(_bits(x), _bits(y)), "%s: %s differs in %d entries" % (what, get, int((_bits(x) != _bits(y)).sum()))
    assert a.count_nonzeros() == b.count_nonzeros(), what


def _same_solution(s, t, what):
    assert s.u.tobytes() == t.u.tobytes(), what
    assert s.nodes == t.nodes and s.score == t.score, what


# ---- 1. restated built-ins, bit for bit ----------------------------------------------------------------------------------
@pytest.mark.parametrize("storage", [0, 1])
@pytest.mark.parametrize("name", list(FAMILIES))
def test_restated_builtin_bitwise(clp, name, storage):
    fam = FAMILIES[name]
    what = "%s storage %d" % (name, storage)
    b = clp.CLIPPER(_builtin(clp, fam), _params(clp, fam.affinityeps), storage=storage)
    c = clp.CLIPPER(_restated(clp, fam), _params(clp, fam.affinityeps), storage=storage)
    b.score_pairwise_consistency(fam.D1, fam.D2, fam.A)
    c.score_pairwise_consistency(fam.D1, fam.D2, fam.A)
    _same_matrices(b, c, what)
    sf.check_dense(sf.Restated(fam), c.get_affinity_matrix(), c.get_constraint_matrix(), storage == 0, what)
    u0 = np.random.default_rng(5).random(fam.m)
    b.solve(u0)
    c.solve(u0)
    _same_solution(b.get_solution(), c.get_solution(), what)


# ---- 2. sharded handles -------------------------------------------------------------------------------------------------
SHARDED = ("S1_d3_ae-1", "S4_pn_ae-1", "S8_m129_d3", "S5_ae0.0001", "S2_d3")


@pytest.mark.parametrize("storage", [0, 1])
@pytest.mark.parametrize("world", [2, 3])
def test_sharded(clp, world, storage):
    from clipper_b200 import distributed as cd
    for name in SHARDED:
        fam = FAMILIES[name]
        what = "%s world %d storage %d" % (name, world, storage)
        full = clp.CLIPPER(_restated(clp, fam), _params(clp, fam.affinityeps), storage=storage)
        full.score_pairwise_consistency(fam.D1, fam.D2, fam.A)
        Cm = full.get_constraint_matrix()
        groups = []
        for make in (lambda: _restated(clp, fam), lambda: _builtin(clp, fam)):
            g = cd.ShardGroup(make, _params(clp, fam.affinityeps), [0] * world, storage=storage, same_device=True)
            g.score_pairwise_consistency(fam.D1, fam.D2, fam.A)
            groups.append(g)
        for r, sh in enumerate(groups[0].shards):   # each shard holds the rows of the unsharded matrix
            r0, nr = cd.shard_rows(fam.m, r, world)
            up = np.triu(np.ones_like(Cm, dtype=bool), 1)[r0:r0 + nr]
            assert sh.count_nonzeros()[1] == int(np.count_nonzero((Cm[r0:r0 + nr] == 1) & up)), "%s rank %d" % (what, r)
            assert sh.count_nonzeros() == groups[1].shards[r].count_nonzeros(), what
        u0 = np.random.default_rng(7).random(fam.m)
        for mode in (6, 0):   # the sweeps whose persistent kernels shards sharing one GPU can run side by side
            for g in groups:
                for sh in g.shards:
                    sh.set_dense_mode(mode)
            sc, sb = groups[0].solve(u0), groups[1].solve(u0)
            for s in sc[1:] + sb:
                _same_solution(sc[0], s, "%s mode %d" % (what, mode))
        del groups


# ---- 3. argument order --------------------------------------------------------------------------------------------------
def _asym_problem():
    rng = np.random.default_rng(3)
    n = 40
    D1 = rng.integers(-3, 4, (2, n)).astype(np.float64)
    D2 = rng.integers(-3, 4, (2, n)).astype(np.float64)
    A = np.asfortranarray(np.stack([rng.integers(0, n, 150), rng.integers(0, n, 150)], 1).astype(np.int32))
    return D1, D2, A


@pytest.mark.parametrize("ae", [1e-4, 0.0])   # both drop the negative scores: M >= 0 (clp_set_dense's contract)
def test_argument_order_matches_host_paths(clp, ae):
    from clipper_b200 import distributed as cd
    D1, D2, A = _asym_problem()
    offset = 0.25

    class HostAsym(clp.invariants.PairwiseInvariant):
        def __call__(self, ai, aj, bi, bj):
            return _asym(ai, aj, bi, bj, offset)

    host = clp.CLIPPER(HostAsym(), _params(clp, ae), storage=1)
    host.score_pairwise_consistency(D1, D2, A)
    M, Cm = host.get_affinity_matrix(), host.get_constraint_matrix()
    assert np.count_nonzero(np.triu(Cm, 1)) > 100
    dev = clp.CLIPPER(clp.invariants.CudaInvariant(ASYM_SRC, (offset,)), _params(clp, ae), storage=1)
    dev.score_pairwise_consistency(D1, D2, A)
    _same_matrices(host, dev, "unsharded ae %g" % ae)

    if LIB not in sys.path:
        sys.path.insert(0, LIB)
    import clipperpy as cp

    class PyAsym(cp.invariants.PairwiseInvariant):
        def __call__(self, ai, aj, bi, bj):
            return _asym(ai, aj, bi, bj, offset)

    p = cp.Params()
    p.affinityeps = ae
    pc = cp.CLIPPER(PyAsym(), p)
    pc.set_device(0, 1)
    pc.score_pairwise_consistency(D1, D2, A)
    assert np.array_equal(_bits(pc.get_affinity_matrix()), _bits(M))
    assert np.array_equal(_bits(pc.get_constraint_matrix()), _bits(Cm))
    cc = cp.CLIPPER(cp.invariants.CudaInvariant(ASYM_SRC, [offset]), p)
    cc.set_device(0, 1)
    cc.score_pairwise_consistency(D1, D2, A)
    assert np.array_equal(_bits(cc.get_affinity_matrix()), _bits(M))
    assert np.array_equal(_bits(cc.get_constraint_matrix()), _bits(Cm))

    # two shards: the same rows as the host matrix, and the same solve as shards loaded with it
    gs = cd.ShardGroup(lambda: clp.invariants.CudaInvariant(ASYM_SRC, (offset,)), _params(clp, ae), [0, 0],
                       storage=1, same_device=True)
    gs.score_pairwise_consistency(D1, D2, A)
    gl = cd.ShardGroup(lambda: HostAsym(), _params(clp, ae), [0, 0], storage=1, same_device=True)
    gl.set_matrix_data(M, Cm)
    for r in range(2):
        assert gs.shards[r].count_nonzeros() == gl.shards[r].count_nonzeros(), r
    u0 = np.random.default_rng(9).random(A.shape[0])
    for mode in (6, 0):
        for sh in gs.shards + gl.shards:
            sh.set_dense_mode(mode)
        sa, sb = gs.solve(u0), gl.solve(u0)
        for s in sa[1:] + sb:
            _same_solution(sa[0], s, "two shards ae %g mode %d" % (ae, mode))


# ---- 4. the notebook's Custom invariant ---------------------------------------------------------------------------------
def _bunny_problem(m=1000, n1=1000, n2o=250, outrat=0.9, noise=0.01, seed=4):
    rng = np.random.default_rng(seed)
    xyz = np.load(os.path.join(ROOT, "tests", "golden", "bun10k_points.npz"))["xyz"].astype(np.float64)
    xyz = (xyz - xyz.min(0)) / (xyz.max(0) - xyz.min(0)).max()
    D1 = xyz[rng.choice(xyz.shape[0], n1, replace=False)].T
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    w, x, y, z = q
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    D2 = R @ D1 + rng.uniform(-5, 5, (3, 1)) + rng.uniform(-noise / 2, noise / 2, D1.shape)
    O2 = rng.normal(size=(3, n2o)); O2 /= np.linalg.norm(O2, axis=0); O2 *= rng.random(n2o) ** (1 / 3)
    D2 = np.hstack([D2, O2 + D2.mean(1, keepdims=True)])
    noa = round(m * outrat)
    good = rng.choice(n1, m - noa, replace=False)
    bad = np.stack([rng.integers(0, n1, noa), rng.integers(0, n1 + n2o, noa)], 1)
    bad[bad[:, 0] == bad[:, 1], 1] = (bad[bad[:, 0] == bad[:, 1], 1] + 1) % (n1 + n2o)
    A = np.asfortranarray(np.vstack([np.stack([good, good], 1), bad]).astype(np.int32))
    return np.asfortranarray(D1), np.asfortranarray(D2), A


def test_notebook_custom_invariant(clp):
    sigma, eps = 0.015, 0.02
    D1, D2, A = _bunny_problem()

    class Custom(clp.invariants.PairwiseInvariant):   # the notebook's class
        def __call__(self, ai, aj, bi, bj):
            c = np.abs(np.linalg.norm(ai - aj) - np.linalg.norm(bi - bj))
            return np.exp(-0.5 * c ** 2 / sigma ** 2) if c < eps else 0

    params = clp.Params()
    host = clp.CLIPPER(Custom(), params, storage=1)
    host.score_pairwise_consistency(D1, D2, A)
    dev = clp.CLIPPER(clp.invariants.CudaInvariant(NOTEBOOK_SRC, (sigma, eps)), params, storage=1)
    dev.score_pairwise_consistency(D1, D2, A)
    Mh, Ch = host.get_affinity_matrix(), host.get_constraint_matrix()
    Md, Cd = dev.get_affinity_matrix(), dev.get_constraint_matrix()
    E1, E2 = D1.T[A[:, 0]], D2.T[A[:, 1]]
    l1 = np.linalg.norm(E1[:, None, :] - E1[None, :, :], axis=2)
    l2 = np.linalg.norm(E2[:, None, :] - E2[None, :, :], axis=2)
    c = np.abs(l1 - l2)
    near = (np.abs(c - eps) < 1e-12) | (np.abs(Mh - params.affinityeps) < 1e-12) | (np.abs(Md - params.affinityeps) < 1e-12)
    assert not np.any((Ch != Cd) & ~near), int(((Ch != Cd) & ~near).sum())
    both = (Ch == 1) & (Cd == 1)
    ulp = np.spacing(np.maximum(np.abs(Mh), np.abs(Md)))
    assert np.all(np.abs(Mh - Md)[both] <= 4 * ulp[both])
    assert np.count_nonzero(np.triu(Cd, 1)) > 1000
    u0 = np.ones(A.shape[0])
    host.solve(u0)
    dev.solve(u0)
    assert sorted(host.get_solution().nodes) == sorted(dev.get_solution().nodes)
    assert len(dev.get_solution().nodes) >= 50


# ---- 5. parameters and entry points -------------------------------------------------------------------------------------
def test_parameter_sets(clp):
    fam = sf.s8_tiles(129)
    for sigma, epsilon in ((0.02, 0.04), (0.05, 0.1)):
        q = dict(fam.params, sigma=sigma, epsilon=epsilon)
        f = sf.Family(fam.name, "euclid", fam.D1, fam.D2, fam.A, q)
        b = clp.CLIPPER(_builtin(clp, f), clp.Params())
        c = clp.CLIPPER(_restated(clp, f), clp.Params())
        b.score_pairwise_consistency(f.D1, f.D2, f.A)
        c.score_pairwise_consistency(f.D1, f.D2, f.A)
        _same_matrices(b, c, "sigma %g epsilon %g" % (sigma, epsilon))


def test_parameter_count_limit(clp):
    fam = sf.s8_tiles(33)
    q = fam.params
    p16 = (q["sigma"], q["epsilon"], q["mindist"]) + (7.0,) * 13
    c = clp.CLIPPER(clp.invariants.CudaInvariant(EUCLID_SRC, p16), clp.Params())
    c.score_pairwise_consistency(fam.D1, fam.D2, fam.A)
    b = clp.CLIPPER(_builtin(clp, fam), clp.Params())
    b.score_pairwise_consistency(fam.D1, fam.D2, fam.A)
    _same_matrices(b, c, "16 parameters")
    c17 = clp.CLIPPER(clp.invariants.CudaInvariant(EUCLID_SRC, p16 + (1.0,)), clp.Params())
    with pytest.raises(clp.ClipperError) as e:
        c17.score_pairwise_consistency(fam.D1, fam.D2, fam.A)
    assert e.value.code == 1


def test_all_to_all(clp):
    fam = sf.s6_distinctness()[2]   # all-to-all 5 x 6
    assert fam.A is None
    for storage in (0, 1):
        b = clp.CLIPPER(_builtin(clp, fam), clp.Params(), storage=storage)
        c = clp.CLIPPER(_restated(clp, fam), clp.Params(), storage=storage)
        b.score_pairwise_consistency(fam.D1, fam.D2)
        c.score_pairwise_consistency(fam.D1, fam.D2)
        _same_matrices(b, c, "all-to-all storage %d" % storage)
        assert np.array_equal(b.get_initial_associations(), c.get_initial_associations())


def test_device_entry_point(clp):
    import ctypes as C
    import torch
    from clipper_b200 import _capi
    fam = sf.s8_tiles(4097)
    q = fam.params
    prm = np.array([q["sigma"], q["epsilon"], q["mindist"]])
    inv = clp.invariants.CudaInvariant(EUCLID_SRC, prm)
    host = clp.CLIPPER(inv, clp.Params())
    host.score_pairwise_consistency(fam.D1, fam.D2, fam.A)
    dev = clp.CLIPPER(inv, clp.Params())
    D1 = torch.from_numpy(np.ascontiguousarray(fam.D1.T)).cuda()   # (n, d) rows = the column-major (d, n) layout
    D2 = torch.from_numpy(np.ascontiguousarray(fam.D2.T)).cuda()
    A = torch.from_numpy(np.ascontiguousarray(fam.A.T)).cuda()     # (2, m) rows = the column-major (m, 2) layout
    torch.cuda.synchronize()
    L = _capi.load()
    _capi.check(dev.handle, L.clp_score_custom_dev(dev.handle, EUCLID_SRC.encode(),
                                                   prm.ctypes.data_as(C.POINTER(C.c_double)), 3, D1.data_ptr(),
                                                   fam.d, D1.shape[0], D2.data_ptr(), D2.shape[0], A.data_ptr(),
                                                   fam.m))
    _same_matrices(host, dev, "device entry point")


# ---- 6. state and cache -------------------------------------------------------------------------------------------------
def test_broken_source_leaves_handle_unchanged(clp):
    import ctypes as C
    from clipper_b200 import _capi
    fam = sf.s8_tiles(129)
    c = clp.CLIPPER(_restated(clp, fam), clp.Params())
    c.score_pairwise_consistency(fam.D1, fam.D2, fam.A)
    M0, C0 = c.get_affinity_matrix(), c.get_constraint_matrix()
    u0 = np.random.default_rng(2).random(fam.m)
    c.solve(u0)
    s0 = c.get_solution()
    broken = EUCLID_SRC.replace("return 0.0;", "return 0.0", 1)
    prm = np.array([0.02, 0.04, 0.0])
    D1b = np.asfortranarray(fam.D1[:, :20])   # another problem (all-to-all 20 x n): nothing of it may be kept
    L = _capi.load()
    rc = L.clp_score_custom(c.handle, broken.encode(), prm.ctypes.data_as(C.POINTER(C.c_double)), 3,
                            D1b.ctypes.data_as(C.POINTER(C.c_double)), fam.d, D1b.shape[1],
                            fam.D2.ctypes.data_as(C.POINTER(C.c_double)), fam.D2.shape[1], None, 0)
    assert rc == 1
    log = L.clp_last_error(c.handle).decode()
    assert "invariant.cu(" in log and "error" in log, log
    assert np.array_equal(_bits(c.get_affinity_matrix()), _bits(M0))
    assert np.array_equal(_bits(c.get_constraint_matrix()), _bits(C0))
    assert np.array_equal(c.get_initial_associations(), fam.A)
    c.solve(u0)
    _same_solution(s0, c.get_solution(), "after the failed call")


def test_second_handle_does_not_recompile(clp):
    from clipper_b200.api import jit_stats
    fam = sf.s8_tiles(128, d=4)
    src = EUCLID_SRC + "\n// test_second_handle_does_not_recompile\n"
    q = fam.params
    a = clp.CLIPPER(clp.invariants.CudaInvariant(src, (q["sigma"], q["epsilon"], 0.0)), clp.Params())
    n0 = jit_stats()[0]
    a.score_pairwise_consistency(fam.D1, fam.D2, fam.A)
    n1 = jit_stats()[0]
    assert n1 == n0 + 1
    b = clp.CLIPPER(clp.invariants.CudaInvariant(src, (q["sigma"] * 2, q["epsilon"], 0.0)), clp.Params())
    b.score_pairwise_consistency(fam.D1, fam.D2, fam.A)
    a.score_pairwise_consistency(fam.D1, fam.D2, fam.A)
    assert jit_stats()[0] == n1


# ---- 7. downstream ------------------------------------------------------------------------------------------------------
def test_downstream_solvers(clp):
    fam = sf.s8_tiles(1000)
    for method in (clp.MCMethod.EXACT, clp.MCMethod.HEU, clp.MCMethod.KCORE):
        out = []
        for inv in (_builtin(clp, fam), _restated(clp, fam)):
            c = clp.CLIPPER(inv, clp.Params())
            c.score_pairwise_consistency(fam.D1, fam.D2, fam.A)
            mp = clp.MCParams()
            mp.method = method
            c.solve_as_maximum_clique(mp)
            out.append(c.get_solution().nodes)
        assert out[0] == out[1] and len(out[0]) > 0, method
    out = []
    for inv in (_builtin(clp, fam), _restated(clp, fam)):
        p = clp.Params()
        p.rounding = clp.Rounding.DSD
        c = clp.CLIPPER(inv, p)
        c.score_pairwise_consistency(fam.D1, fam.D2, fam.A)
        c.solve(np.random.default_rng(1).random(fam.m))
        out.append(c.get_solution())
    _same_solution(out[0], out[1], "Rounding.DSD")


# ---- 8. C++ -------------------------------------------------------------------------------------------------------------
def test_cpp_custom_invariant_tests(built):
    out = subprocess.run([os.path.join(LIB, "custom_invariant_tests")], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "2 tests" in out.stdout and "0 failures" in out.stdout
