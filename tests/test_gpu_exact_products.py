"""Every sweep and solver kernel against an exact fp64 product of the matrix the library actually stores.

The reference is the stored matrix itself (get_affinity_matrix / get_constraint_matrix, or the inputs rounded the way
fp32 storage rounds them), held as fp64 CSR.  The tolerance is a rounding-error bound that holds for any summation order
(Higham, Accuracy and Stability of Numerical Algorithms, section 3.1): with u = 2^-53 and gamma(k) = k u / (1 - k u), a
sum of k products computed in fp64 is within gamma(k) * sum |terms| of the exact value.  Kernel and reference each carry
such an error, hence the factor 2.  Fillers, padding and the zeros of the dense sweeps add exact zeros, so one wrong
bit in a stored value, a dropped entry or an entry credited to the wrong column exceeds the bound by orders of
magnitude, and a row whose |M| |v| is 0 must come back exactly 0.

Families (tests/packed_families.py): F1 packed-delta edges, F2 the exponent window and its fall-backs, F3 imbalance at
the resident limit, F4 tile / stripe / segment edges, F5 scored and tiny problems.
"""
import ctypes as C
import math
import os
from decimal import ROUND_HALF_UP, Decimal

import numpy as np
import pytest
import scipy.sparse as sp

import packed_families as pf
from fixtures import bytes_per_pass

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
MODES = (4, 0, 2, 3, 6)
DENSE_LOAD_MAX_M = 4097   # larger pair-list cases are loaded with set_sparse_matrix_data


def gamma(k):
    k = np.asarray(k, np.float64)
    return k * U / (1.0 - k * U)


@pytest.fixture(scope="module")
def clp(built):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import clipper_b200 as clipperpy
    return clipperpy


class _env:
    """sets environment variables for the handles created inside (they are read when a handle is created)"""
    def __init__(self, **kw):
        self.kw = {k: str(v) for k, v in kw.items()}

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.kw}
        os.environ.update(self.kw)

    def __exit__(self, *exc):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# ---- the reference: the stored matrix on the host ----------------------------------------------------------------------
class Stored:
    """Mhat = M - I and Chat = C - I of the stored matrix as fp64 CSR; k[i] = stored off-diagonal entries of row i"""

    def __init__(self, Mh, Ch):
        self.Mh, self.Ch = sp.csr_matrix(Mh), sp.csr_matrix(Ch)
        self.Mh.eliminate_zeros(); self.Ch.eliminate_zeros()
        self.m = self.Mh.shape[0]
        K = (abs(self.Mh) + self.Ch).tocsr(); K.eliminate_zeros()
        self.K = K.astype(bool)
        self.k = np.diff(self.K.indptr).astype(np.float64)

    @classmethod
    def read_back(cls, c):
        A = c.get_affinity_matrix(); np.fill_diagonal(A, 0.0)
        Cm = c.get_constraint_matrix(); np.fill_diagonal(Cm, 0.0)
        return cls(sp.csr_matrix(A), sp.csr_matrix(Cm))

    @classmethod
    def from_case(cls, case, f32):
        Mh, Ch, _ = case.stored(f32)
        return cls(Mh, Ch)


def check_matvec(ref, v, d, y, Mv, Cv, what, exact_c=False):
    """Mv, Cv and y = Md v of clp_matvec (y_i = (1 + d) v_i - d sum(v) + (Mhat v)_i + d (Chat v)_i, clipper.cpp:219)
    against the stored matrix"""
    m, k = ref.m, ref.k
    av = np.abs(v)
    rM, rC = ref.Mh @ v, ref.Ch @ v
    aM, aC = ref.Mh @ av, ref.Ch @ av
    _within(Mv, rM, 2 * gamma(k + 2) * aM, what + " Mv")
    if exact_c:
        bad = np.flatnonzero(Cv != rC)
        assert bad.size == 0, "%s Cv: row %d is %r, exactly %r" % (what, bad[0], Cv[bad[0]], rC[bad[0]])
    else:
        _within(Cv, rC, 2 * gamma(k + 2) * aC, what + " Cv")
    ry = ((1 + d) * v - d * v.sum()) + rM + d * rC
    by = 2 * gamma(k + m + 6) * ((1 + abs(d)) * av + abs(d) * av.sum() + aM + abs(d) * aC)
    _within(y, ry, by, what + " y")


def _within(x, r, bound, what):
    err = np.abs(x - r)
    bad = np.flatnonzero(~(err <= bound))
    if bad.size:
        i = bad[np.argmax(err[bad] - bound[bad])]
        raise AssertionError("%s: %d rows outside the bound; row %d: got %r, exact %r, |error| %.3e > bound %.3e"
                             % (what, bad.size, i, x[i], r[i], err[i], bound[i]))


def _round_half_away(x):
    return int(Decimal(x).quantize(Decimal(1), rounding=ROUND_HALF_UP))


def check_solution(clp, ref, s, what):
    """a solve that ended through the penalty test: score is the objective of the returned u at d_final, u is a unit
    vector in the non-negative orthant, the nodes are the round(score) largest entries of u (Rounding::DSD_HEU)"""
    u, d, m = s.u, s.d_final, ref.m
    assert np.all(u >= 0), "%s: negative entry in u" % what
    # sum of m squares, its square root and the division of the kernel (gamma(m) / 2 + 2u) and this test's square root
    nrm = math.sqrt(math.fsum(u * u))
    assert abs(nrm - 1.0) <= gamma(m + 3), "%s: |u| = %r" % (what, nrm)
    S = u.sum()
    g = (((1 + d) * u - d * S) + ref.Mh @ u) + d * (ref.Ch @ u)
    F = math.fsum(u * g)
    B = float(np.sum(u * ((1 + abs(d)) * u + abs(d) * S + ref.Mh @ u + abs(d) * (ref.Ch @ u))))
    kmax = float(ref.k.max()) if m else 0.0
    bound = 4 * gamma(2 * m + kmax + 8) * B
    assert abs(s.score - F) <= bound, "%s: score %r, exact objective of u %r, |error| %.3e > bound %.3e" % (
        what, s.score, F, abs(s.score - F), bound)
    assert list(s.nodes) == clp.utils.find_indices_of_k_largest(u, _round_half_away(s.score)).tolist(), what


def solve_converged(clp, c, m, what, seeds=(1, 2, 3)):
    """solve from u0 seeds in turn until one ends through the penalty test (ifinal < maxoliters)"""
    maxol = clp.Params().maxoliters
    for seed in seeds:
        c.solve(np.random.default_rng(seed).random(m))
        s = c.get_solution()
        if s.ifinal < maxol:
            return s
    raise AssertionError("%s: no start vector of %s converged within maxoliters" % (what, seeds))


def _vectors(m, seed):
    rng = np.random.default_rng(seed)
    return rng.random(m), rng.integers(0, 1 << 20, m).astype(np.float64)


# ---- loading ----------------------------------------------------------------------------------------------------------
def _handle(clp, storage, pack=1):
    with _env(CLP_PACK=pack):
        return clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()), clp.Params(),
                           storage=storage)


def _load(c, case, how):
    if how == "dense":
        c.set_matrix_data(*case.dense_upper())
    else:
        c.set_sparse_matrix_data(*case.upper())


def _score(clp, prob, storage, pack=1, mode=None):
    cfg = prob["cfg"]
    if cfg["kind"] == "euclidean":
        ip = clp.invariants.EuclideanDistanceParams(); ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
        inv = clp.invariants.EuclideanDistance(ip)
    else:
        ip = clp.invariants.PointNormalDistanceParams()
        ip.sigp, ip.epsp, ip.sign, ip.epsn = cfg["sigp"], cfg["epsp"], cfg["sign"], cfg["epsn"]
        inv = clp.invariants.PointNormalDistance(ip)
    with _env(CLP_PACK=pack):
        c = clp.CLIPPER(inv, clp.Params(), storage=storage)
    if mode is not None:
        c.set_dense_mode(mode)
    c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
    return c


SCORED = (("c2", 100), ("c2", 3001), ("c2", 9000), ("c3", 700))


def _scored_problem(name, m):
    from clipper_b200 import datagen
    return datagen.config_problem(name, m)


def _gate_from_ref(ref):
    """rule 1 on the stored fp32 values (read back): plain (every kept entry has an affinity and a constraint bit) and
    every kept exponent field >= b + 1, b = max(largest field - 15, 0)"""
    if ref.K.nnz == 0:
        return True
    if not (ref.Mh.nnz == ref.Ch.nnz == ref.K.nnz):
        return False
    E = pf.f32_field(ref.Mh.data)
    return bool(E.min() >= max(int(E.max()) - 15, 0) + 1)


# ---- section 1: every sweep against the stored matrix, and the solvers on the same matrices ---------------------------
def _run_all_modes(clp, c, ref, m, storage, packed, what, load_again):
    """modes 4, 0, 2, 3, 6 on handle c (default CLP_PACK): effective mode, sparse_info, Mv / Cv / y bounds and the solve
    identity; then mode 6 under CLP_PACK=0 on a fresh handle made by load_again"""
    f32 = storage == 0
    esize = 4 if f32 else 8
    v, vint = _vectors(m, m)
    for mode in MODES:
        c.set_dense_mode(mode)
        eff = c.dense_mode()
        assert eff == pf.predict_mode(mode, m, ref.K, f32, packed), "%s: mode %d ran as %d" % (what, mode, eff)
        tag = "%s mode %d->%d" % (what, mode, eff)
        if eff == 6:
            assert c.sparse_info() == (ref.K.nnz, bytes_per_pass(ref.K, packed, esize)), tag
        elif eff == 3:
            assert c.sparse_info() == (ref.K.nnz, pf.seg_bytes_per_pass(ref.K, esize)[0]), tag
        for vec, d, exact in ((v, 0.7, False), (vint, 1.3, True)):
            check_matvec(ref, vec, d, *c.matvec(vec, d), tag, exact_c=exact)
        check_solution(clp, ref, solve_converged(clp, c, m, tag), tag)
    if f32:
        c0 = load_again(0)
        c0.set_dense_mode(6)
        eff = c0.dense_mode()
        tag = "%s CLP_PACK=0 mode 6->%d" % (what, eff)
        if eff == 6:
            assert c0.sparse_info() == (ref.K.nnz, bytes_per_pass(ref.K, False)), tag
        check_matvec(ref, v, 0.7, *c0.matvec(v, 0.7), tag)
        check_matvec(ref, vint, 1.3, *c0.matvec(vint, 1.3), tag, exact_c=True)
        check_solution(clp, ref, solve_converged(clp, c0, m, tag), tag)


PAIR_CASES = {c.name: c for c in pf.pair_cases()}


@pytest.mark.parametrize("storage", [0, 1])
@pytest.mark.parametrize("name", list(PAIR_CASES))
def test_pair_families_vs_stored_matrix(clp, name, storage):
    case = PAIR_CASES[name]
    m = case.m
    how = "dense" if m <= DENSE_LOAD_MAX_M else "sparse"

    def load_again(pack):
        c = _handle(clp, storage, pack); _load(c, case, how); return c
    c = load_again(1)
    ref = Stored.read_back(c)
    # the stored matrix is the input rounded the way the storage type rounds it
    exp = Stored.from_case(case, storage == 0)
    assert (ref.Mh != exp.Mh).nnz == 0 and (ref.Ch != exp.Ch).nnz == 0, name
    packed = storage == 0 and pf.pack_gate(case)[0]
    assert packed == (storage == 0 and _gate_from_ref(ref))
    _run_all_modes(clp, c, ref, m, storage, packed, "%s storage %d" % (name, storage), load_again)


@pytest.mark.parametrize("storage", [0, 1])
@pytest.mark.parametrize("m", [27648, 27649])
def test_f3_imbalance_vs_stored_matrix(clp, m, storage):
    """F3 loaded with set_sparse_matrix_data; the reference is built from the inputs (a dense read-back would be 6 GB)"""
    case, _, _ = pf.f3_imbalance(m)

    def load_again(pack):
        c = _handle(clp, storage, pack); _load(c, case, "sparse"); return c
    c = load_again(1)
    ref = Stored.from_case(case, storage == 0)
    assert c.count_nonzeros() == (case.i.size, case.i.size)
    packed = storage == 0 and pf.pack_gate(case)[0]
    _run_all_modes(clp, c, ref, m, storage, packed, "F3 m=%d storage %d" % (m, storage), load_again)


@pytest.mark.parametrize("storage", [0, 1])
@pytest.mark.parametrize("name,m", SCORED)
def test_scored_problems_vs_stored_matrix(clp, name, m, storage):
    """F5: scored problems (fp32 storage counts the kept entries inside the scoring kernel)"""
    prob = _scored_problem(name, m)
    c = _score(clp, prob, storage)
    ref = Stored.read_back(c)
    packed = storage == 0 and _gate_from_ref(ref)
    assert packed or storage == 1, "a scored fp32 matrix is plain and fits the exponent window"
    _run_all_modes(clp, c, ref, m, storage, packed, "%s m=%d storage %d" % (name, m, storage),
                   lambda pack: _score(clp, prob, storage, pack))


# ---- the build paths must meet ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("storage", [0, 1])
@pytest.mark.parametrize("name", ["F1_deltas_m641", "F2_1_subnormal", "F2_1_mc0", "F2_1_m0c1", "F2_2m115_in", "F4_m2049"])
def test_dense_and_sparse_loading_store_the_same_matrix(clp, name, storage):
    case = PAIR_CASES[name]
    a, b = _handle(clp, storage), _handle(clp, storage)
    _load(a, case, "dense"); _load(b, case, "sparse")
    assert np.array_equal(a.get_affinity_matrix(), b.get_affinity_matrix())
    assert np.array_equal(a.get_constraint_matrix(), b.get_constraint_matrix())
    v, _ = _vectors(case.m, 5)
    for mode in MODES:
        a.set_dense_mode(mode); b.set_dense_mode(mode)
        assert a.dense_mode() == b.dense_mode() and a.sparse_info() == b.sparse_info()
        for x, y in zip(a.matvec(v, 0.9), b.matvec(v, 0.9)):
            assert x.tobytes() == y.tobytes(), (name, mode)


@pytest.mark.parametrize("pack", [1, 0])
@pytest.mark.parametrize("name,m", SCORED)
def test_fused_counts_equal_counting_kernel(clp, name, m, pack):
    """mode 6 built from the counts of the scoring kernel, then re-finalised through mode 0 (the counting kernel):
    the same layout and the same mat-vec bit for bit"""
    prob = _scored_problem(name, m)
    c = _score(clp, prob, 0, pack, mode=6)
    v, _ = _vectors(m, 6)
    assert c.dense_mode() == 6
    info, mv = c.sparse_info(), c.matvec(v, 0.4)
    c.set_dense_mode(0); c.set_dense_mode(6)
    assert c.dense_mode() == 6 and c.sparse_info() == info
    for x, y in zip(c.matvec(v, 0.4), mv):
        assert x.tobytes() == y.tobytes()


def test_matvec_dev_equals_matvec(clp):
    import torch
    case = PAIR_CASES["F1_deltas_m641"]
    c = _handle(clp, 0); _load(c, case, "dense"); c.set_dense_mode(6)
    assert c.sparse_info()[1] == bytes_per_pass(case.stored(True)[2], True)   # packed
    v, _ = _vectors(case.m, 7)
    host = c.matvec(v, 0.8)
    vd = torch.from_numpy(v).cuda()
    outs = [torch.zeros(case.m, dtype=torch.float64, device="cuda") for _ in range(3)]
    ms = C.c_double()
    from clipper_b200 import _capi
    L = _capi.load()
    _capi.check(c.handle, L.clp_matvec_dev(c.handle, vd.data_ptr(), 0.8, outs[0].data_ptr(), outs[1].data_ptr(),
                                           outs[2].data_ptr(), 1, C.byref(ms)))
    torch.cuda.synchronize()
    for x, y in zip(outs, host):
        assert x.cpu().numpy().tobytes() == y.tobytes()


# ---- section 2: the sharded and the batched solvers ---------------------------------------------------------------------
SHARD_CASES = ("F1_deltas_m641", "F2_1_in", "F2_1_mc0", "F2_1_m0c1", "c2_3000")


@pytest.mark.parametrize("storage", [0, 1])
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_solvers_vs_stored_matrix(clp, world, storage):
    """ShardGroup on one GPU (grid cap SMs / world, one CTA per SM), modes 6, 3 and 0 on the shards; the reference is the
    matrix an unsharded handle stores for the same input; all ranks bit-identical"""
    from clipper_b200 import distributed as cd
    for name in SHARD_CASES:
        if name == "c2_3000":
            prob = _scored_problem("c2", 3000)
            single = _score(clp, prob, storage)
            cfg = prob["cfg"]

            def inv():
                ip = clp.invariants.EuclideanDistanceParams(); ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
                return clp.invariants.EuclideanDistance(ip)
            g = cd.ShardGroup(inv, clp.Params(), [0] * world, storage=storage, same_device=True)
            g.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
        else:
            case = PAIR_CASES[name]
            single = _handle(clp, storage); _load(single, case, "dense")
            g = cd.ShardGroup(lambda: clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()),
                              clp.Params(), [0] * world, storage=storage, same_device=True)
            g.set_matrix_data(*case.dense_upper())
        ref = Stored.read_back(single)
        m = ref.m
        assert g.count_nonzeros() == single.count_nonzeros()
        maxol = clp.Params().maxoliters
        for mode in (6, 3, 0):
            for sh in g.shards:
                sh.set_dense_mode(mode)
                assert sh.dense_mode() == mode
            tag = "%s world %d storage %d mode %d" % (name, world, storage, mode)
            for seed in (1, 2, 3):
                sols = g.solve(np.random.default_rng(seed).random(m))
                if sols[0].ifinal < maxol:
                    break
            else:
                raise AssertionError("%s: no start vector converged within maxoliters" % tag)
            for s in sols[1:]:
                assert s.u.tobytes() == sols[0].u.tobytes() and s.score == sols[0].score, tag
                assert s.d_final == sols[0].d_final and s.nodes == sols[0].nodes, tag
            check_solution(clp, ref, sols[0], tag)
        del g


def test_batch_solver_vs_stored_matrix(clp):
    """every problem of a batch: the identity on the matrix a single-problem handle stores for the same inputs"""
    from test_gpu_batch import _euclid, _problems
    sizes = [64, 100, 256, 333, 512, 777, 1000, 1024, 1500, 2048, 65, 129, 12, 4, 640, 900]
    probs = _problems(sizes, 500)
    sigma, eps = 0.015, 0.05
    b = clp.BatchCLIPPER(_euclid(clp, sigma, eps), clp.Params())
    maxol = clp.Params().maxoliters
    sols = b.solve_many(probs)
    nnz_batch = b.info()[2]
    for seed in (1, 2):   # problems that did not end through the penalty test start again from other vectors
        redo = [k for k, s in enumerate(sols) if s.ifinal >= maxol]
        if not redo:
            break
        again = b.solve_many([dict(probs[k], u0=np.random.default_rng(seed).random(sizes[k])) for k in redo])
        for k, s in zip(redo, again):
            sols[k] = s
    nnz = 0
    for k, (p, s) in enumerate(zip(probs, sols)):
        tag = "batch problem %d (m=%d)" % (k, sizes[k])
        assert s.ifinal < maxol, tag
        c = clp.CLIPPER(_euclid(clp, sigma, eps), clp.Params())
        c.score_pairwise_consistency(p["D1"], p["D2"], p["A"])
        ref = Stored.read_back(c)
        nnz += ref.K.nnz // 2
        check_solution(clp, ref, s, tag)
    assert nnz_batch == nnz
