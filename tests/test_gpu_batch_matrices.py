"""Batches of problems given as (M, C) matrices in one launch (clp_batch_solve_matrices, MatrixBatchCLIPPER): every
problem against an fp32 single-problem handle loaded with the same matrices, the stored-matrix identity of
test_gpu_exact_products, the CPU oracle, the scored batch on the same matrices, the error codes and reproducibility."""
import ctypes as C

import numpy as np
import pytest

import packed_families as pf
from test_gpu_exact_products import Stored, check_solution

pytestmark = pytest.mark.gpu

BATCH_CASES = [c for c in pf.pair_cases() if c.m <= 4096]


@pytest.fixture(scope="module")
def clp(built):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import clipper_b200 as clipperpy
    return clipperpy


def _params(clp, rounding=None):
    p = clp.Params()
    if rounding is not None:
        p.rounding = rounding
    return p


def _single(clp, M, Cm, u0, params=None, dense=False):
    """fp32 handle loaded with set_matrix_data / set_sparse_matrix_data, solved from u0"""
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()),
                    params if params is not None else clp.Params(), storage=clp.STORE_F32)
    if dense:
        c.set_matrix_data(M, Cm)
    else:
        c.set_sparse_matrix_data(M, Cm)
    c.solve(u0)
    return c.get_solution()


def _same_bits(a, b):
    return a.u.tobytes() == b.u.tobytes() and a.score == b.score and a.nodes == b.nodes


def _agrees_with_single(s, s1, tag, same_evals=True):
    """the decisions of the batch and of a single handle agree.  The two run the same arithmetic with a different
    summation order (one 256-thread CTA against the single handle's grid and layout), so objective values differ in the
    last bits.  For affinities near the reference's contract (M in [0, 1]; the F2_2m family reaches 2 - 2^-23) that
    does not move a line-search decision; with affinities up to 2^20 (the F2_2p20 family) the objective is about 2^40
    times larger and the last-bit differences change how many evaluations a line search takes (2318 against 2239 on
    the H100 for F2_2p20_in), with the same nodes and ifinal"""
    assert s.nodes == s1.nodes, tag
    assert s.ifinal == s1.ifinal, (tag, s.ifinal, s1.ifinal)
    if same_evals:
        assert s.n_evals == s1.n_evals, (tag, s.n_evals, s1.n_evals)
    assert abs(s.score - s1.score) <= 1e-9 * max(1.0, abs(s1.score)), (tag, s.score, s1.score)


# ---- 1. the packed families in one call --------------------------------------------------------------------------------
def test_families_in_one_call(clp):
    """every pair-list case with m <= 4096 (sizes 1 to 4096, plain and non-plain, subnormal, empty) in ONE call"""
    b = clp.MatrixBatchCLIPPER()
    maxol = clp.Params().maxoliters
    probs = [dict(zip(("M", "C"), case.upper()), u0=np.random.default_rng(1).random(case.m)) for case in BATCH_CASES]
    sols = b.solve_many(probs)
    first = list(sols)
    assert b.info()[2] == sum(Stored.from_case(case, True).K.nnz // 2 for case in BATCH_CASES)
    for seed in (2, 3):   # problems that did not end through the penalty test start again from other vectors
        redo = [k for k, s in enumerate(sols) if s.ifinal >= maxol]
        if not redo:
            break
        again = b.solve_many([dict(probs[k], u0=np.random.default_rng(seed).random(BATCH_CASES[k].m)) for k in redo])
        for k, s in zip(redo, again):
            sols[k] = s
    for case, p, s in zip(BATCH_CASES, probs, sols):
        tag = "%s (m=%d)" % (case.name, case.m)
        assert s.ifinal < maxol, tag
        check_solution(clp, Stored.from_case(case, True), s, tag)
        _agrees_with_single(s, _single(clp, *case.upper(), s.u0), tag, same_evals=not case.name.startswith("F2_2p20"))
    # the same cases as dense arrays: the same CSC, the same bits
    dense = b.solve_many([dict(zip(("M", "C"), case.dense_upper()), u0=p["u0"]) for case, p in zip(BATCH_CASES, probs)])
    for case, a, d in zip(BATCH_CASES, first, dense):
        assert _same_bits(a, d), case.name


# ---- 2. against the CPU oracle -----------------------------------------------------------------------------------------
def _weighted_set():
    from clipper_b200 import datagen
    sizes = np.unique(np.geomspace(4, 4096, 32).astype(int))
    out = []
    for k, m in enumerate(sizes):
        dens = 0.05 + 0.10 * (k % 5) / 4
        out.append(datagen.weighted_matrix_problem(int(m), dens, 4200 + k, odd=0.1 if k % 3 == 2 else 0.0))
    return out


def _oracle_problems(clp):
    import fixtures as fx
    import scipy.sparse as sp
    probs = []
    M, Cm = fx.m20()
    probs.append(dict(M=M, C=Cm, u0=np.random.default_rng(20).random(20)))
    model, data = fx.toy_problem()
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()), clp.Params())
    c.score_pairwise_consistency(model, data)
    probs.append(dict(M=c.get_affinity_matrix(), C=c.get_constraint_matrix(), u0=np.full(12, 0.5)))
    for p in _weighted_set():
        probs.append(dict(M=sp.csc_matrix(p["M"]), C=p["C"], u0=p["u0"]))
    return probs


@pytest.mark.parametrize("rounding", ["DSD_HEU", "NONZERO"])
def test_weighted_vs_oracle(clp, rounding):
    """the reference's 20 x 20 weighted matrix, the toy problem's matrices read back, and seeded weighted problems
    (m 4 to 4096, 5-15 % density, planted cluster, some with (M = 0, C = 1) and (M > 0, C = 0) pairs); the oracle holds
    M rounded to fp32, so both solve the same matrix"""
    import scipy.sparse as sp
    from oracle import clipper_oracle as orc
    rnd = getattr(clp.Rounding, rounding)
    probs = _oracle_problems(clp)
    sols = clp.MatrixBatchCLIPPER(_params(clp, rnd)).solve_many(probs)
    orc_round = orc.NONZERO if rounding == "NONZERO" else orc.default_params().rounding
    for k, (p, s) in enumerate(zip(probs, sols)):
        M = p["M"].toarray() if sp.issparse(p["M"]) else np.array(p["M"])
        Cm = p["C"].toarray() if sp.issparse(p["C"]) else np.array(p["C"])
        M32 = np.triu(M, 1).astype(np.float32).astype(np.float64)
        M32 = M32 + M32.T + np.eye(M.shape[0])
        Cu = np.triu(Cm, 1)
        o = orc.Oracle(orc.default_params(rounding=orc_round))
        o.set_matrix_data(M32, Cu + Cu.T + np.eye(M.shape[0]))
        so = o.solve(p["u0"])
        tag = "problem %d (m=%d) %s" % (k, M.shape[0], rounding)
        assert sorted(s.nodes) == sorted(so.nodes.tolist()), tag
        assert abs(s.score - so.score) <= 1e-9 * max(1.0, abs(so.score)), (tag, s.score, so.score)
        assert np.abs(s.u - so.u).max() <= 1e-8, (tag, np.abs(s.u - so.u).max())


# ---- 3. the scored batch and the matrix batch on the same stored matrices -------------------------------------------
def test_scored_and_matrix_batches_agree_bit_for_bit(clp):
    from test_gpu_batch import _euclid, _problems
    sizes = [64, 100, 256, 333, 512, 777, 1000, 1024, 1500, 2048, 65, 129, 12, 4, 640, 900]
    probs = _problems(sizes, 500)
    sigma, eps = 0.015, 0.05
    scored = clp.BatchCLIPPER(_euclid(clp, sigma, eps), clp.Params()).solve_many(probs)
    mats = []
    for p in probs:
        c = clp.CLIPPER(_euclid(clp, sigma, eps), clp.Params())
        c.score_pairwise_consistency(p["D1"], p["D2"], p["A"])
        mats.append(dict(M=c.get_affinity_matrix(), C=c.get_constraint_matrix(), u0=p["u0"]))
    b = clp.MatrixBatchCLIPPER()
    given = b.solve_many(mats)
    for k, (s, g) in enumerate(zip(scored, given)):
        assert _same_bits(s, g), "problem %d (m=%d)" % (k, sizes[k])
        assert s.ifinal == g.ifinal and s.n_evals == g.n_evals and s.d_final == g.d_final


# ---- 4. errors -----------------------------------------------------------------------------------------------------------
def _raw(clp, b, items, u0s=None):
    """clp_batch_solve_matrices on raw CSC triples: items[p] = (m, cpM, riM, vM, cpC, riC, vC); u0s[p] None -> NULL"""
    from clipper_b200 import _capi
    n = len(items)
    vp = C.c_void_p
    keep = []
    m = (C.c_int64 * n)(*[it[0] for it in items])
    ptrs = [(vp * n)() for _ in range(6)]
    u0p, up, np_ = (vp * n)(), (vp * n)(), (vp * n)()
    for k, it in enumerate(items):
        arrs = [np.ascontiguousarray(it[1 + q], (np.int64, np.int32, np.float64)[q % 3]) for q in range(6)]
        keep.append(arrs)
        for q in range(6):
            ptrs[q][k] = arrs[q].ctypes.data if arrs[q].size else None
        mk = max(int(it[0]), 1)
        u0 = np.full(mk, 0.5) if (u0s is None or u0s[k] is not None) else None
        uk, nk = np.zeros(mk), np.zeros(mk, np.int32)
        keep += [u0, uk, nk]
        u0p[k] = u0.ctypes.data if u0 is not None else None
        up[k], np_[k] = uk.ctypes.data, nk.ctypes.data
    sols = (_capi.ClpSolution * n)()
    rc = b._lib.clp_batch_solve_matrices(b._b, n, m, *ptrs, u0p, sols, up, np_)
    msg = b._lib.clp_batch_last_error(b._b)
    return rc, (msg.decode() if msg else "")


def _valid():
    """m = 4: M entries (0,1) (0,2) (1,3), C entries (0,1) (0,2) (1,3) (2,3)"""
    cp = np.array([0, 0, 1, 2, 4]); ri = np.array([0, 0, 1, 2])
    return (4, np.array([0, 0, 1, 2, 3]), np.array([0, 0, 1]), np.array([0.5, 0.25, 0.75]), cp, ri, np.ones(4))


def _variant(**kw):
    names = ("m", "cpM", "riM", "vM", "cpC", "riC", "vC")
    v = dict(zip(names, _valid()))
    v.update(kw)
    return tuple(v[n] for n in names)


INVALID, UNSUPPORTED = 1, 4
ERROR_CASES = {
    "m0": (_variant(m=0, cpM=np.zeros(1), riM=np.zeros(0), vM=np.zeros(0), cpC=np.zeros(1), riC=np.zeros(0), vC=np.zeros(0)), INVALID),
    "colptr0": (_variant(cpM=np.array([1, 1, 2, 3, 4])), INVALID),
    "colptr_decreasing": (_variant(cpC=np.array([0, 0, 2, 1, 4])), INVALID),
    "row_ge_column": (_variant(riC=np.array([0, 0, 1, 3])), INVALID),
    "row_negative": (_variant(riM=np.array([0, -1, 1])), INVALID),
    "duplicate_row": (_variant(cpC=np.array([0, 0, 1, 2, 5]), riC=np.array([0, 0, 1, 1, 2]), vC=np.ones(5)), INVALID),
    "unsorted_rows": (_variant(riC=np.array([0, 0, 2, 1])), INVALID),
    "m_negative": (_variant(vM=np.array([0.5, -0.25, 0.75])), UNSUPPORTED),
    "c_half": (_variant(vC=np.array([1.0, 0.5, 1.0, 1.0])), UNSUPPORTED),
    "c_nan": (_variant(vC=np.array([1.0, np.nan, 1.0, 1.0])), UNSUPPORTED),
    # the single path's order: structure before M, M before C
    "structure_before_values": (_variant(vM=np.array([-0.5, 0.25, 0.75]), riC=np.array([0, 0, 1, 3])), INVALID),
}


def test_errors_leave_the_handle_usable(clp):
    b = clp.MatrixBatchCLIPPER()
    good = _raw(clp, b, [_valid()])
    assert good[0] == 0, good
    for name, (bad, code) in ERROR_CASES.items():
        rc, msg = _raw(clp, b, [_valid(), bad])
        assert rc == code, (name, rc, msg)
        assert "problem 1" in msg, (name, msg)
        assert _raw(clp, b, [_valid()])[0] == 0, name
    # a negative M in problem 0 and a structural error in problem 1: structure first
    rc, msg = _raw(clp, b, [ERROR_CASES["m_negative"][0], ERROR_CASES["row_ge_column"][0]])
    assert rc == INVALID and "problem 1" in msg, msg
    rc, msg = _raw(clp, b, [_valid(), _valid()], u0s=[np.ones(4), None])
    assert rc == INVALID, msg
    # problems too large for a batch: the F4 cases m = 4097 and 8193
    for case in (c for c in pf.pair_cases() if c.m > 4096):
        with pytest.raises(clp.ClipperError) as e:
            b.solve_many([dict(zip(("M", "C"), case.upper()), u0=np.full(case.m, 0.5))])
        assert e.value.code == INVALID, case.name
        assert _raw(clp, b, [_valid()])[0] == 0
    # the Python front-end: u0 of the wrong length, Rounding::DSD
    M, Cm = pf.f5_small(17).dense_upper()
    with pytest.raises(ValueError):
        b.solve_many([dict(M=M, C=Cm, u0=np.ones(16))])
    with pytest.raises(clp.ClipperError) as e:
        clp.MatrixBatchCLIPPER(_params(clp, clp.Rounding.DSD)).solve_many([dict(M=M, C=Cm, u0=np.ones(17))])
    assert e.value.code == UNSUPPORTED
    assert len(b.solve_many([dict(M=M, C=Cm, u0=np.ones(17))])) == 1


# ---- 5. reproducibility and a grid smaller than the batch ---------------------------------------------------------------
def test_reproducible_and_order_independent(clp):
    probs = _weighted_set()[::3]
    b = clp.MatrixBatchCLIPPER()
    one, two = b.solve_many(probs), b.solve_many(probs)
    rev = b.solve_many(probs[::-1])[::-1]
    for k, (x, y, z) in enumerate(zip(one, two, rev)):
        assert _same_bits(x, y) and _same_bits(x, z), k


def test_more_problems_than_ctas(clp):
    """256 problems of m = 2048 in one call (the grid holds at most the co-resident CTAs): a sample against single
    handles"""
    from clipper_b200 import datagen
    base = [datagen.weighted_matrix_problem(2048, 0.03, 9100 + k) for k in range(16)]
    probs = [dict(base[k % 16], u0=np.random.default_rng(k).random(2048)) for k in range(256)]
    b = clp.MatrixBatchCLIPPER()
    sols = b.solve_many(probs)
    assert 1 <= b.info()[0] <= len(probs)
    for k in range(0, 256, 32):
        _agrees_with_single(sols[k], _single(clp, probs[k]["M"], probs[k]["C"], probs[k]["u0"]), "problem %d" % k)
