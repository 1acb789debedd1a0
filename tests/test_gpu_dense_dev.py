"""Matrices already on the GPU: CLIPPER.set_matrix_data_dev (clp_set_dense_dev) against set_matrix_data on the same
values, and MatrixBatchCLIPPER.solve_dense_dev (clp_batch_solve_dense_dev) against solve_many on the same values, bit
for bit; their error codes, and calls on a caller's stream."""
import ctypes as C

import numpy as np
import pytest

import packed_families as pf
from test_gpu_exact_products import Stored, check_solution

pytestmark = pytest.mark.gpu

SINGLE_CASES = [c for c in pf.pair_cases() if c.m <= 4097]
BATCH_CASES = [c for c in pf.pair_cases() if c.m <= 4096]


@pytest.fixture(scope="module")
def clp(built):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import clipper_b200 as clipperpy
    return clipperpy


def _dense(case):
    """(M, C) of a case as dense fp64 arrays, strict upper triangle only"""
    M, Cm = case.upper()
    return M.toarray(), Cm.toarray()


def _poison(X):
    """X with NaN on the diagonal and -1 in the lower triangle: what the device loads must not read"""
    X = X.copy()
    X[np.tril_indices(X.shape[0], -1)] = -1.0
    np.fill_diagonal(X, np.nan)
    return X


def _layouts(torch, X, dtype):
    """the same matrix as a contiguous tensor, a .t() view of its transpose and a slice of a larger tensor"""
    m = X.shape[0]
    t = torch.from_numpy(X).to(device="cuda", dtype=dtype)
    big = torch.full((m + 3, m + 5), -1.0, dtype=dtype, device="cuda")
    big[2:m + 2, 3:m + 3] = t
    return {"contiguous": t.contiguous(), "transposed": t.t().contiguous().t(), "slice": big[2:m + 2, 3:m + 3]}


def _handle(clp, storage):
    return clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()), clp.Params(),
                       storage=storage)


def _state(c, bits):
    s = dict(nnz=c.count_nonzeros(), info=c.sparse_info(), mode=c.dense_mode())
    if bits:
        s["M"] = c.get_affinity_matrix().tobytes()
        s["C"] = c.get_constraint_matrix().tobytes()
    return s


def _solve(c, u0):
    c.solve(u0)
    s = c.get_solution()
    return (s.u.tobytes(), s.score, s.d_final, s.ifinal, s.n_evals, list(s.nodes))


def _check_single(clp, torch, storage, M, Cm, load_ref, u0, bits, layouts=("contiguous", "transposed", "slice")):
    """set_matrix_data_dev from fp64 and fp32 tensors of (M, C) against the host loads load_ref(c, M, C)"""
    for dtype in (torch.float64, torch.float32):
        Mr, Cr = (M, Cm) if dtype == torch.float64 else (M.astype(np.float32).astype(np.float64),
                                                         Cm.astype(np.float32).astype(np.float64))
        ref = _handle(clp, storage)
        load_ref(ref, Mr, Cr)
        want_state, want = _state(ref, bits), _solve(ref, u0)
        tM, tC = _layouts(torch, _poison(M), dtype), _layouts(torch, _poison(Cm), dtype)
        for lay in layouts:
            c = _handle(clp, storage)
            c.set_matrix_data_dev(tM[lay], tC[lay])
            tag = (storage, str(dtype), lay, M.shape[0])
            assert _state(c, bits) == want_state, tag
            assert _solve(c, u0) == want, tag


# ---- 1. single handle ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("storage", [0, 1])
def test_single_families(clp, storage):
    import torch
    for case in SINGLE_CASES:
        M, Cm = _dense(case)
        u0 = np.random.default_rng(1).random(case.m)
        _check_single(clp, torch, storage, M, Cm, lambda c, a, b: c.set_matrix_data(a, b), u0, bits=True)


@pytest.mark.parametrize("m", [9000, 27649])
def test_single_large(clp, m):
    """seeded weighted problems; the host reference is the sparse load of the same values (the same stored matrix)"""
    import torch
    from clipper_b200 import datagen
    prob = datagen.weighted_matrix_problem(m, 0.002, seed=m, odd=0.1)
    Ms, Cs = prob["M"].tocoo(), prob["C"].tocoo()
    dense = lambda S, dt: torch.sparse_coo_tensor(np.vstack((S.row, S.col)), S.data, (m, m)).to("cuda").to_dense().to(dt)
    for dtype in (torch.float64, torch.float32):
        Mr = Ms.astype(np.float32).astype(np.float64) if dtype == torch.float32 else Ms
        ref = _handle(clp, 0)
        ref.set_sparse_matrix_data(Mr.tocsc(), Cs.tocsc())
        want_state, want = _state(ref, m <= 9000), _solve(ref, prob["u0"])
        del ref
        for lay in ("contiguous", "transposed"):
            tM, tC = dense(Ms, dtype), dense(Cs, dtype)
            if lay == "transposed":
                tM, tC = tM.t().contiguous().t(), tC.t().contiguous().t()
            c = _handle(clp, 0)
            c.set_matrix_data_dev(tM, tC)
            del tM, tC
            assert _state(c, m <= 9000) == want_state, (m, str(dtype), lay)
            assert _solve(c, prob["u0"]) == want, (m, str(dtype), lay)
            del c
            torch.cuda.empty_cache()


# ---- 2. batch --------------------------------------------------------------------------------------------------------------
def _batch_tensors(torch, cases, dtype):
    """M, C (B, m_max, m_max) with NaN and -1 in the padding, the diagonal and the lower triangles; u0 (B, m_max)"""
    mmax = max(c.m for c in cases)
    B = len(cases)
    M = np.full((B, mmax, mmax), np.nan); Cm = np.full((B, mmax, mmax), -1.0)
    u0 = np.full((B, mmax), np.nan)
    dense = []
    for k, case in enumerate(cases):
        Mk, Ck = _dense(case)
        dense.append((Mk, Ck))
        M[k, :case.m, :case.m] = _poison(Mk); Cm[k, :case.m, :case.m] = _poison(Ck)
        u0[k, :case.m] = np.random.default_rng(1).random(case.m)
    to = lambda X, dt: torch.from_numpy(X).to(device="cuda", dtype=dt)
    return to(M, dtype), to(Cm, dtype), to(u0, torch.float64), dense, u0


@pytest.mark.parametrize("rounding", ["DSD_HEU", "NONZERO"])
def test_batch_families(clp, rounding):
    import torch
    params = clp.Params()
    params.rounding = getattr(clp.Rounding, rounding)
    for dtype in (torch.float64, torch.float32):
        tM, tC, tu0, dense, u0 = _batch_tensors(torch, BATCH_CASES, dtype)
        before = (tM.clone(), tC.clone(), tu0.clone())
        if dtype == torch.float32:
            dense = [(Mk.astype(np.float32).astype(np.float64), Ck.astype(np.float32).astype(np.float64)) for Mk, Ck in dense]
        ref = clp.MatrixBatchCLIPPER(params)
        want = ref.solve_many([dict(M=Mk, C=Ck, u0=u0[k, :c.m]) for k, ((Mk, Ck), c) in enumerate(zip(dense, BATCH_CASES))])
        b = clp.MatrixBatchCLIPPER(params)
        got = b.solve_dense_dev(tM, tC, tu0, m=[c.m for c in BATCH_CASES])
        assert b.info()[2] == ref.info()[2]
        for case, (Mk, Ck), s, w in zip(BATCH_CASES, dense, got, want):
            tag = (case.name, case.m, str(dtype), rounding)
            u = s.u.cpu().numpy()
            assert u.tobytes() == w.u.tobytes(), tag
            assert (s.score, s.d_final, s.ifinal, s.n_evals, s.n_inner, s.nodes) == \
                   (w.score, w.d_final, w.ifinal, w.n_evals, w.n_inner, w.nodes), tag
            assert s.u0.cpu().numpy().tobytes() == u0[BATCH_CASES.index(case), :case.m].tobytes(), tag
            if rounding == "DSD_HEU" and w.ifinal < params.maxoliters and case.m > 1:
                check_solution(clp, Stored.from_case(case, True), w, str(tag))
        for x, y in zip((tM, tC, tu0), before):
            assert torch.equal(x.isnan(), y.isnan()) and torch.equal(x.nan_to_num(), y.nan_to_num())


# ---- 3. errors -------------------------------------------------------------------------------------------------------------
def _raw_batch(clp, b, tM, tC, tu0, ms, dtype=0, strides=None, u0=True):
    n = len(ms)
    from clipper_b200 import _capi
    sols = (_capi.ClpSolution * n)()
    bs, rs, cs = strides if strides is not None else tM.stride()
    return b._lib.clp_batch_solve_dense_dev(b._b, n, (C.c_int64 * n)(*ms), dtype, tM.data_ptr(), tC.data_ptr(), bs, rs, cs,
                                            tu0.data_ptr() if u0 else None, tu0.stride(0), sols, None, 0, None)


def test_batch_errors(clp):
    import torch
    from clipper_b200 import datagen
    probs = [datagen.weighted_matrix_problem(64, 0.2, seed=s) for s in range(5)]
    M = torch.zeros((5, 64, 64), dtype=torch.float32, device="cuda"); Cm = torch.zeros_like(M)
    for k, p in enumerate(probs):
        M[k] = torch.from_numpy(p["M"].toarray()).float(); Cm[k] = torch.from_numpy(p["C"].toarray()).float()
    u0 = torch.from_numpy(np.stack([p["u0"] for p in probs])).cuda()
    b = clp.MatrixBatchCLIPPER()
    good = [(s.u.cpu().numpy().tobytes(), s.nodes) for s in clp.MatrixBatchCLIPPER().solve_dense_dev(M, Cm, u0)]

    def still_good():
        assert [(s.u.cpu().numpy().tobytes(), s.nodes) for s in b.solve_dense_dev(M, Cm, u0)] == good

    Mb, Cb = M.clone(), Cm.clone()
    Mb[3, 1, 7] = -0.5
    Cb[1, 2, 9] = 0.5
    with pytest.raises(clp.ClipperError) as e:
        b.solve_dense_dev(Mb, Cb, u0)
    assert e.value.code == 4 and "problem 3" in str(e.value)
    still_good()
    with pytest.raises(clp.ClipperError) as e:
        b.solve_dense_dev(M, Cb, u0)
    assert e.value.code == 4 and "problem 1" in str(e.value)
    still_good()
    Cn = Cm.clone(); Cn[2, 0, 5] = float("nan")
    with pytest.raises(clp.ClipperError) as e:
        b.solve_dense_dev(M, Cn, u0)
    assert e.value.code == 4 and "problem 2" in str(e.value)
    still_good()
    for ms, kw in [([64, 0, 64, 64, 64], {}), ([64, 4097, 64, 64, 64], {}), ([64] * 5, dict(strides=(4096, 2, 128))),
                   ([64] * 5, dict(u0=False)), ([64] * 5, dict(dtype=7))]:
        assert _raw_batch(clp, b, M, Cm, u0, ms, **kw) == 1, (ms, kw)
        still_good()
    p = clp.Params(); p.rounding = clp.Rounding.DSD
    with pytest.raises(clp.ClipperError) as e:
        clp.MatrixBatchCLIPPER(p).solve_dense_dev(M, Cm, u0)
    assert e.value.code == 4
    with pytest.raises(TypeError):
        b.solve_dense_dev(M.half(), Cm.half(), u0)
    with pytest.raises(ValueError):
        b.solve_dense_dev(M.cpu(), Cm.cpu(), u0)


def test_single_errors(clp):
    import torch
    from clipper_b200 import datagen
    p = datagen.weighted_matrix_problem(300, 0.1, seed=4)
    M, Cm = p["M"].toarray(), p["C"].toarray()
    fresh = _handle(clp, 0)
    fresh.set_matrix_data(M, Cm)
    want = _solve(fresh, p["u0"])
    for bad in ("M", "C"):
        Mb, Cb = M.copy(), Cm.copy()
        if bad == "M":
            Mb[3, 50] = -1.0
        else:
            Cb[3, 50] = 0.5
        host, dev = _handle(clp, 0), _handle(clp, 0)
        with pytest.raises(clp.ClipperError) as eh:
            host.set_matrix_data(Mb, Cb)
        with pytest.raises(clp.ClipperError) as ed:
            dev.set_matrix_data_dev(torch.from_numpy(Mb).cuda(), torch.from_numpy(Cb).cuda())
        assert (ed.value.code, str(ed.value)) == (eh.value.code, str(eh.value))
        codes = []
        for c in (host, dev):
            with pytest.raises(clp.ClipperError) as es:
                c.solve(p["u0"])
            codes.append((es.value.code, str(es.value)))
        assert codes[0] == codes[1]
        dev.set_matrix_data_dev(torch.from_numpy(M).cuda(), torch.from_numpy(Cm).cuda())
        assert _solve(dev, p["u0"]) == want
    c = _handle(clp, 0)
    tM, tC = torch.from_numpy(M).cuda(), torch.from_numpy(Cm).cuda()
    L = c._lib
    assert L.clp_set_dense_dev(c.handle, tM.data_ptr(), tC.data_ptr(), 300, 1, 2, 600) == 1   # no unit stride
    assert L.clp_set_dense_dev(c.handle, tM.data_ptr(), tC.data_ptr(), 300, 5, 300, 1) == 1   # unknown dtype
    assert L.clp_set_dense_dev(c.handle, None, tC.data_ptr(), 300, 1, 300, 1) == 1
    with pytest.raises(TypeError):
        c.set_matrix_data_dev(tM.float(), tC)
    with pytest.raises(ValueError):
        c.set_matrix_data_dev(tM.cpu(), tC.cpu())
    s = _handle(clp, 0)
    assert L.clp_shard_config(s.handle, 0, 2) == 0
    assert L.clp_set_dense_dev(s.handle, tM.data_ptr(), tC.data_ptr(), 300, 1, 300, 1) == 4


# ---- 4. streams ------------------------------------------------------------------------------------------------------------
def test_caller_stream(clp):
    """M made by a torch kernel on a side stream and loaded on that stream without a synchronisation"""
    import torch
    from clipper_b200 import datagen
    probs = [datagen.weighted_matrix_problem(1500, 0.05, seed=s) for s in range(8)]
    Mh = torch.from_numpy(np.stack([p["M"].toarray() for p in probs])).float()
    Ch = torch.from_numpy(np.stack([p["C"].toarray() for p in probs])).float()
    u0 = torch.from_numpy(np.stack([p["u0"] for p in probs])).cuda()
    u0_before = u0.clone()
    M2, Cd = (2.0 * Mh).cuda(), Ch.cuda()
    torch.cuda.synchronize()
    want = [(s.u.cpu().numpy().tobytes(), s.nodes) for s in clp.MatrixBatchCLIPPER().solve_dense_dev(M2 * 0.5, Cd, u0)]
    c0 = _handle(clp, 0)
    c0.set_matrix_data_dev(M2[0] * 0.5, Cd[0])
    want1 = _solve(c0, probs[0]["u0"])
    side = torch.cuda.Stream()
    b = clp.MatrixBatchCLIPPER()
    b.set_stream(side.cuda_stream)
    c = _handle(clp, 0)
    c.set_stream(side.cuda_stream)
    for _ in range(2):
        with torch.cuda.stream(side):
            M = M2 * 0.5   # a torch kernel on the side stream, not waited for
            got = [(s.u.cpu().numpy().tobytes(), s.nodes) for s in b.solve_dense_dev(M, Cd, u0)]
            Mc = M2 * 0.5
            c.set_matrix_data_dev(Mc[0], Cd[0])
        assert got == want
        assert _solve(c, probs[0]["u0"]) == want1
    torch.cuda.synchronize()
    assert torch.equal(M, M2 * 0.5) and torch.equal(Cd, Ch.cuda()) and torch.equal(u0, u0_before)
