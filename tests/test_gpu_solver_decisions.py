"""Every solver entry point against the oracle fed the matrix that entry point stores, decision for decision.

The reference is the C oracle (oracle/clipper_oracle.c) run on the stored matrix: a handle's own read-back, the read-
back of a single handle scored with the same inputs for a scored batch, or the given matrices (whose weights are fp32-
representable, so fp32 storage keeps them exactly).  Never the unrounded matrix.  The cases come from
tests/solver_families.py, whose CPU test proves every decision of every case used here robust: its margin exceeds a
rounding bound (see that file for what the bound covers).  So ifinal, n_evals, n_inner and the nodes (in order) must
be identical, with fp32 storage as with fp64.

The tolerances on d_final and score (2e-11 relative) and on u (1e-10) are measured, not derived: they are the ones
test_gpu_parity.py's test_sweep_modes_agree uses between kernels.  NaN must be NaN where the oracle's
is (u0 = 0).

Doors: the single handle in fp32 (mode 6 packed, mode 6 with CLP_PACK=0, modes 0, 2 and 3), in fp64 (modes 6 and 0),
ShardGroup with 2 and 3 shards on one GPU (modes 6 and 3), BatchCLIPPER.solve_many / solve_many_dev, a batch scored
with a CudaInvariant restating Euclidean distance, MatrixBatchCLIPPER.solve_many / solve_dense_dev, and clipperpy
through the C++ shell.  The full parameter grid runs on the default door and on mode 0 (solver_kernel); the others
run solver_families.DOOR_GRID.  Truncated runs (maxoliters = k) are checked against the oracle's run at k and rows
of its full run's trace on every single-handle door, the shards, the matrix batch and the segmented hand-over.  The
case with F > 2^31 must keep all m nodes on the single handle, the shards and both matrix-batch calls.
"""
import math
import os
import sys

import numpy as np
import pytest

import solver_families as sf

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAMS = sf.families()
SMALL = [n for n, c in FAMS.items() if c.m <= 4096]
PREFIX_CASES = ("T1_edgeless", "T5_mixed", "T7_m33")


@pytest.fixture(scope="module")
def clp(built):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import clipper_b200
    return clipper_b200


class _env:
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


_REF = {}


def oracle_ref(case, gname, key=None, trace_cap=0):
    """the oracle on the case's matrix (cached: every fp32 / fp64 door of a given case stores the same matrix)"""
    k = (key or case.name, gname, trace_cap)
    if k not in _REF:
        _REF[k] = case.oracle(sf.params(gname), trace_cap=trace_cap)[1]
    return _REF[k]


def grid_of(case, full):
    """the parameter sets a door runs on a case: the full grid (with Rounding::DSD) on the two full doors, DOOR_GRID on
    the others; a case with a grid of its own runs that"""
    return sf.grid_for(case, sf.FULL_GRID + ("dsd",) if full else sf.DOOR_GRID)


def _params(clp, P):
    p = clp.Params()
    for k, v in P.items():
        setattr(p, k, v)
    return p


def _host(x):
    return x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)


def check(s, o, what):
    got = (s.ifinal, s.n_evals, s.n_inner)
    assert got == (o.ifinal, o.n_evals, o.n_inner), "%s: (ifinal, n_evals, n_inner) %s, oracle %s" % (
        what, got, (o.ifinal, o.n_evals, o.n_inner))
    assert list(s.nodes) == o.nodes.tolist(), "%s: nodes %s, oracle %s" % (what, list(s.nodes), o.nodes.tolist())
    for name, a, b in (("d_final", s.d_final, o.d_final), ("score", s.score, o.score)):
        if math.isnan(b):
            assert math.isnan(a), "%s: %s %r, oracle NaN" % (what, name, a)
        else:
            assert abs(a - b) <= 2e-11 * abs(b), "%s: %s %r, oracle %r" % (what, name, a, b)
    u = _host(s.u)
    nan = np.isnan(o.u)
    assert np.array_equal(np.isnan(u), nan), "%s: NaN pattern of u" % what
    if (~nan).any():
        err = np.abs(u[~nan] - o.u[~nan]).max()
        assert err <= 1e-10, "%s: |u - u_oracle| = %.3e" % (what, err)


# ---- the single handle ---------------------------------------------------------------------------------------------
def _inv(clp):
    return clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams())


def single(clp, case, P, storage, mode, pack=1):
    with _env(CLP_PACK=pack):
        c = clp.CLIPPER(_inv(clp), _params(clp, P), storage=storage)
    if case.m <= 4096:
        c.set_matrix_data(*case.dense())
    else:
        c.set_sparse_matrix_data(*case.upper())
    c.set_dense_mode(mode)
    return c


SINGLE_DOORS = [  # (storage, mode, CLP_PACK, full grid)
    (0, 6, 1, True), (0, 0, 1, True), (0, 6, 0, False), (0, 2, 1, False), (0, 3, 1, False),
    (1, 6, 1, False), (1, 0, 1, False)]


@pytest.mark.parametrize("storage,mode,pack,full", SINGLE_DOORS)
def test_single_handle(clp, storage, mode, pack, full):
    checked = 0
    for name in SMALL:
        case = FAMS[name]
        M0, C0 = case.dense()
        for q, g in enumerate(grid_of(case, full)):
            P = sf.params(g)
            c = single(clp, case, P, storage, mode, pack)
            assert c.dense_mode() == mode, (name, mode, c.dense_mode())
            if q == 0:
                assert np.array_equal(c.get_affinity_matrix(), M0), "%s: stored affinities differ" % name
                assert np.array_equal(c.get_constraint_matrix(), C0), "%s: stored constraints differ" % name
            c.solve(case.u0)
            check(c.get_solution(), oracle_ref(case, g), "%s %s storage %d mode %d pack %d" % (name, g, storage, mode, pack))
            checked += 1
    assert checked > 0


# ---- trajectory prefixes -------------------------------------------------------------------------------------------
def prefix_params(case):
    """(k, params) of the truncated runs of a case: maxoliters = 1, 2, ceil(ifinal / 2) and ifinal of its full run"""
    full = oracle_ref(case, "defaults", trace_cap=1000)
    ks = sorted({k for k in (1, 2, -(-full.ifinal // 2), full.ifinal) if 1 <= k <= full.ifinal + 1})
    return [(k, dict(sf.params("defaults"), maxoliters=k)) for k in ks]


def check_prefix(s, case, k, what, full_g="defaults"):
    """a run truncated at maxoliters = k is a prefix of the full run: decision for decision the oracle's run at k, its
    score row k-1 of the full run's trace (F after the k-th inner loop), its d_final the d the full run used in
    iteration k (after the k-th ramp), its n_inner the inner steps of the first k rows"""
    full = oracle_ref(case, full_g, trace_cap=1000)
    tr = full.trace
    P = dict(sf.params(full_g), maxoliters=k)
    key = (case.name, "prefix", full_g, k)
    if key not in _REF:
        _REF[key] = case.oracle(P)[1]
    check(s, _REF[key], what)
    assert s.ifinal == min(k, full.ifinal), what
    assert abs(s.score - tr[k - 1, 0]) <= 2e-11 * abs(tr[k - 1, 0]), what
    if k < tr.shape[0]:
        assert abs(s.d_final - tr[k, 1]) <= 2e-11 * abs(tr[k, 1]), what
    assert s.n_inner == int(tr[:k, 2].sum()), what


@pytest.mark.parametrize("storage,mode,pack,full", SINGLE_DOORS)
def test_trajectory_prefixes_single(clp, storage, mode, pack, full):
    for name in PREFIX_CASES:
        case = FAMS[name]
        for k, P in prefix_params(case):
            c = single(clp, case, P, storage, mode, pack)
            assert c.dense_mode() == mode
            c.solve(case.u0)
            check_prefix(c.get_solution(), case, k, "%s maxoliters=%d storage %d mode %d pack %d" % (
                name, k, storage, mode, pack))


def test_segmented_handover(clp):
    """m = 27 649: mode 6 hands over to the segmented solver (mode 3); a short run, decision for decision"""
    case = sf.big_case()
    for g in case.grid:
        P = sf.params(g)
        c = single(clp, case, P, 0, 6)
        assert c.dense_mode() == 3
        c.solve(case.u0)
        s = c.get_solution()
        check(s, oracle_ref(case, g), "%s %s" % (case.name, g))
        if g == "short1":   # one outer iteration of short2's run (both take one inner step per outer iteration)
            check_prefix(s, case, 1, "%s prefix of short2" % case.name, full_g="short2")


@pytest.mark.parametrize("storage", [0, 1])
@pytest.mark.parametrize("name,m", sf.SCORED)
def test_scored_single(clp, name, m, storage):
    """T8: the reference is the oracle fed the handle's own read-back"""
    from clipper_b200 import datagen
    prob = datagen.config_problem(name, m); cfg = prob["cfg"]
    for g in sf.T8_GRID:
        P = sf.params(g)
        if cfg["kind"] == "euclidean":
            ip = clp.invariants.EuclideanDistanceParams(); ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
            inv = clp.invariants.EuclideanDistance(ip)
        else:
            ip = clp.invariants.PointNormalDistanceParams()
            ip.sigp, ip.epsp, ip.sign, ip.epsn = cfg["sigp"], cfg["epsp"], cfg["sign"], cfg["epsn"]
            inv = clp.invariants.PointNormalDistance(ip)
        c = clp.CLIPPER(inv, _params(clp, P), storage=storage)
        c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
        import scipy.sparse as sp
        Mr = c.get_affinity_matrix(); np.fill_diagonal(Mr, 0); Cr = c.get_constraint_matrix(); np.fill_diagonal(Cr, 0)
        ref = sf.Case("readback", "T8", sp.csr_matrix(Mr), sp.csr_matrix(Cr), prob["u0"])
        r = ref.restate(P)   # the read-back may differ from the oracle's fp32-rounded scores in the last bit
        assert r["margins"].robust, "%s m=%d %s storage %d: not robust %s" % (name, m, g, storage, r["margins"].worst)
        c.solve(prob["u0"])
        check(c.get_solution(), oracle_ref(ref, g, key=(name, m, storage)), "%s m=%d %s storage %d" % (name, m, g, storage))


# ---- sharded -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3])
def test_sharded(clp, world):
    from clipper_b200 import distributed as cd
    runs = [(FAMS[n], g, sf.params(g), None) for n in ("T3_isolated", "T5_mixed", "T6_huge", "T7_m129", "T7_m4096", "U_zero")
            for g in grid_of(FAMS[n], False)]
    runs += [(FAMS[n], "prefix", P, k) for n in PREFIX_CASES for k, P in prefix_params(FAMS[n])]
    for case, g, P, k in runs:
        grp = cd.ShardGroup(lambda: _inv(clp), _params(clp, P), [0] * world, storage=0, same_device=True)
        grp.set_matrix_data(*case.dense())
        for mode in (6, 3):
            for sh in grp.shards:
                sh.set_dense_mode(mode)
                assert sh.dense_mode() == mode
            sols = grp.solve(case.u0)
            what = "%s %s%s world %d mode %d" % (case.name, g, "" if k is None else " maxoliters=%d" % k, world, mode)
            for s in sols[1:]:
                assert s.u.tobytes() == sols[0].u.tobytes() and list(s.nodes) == list(sols[0].nodes), what
            if k is None:
                check(sols[0], oracle_ref(case, g), what)
            else:
                check_prefix(sols[0], case, k, what)
        del grp


# ---- batches of given matrices -------------------------------------------------------------------------------------
def _matrix_batch_runs():
    """(parameter set, params, case names, maxoliters of a prefix run or None): every case in every parameter set of
    its grid (DOOR_GRID, or the case's own, e.g. T6_huge's), and the prefix runs"""
    runs = []
    for g in list(sf.DOOR_GRID) + sorted({x for c in FAMS.values() if c.grid for x in c.grid} - set(sf.DOOR_GRID)):
        use = [n for n in SMALL if g in sf.grid_for(FAMS[n], sf.DOOR_GRID)]
        if use:
            runs.append((g, sf.params(g), use, None))
    for k in (1, 2):
        use = [n for n in PREFIX_CASES if k in [q for q, _ in prefix_params(FAMS[n])]]
        runs.append(("prefix", dict(sf.params("defaults"), maxoliters=k), use, k))
    return runs


def test_matrix_batch(clp):
    import torch
    runs = _matrix_batch_runs()
    assert any("T6_huge" in use for _, _, use, _ in runs) and any("T7_m1" in use for _, _, use, _ in runs)
    for g, P, use, k in runs:
        b = clp.MatrixBatchCLIPPER(_params(clp, P))
        probs = [dict(zip(("M", "C"), FAMS[n].dense()), u0=FAMS[n].u0) for n in use]

        def verify(n, s, door):
            what = "MatrixBatch.%s %s %s" % (door, n, g if k is None else "maxoliters=%d" % k)
            if k is None:
                check(s, oracle_ref(FAMS[n], g), what)
            else:
                check_prefix(s, FAMS[n], k, what)
            if n == "T6_huge":   # F > 2^31: round(F) clamped to m keeps every node
                assert s.score > 2.0 ** 31 and sorted(s.nodes) == list(range(FAMS[n].m)), what
        for n, s in zip(use, b.solve_many(probs)):
            verify(n, s, "solve_many")
        mm = max(FAMS[n].m for n in use)
        M = torch.zeros((len(use), mm, mm), dtype=torch.float64); Cm = torch.zeros_like(M)
        u0 = torch.zeros((len(use), mm), dtype=torch.float64)
        for q, n in enumerate(use):
            c = FAMS[n]; Md, Cd = c.dense()
            M[q, :c.m, :c.m] = torch.from_numpy(Md); Cm[q, :c.m, :c.m] = torch.from_numpy(Cd)
            u0[q, :c.m] = torch.from_numpy(c.u0)
        sols = b.solve_dense_dev(M.cuda(), Cm.cuda(), u0.cuda(), m=[FAMS[n].m for n in use])
        for n, s in zip(use, sols):
            verify(n, s, "solve_dense_dev")


# ---- scored batches ------------------------------------------------------------------------------------------------
def _batch_problems():
    from test_gpu_batch import _problems
    return _problems([64, 100, 257, 333], 900)


@pytest.mark.parametrize("door", ["solve_many", "solve_many_dev", "cuda_invariant"])
def test_scored_batch(clp, door):
    """the reference of batch problem p is the oracle fed the read-back of a single fp32 handle scored with p's inputs"""
    import torch
    import scipy.sparse as sp
    from test_gpu_batch import _euclid
    from test_gpu_custom_invariant import EUCLID_SRC
    sigma, eps = 0.015, 0.05
    probs = _batch_problems()
    for g in sf.T8_GRID:
        P = sf.params(g)
        if door == "cuda_invariant":
            b = clp.BatchCLIPPER(clp.invariants.CudaInvariant(EUCLID_SRC, (sigma, eps, 0.0)), _params(clp, P))
        else:
            b = clp.BatchCLIPPER(_euclid(clp, sigma, eps), _params(clp, P))
        if door == "solve_many_dev":
            d = probs[0]["D1"].shape[0]
            n1 = max(p["D1"].shape[1] for p in probs); n2 = max(p["D2"].shape[1] for p in probs)
            mm = max(p["A"].shape[0] for p in probs)
            D1 = torch.zeros((len(probs), d, n1), dtype=torch.float64); D2 = torch.zeros((len(probs), d, n2), dtype=torch.float64)
            A = torch.zeros((len(probs), mm, 2), dtype=torch.int32); U0 = torch.zeros((len(probs), mm), dtype=torch.float64)
            for q, p in enumerate(probs):
                D1[q, :, :p["D1"].shape[1]] = torch.from_numpy(np.ascontiguousarray(p["D1"]))
                D2[q, :, :p["D2"].shape[1]] = torch.from_numpy(np.ascontiguousarray(p["D2"]))
                A[q, :p["A"].shape[0]] = torch.from_numpy(np.ascontiguousarray(p["A"]))
                U0[q, :p["A"].shape[0]] = torch.from_numpy(p["u0"])
            sols = b.solve_many_dev(D1.cuda(), D2.cuda(), A.cuda(), U0.cuda(), n1=[p["D1"].shape[1] for p in probs],
                                    n2=[p["D2"].shape[1] for p in probs], m=[p["A"].shape[0] for p in probs])
        else:
            sols = b.solve_many(probs)
        for q, (p, s) in enumerate(zip(probs, sols)):
            c = clp.CLIPPER(_euclid(clp, sigma, eps), clp.Params())
            c.score_pairwise_consistency(p["D1"], p["D2"], p["A"])
            Mr = c.get_affinity_matrix(); np.fill_diagonal(Mr, 0); Cr = c.get_constraint_matrix(); np.fill_diagonal(Cr, 0)
            ref = sf.Case("batch%d" % q, "T8", sp.csr_matrix(Mr), sp.csr_matrix(Cr), p["u0"])
            if door == "solve_many":   # the read-back does not depend on the door
                r = ref.restate(P)
                assert r["margins"].robust, "problem %d %s: not robust %s" % (q, g, r["margins"].worst)
            check(s, oracle_ref(ref, g, key=("batch", q)), "%s problem %d %s" % (door, q, g))


# ---- clipperpy through the C++ shell -------------------------------------------------------------------------------
def test_clipperpy_shell(clp):
    lib = os.path.join(ROOT, "clipper_b200", "lib")
    if lib not in sys.path:
        sys.path.insert(0, lib)
    import clipperpy as cp
    rounding = {0: cp.Rounding.NONZERO, 1: cp.Rounding.DSD, 2: cp.Rounding.DSD_HEU}
    for name in ("T3_isolated", "T4_two_cliques", "T5_mixed", "T7_m129"):
        case = FAMS[name]
        for g in sf.grid_for(case, sf.DOOR_GRID + ("maxoliters1", "maxoliters2", "beta0.5_eps1e-3", "tolu0_tolF1e-3",
                                                    "tolu1e-2_tolF0", "nonzero")):
            P = sf.params(g)
            p = cp.Params()
            for k, v in P.items():
                setattr(p, k, rounding[v] if k == "rounding" else v)
            c = cp.CLIPPER(cp.invariants.EuclideanDistance(cp.invariants.EuclideanDistanceParams()), p)
            c.set_matrix_data(*case.dense())
            c.solve(case.u0)
            s = c.get_solution()
            o = oracle_ref(case, g)
            what = "clipperpy %s %s" % (name, g)
            assert s.ifinal == o.ifinal and list(s.nodes) == o.nodes.tolist(), what   # clipperpy has no counters
            assert abs(s.score - o.score) <= 2e-11 * abs(o.score), what
            assert np.abs(np.asarray(s.u) - o.u).max() <= 1e-10, what
