"""The solver cases of tests/solver_families.py on the CPU: the numpy restatement equals the C oracle, every case the
GPU test uses is robust, every family keeps the edge it exists for, and the cases are deterministic."""
import math

import numpy as np
import pytest

import solver_families as sf

FAMS = sf.families()


def _pairs():
    out = [(n, g) for n, c in FAMS.items() for g in sf.grid_for(c, sf.FULL_GRID + ("dsd",))]
    return out


def _same_as_oracle(case, g, r, o):
    what = "%s %s" % (case.name, g)
    assert (r["ifinal"], r["n_evals"], r["n_inner"]) == (o.ifinal, o.n_evals, o.n_inner), what
    assert r["nodes"].tolist() == o.nodes.tolist(), what
    for a, b in ((r["d_final"], o.d_final), (r["score"], o.score)):
        assert (math.isnan(a) and math.isnan(b)) or a == b, (what, a, b)
    assert np.array_equal(np.isnan(r["u"]), np.isnan(o.u)), what
    ok = ~np.isnan(o.u)
    if ok.any():
        assert np.abs(r["u"][ok] - o.u[ok]).max() <= 1e-13, what
        assert r["u"].tobytes() == o.u.tobytes(), what   # the same additions in the same order
    if o.trace is not None:   # the oracle's rows past the last outer iteration are not written
        n = r["trace"].shape[0]
        assert np.array_equal(r["trace"][:, 2], o.trace[:n, 2]), what


@pytest.mark.parametrize("name,g", _pairs())
def test_restatement_equals_oracle_and_is_robust(name, g):
    case = FAMS[name]
    P = sf.params(g)
    r = case.restate(P)
    _, o = case.oracle(P, trace_cap=1000)
    _same_as_oracle(case, g, r, o)
    assert r["margins"].robust, "%s %s: %s" % (name, g, r["margins"].worst)


def test_segmented_handover_case():
    case = sf.big_case()
    assert case.m == 27649
    for g in case.grid:
        P = sf.params(g)
        r = case.restate(P)
        _same_as_oracle(case, g, r, case.oracle(P)[1])
        assert r["margins"].robust, (g, r["margins"].worst)


@pytest.mark.parametrize("f32", [False, True])
@pytest.mark.parametrize("name,m", sf.SCORED)
def test_scored_cases_are_robust(name, m, f32):
    """T8 on the oracle's scores and on the same scores rounded to fp32, for the parameter sets every door runs"""
    case = sf.scored_case(name, m, f32)
    for g in sf.T8_GRID:
        P = sf.params(g)
        r = case.restate(P)
        assert r["margins"].robust, "%s %s: %s" % (case.name, g, r["margins"].worst)
        if m <= 700:
            _same_as_oracle(case, g, r, case.oracle(P)[1])


@pytest.mark.parametrize("name", list(FAMS))
def test_family_claims(name):
    case = FAMS[name]
    g = case.grid[0] if case.grid else "defaults"
    desc, claim = case.claim
    assert claim(case, case.restate(sf.params(g))), "%s: %s" % (name, desc)


def test_exclusions_are_not_robust():
    """every excluded pair is excluded for the reason given: the restatement finds a decision that is not robust"""
    for (name, g), why in sf.EXCLUDE.items():
        r = FAMS[name].restate(sf.params(g))
        assert not r["margins"].robust and why, (name, g)


def test_every_family_is_present():
    fams = {c.family for c in FAMS.values()} | {sf.big_case().family}
    assert fams >= {"T1", "T2", "T3", "T4", "T5", "T6", "T7", "T9", "U"}
    assert sorted(c.m for c in FAMS.values() if c.family == "T7") == [1, 2, 31, 32, 33, 127, 128, 129, 4096]


def test_cases_are_deterministic():
    again = sf.families()
    for n, c in FAMS.items():
        d = again[n]
        assert (c.Mh != d.Mh).nnz == 0 and (c.Ch != d.Ch).nnz == 0 and c.u0.tobytes() == d.u0.tobytes(), n


def test_weights_are_fp32_exact():
    """fp32 and fp64 storage keep the same matrix, so one oracle run is the reference for both"""
    for n, c in FAMS.items():
        assert np.array_equal(sf.f32(c.Mh.data), c.Mh.data) and np.all(c.Mh.data >= 0), n
        assert np.all(c.Ch.data == 1.0), n


def test_node_count_is_defined():
    """round(F) is clamped to [0, m] before the conversion and NaN keeps no node: F > 2^31 keeps all m nodes, u0 = 0
    (F NaN) keeps none.  (The reference's (int)std::round(F) is undefined in both cases.)"""
    huge = FAMS["T6_huge"]
    _, o = huge.oracle(sf.params("short"))
    assert o.score > 2.0 ** 31 and o.nodes.size == huge.m
    assert sorted(o.nodes.tolist()) == list(range(huge.m))
    zero = FAMS["U_zero"]
    _, o = zero.oracle(sf.params("defaults"))
    assert math.isnan(o.score) and o.nodes.size == 0 and np.all(np.isnan(o.u))
    assert (o.ifinal, o.n_inner, o.n_evals) == (0, 200, 200)
