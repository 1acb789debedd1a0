"""CPU checks of the matrix families of tests/test_gpu_exact_products.py: the host restatements of the packed gate, the
packed row encoding and the segmentation behave as DESIGN.md section 2 describes, and every family contains the
structures it is meant to put in front of the kernels."""
import numpy as np
import pytest

import packed_families as pf
from fixtures import bytes_per_pass


def _case(vals, cvals=None, m=40):
    vals = np.asarray(vals, np.float64)
    n = vals.size
    return pf.Case("t", m, np.zeros(n, np.int64), np.arange(1, n + 1), vals,
                   np.ones(n) if cvals is None else np.asarray(cvals, np.float64))


def test_pack_gate_restatement():
    assert pf.pack_gate(_case([1.0, 2.0 ** -14])) == (True, 112)                  # code 1 = 2^-14 x 1.0
    assert pf.pack_gate(_case([1.0, 2.0 ** -15]))[0] is False                     # one binade below
    assert pf.pack_gate(_case([2.0 - 2.0 ** -23, 2.0 ** -14])) == (True, 112)
    assert pf.pack_gate(_case([2.0 ** 20, 2.0 ** 6])) == (True, 132)
    assert pf.pack_gate(_case([2.0 ** 20, 2.0 ** 5]))[0] is False
    assert pf.pack_gate(_case([2.0 ** -115, 2.0 ** -126])) == (True, 0)           # b = 0: every normal value fits
    assert pf.pack_gate(_case([2.0 ** -115, 2.0 ** -130]))[0] is False            # fp32 subnormal
    assert pf.pack_gate(_case([1.0, 0.5], [1.0, 0.0]))[0] is False                # (M > 0, C = 0)
    assert pf.pack_gate(_case([1.0, 0.0], [1.0, 1.0]))[0] is False                # (M = 0, C = 1)
    assert pf.pack_gate(_case([])) == (True, 0)                                   # nothing kept: all fillers


@pytest.mark.parametrize("case", pf.pair_cases()[:3], ids=lambda c: c.name)
def test_pack_row_round_trip_f1(case):
    """every whole row of F1 encodes with deltas of 1..31 and decodes to its own columns and fp32 values"""
    packed, bias = pf.pack_gate(case)
    assert packed
    Mh, _, K = case.stored(True)
    m = case.m
    deltas = []
    for r in range(m):
        cols = K.indices[K.indptr[r]:K.indptr[r + 1]]
        vals = np.asarray(Mh[r, cols].todense()).ravel()
        words, delta = pf.pack_row(cols, vals, m, bias)
        c2, v2 = pf.unpack_row(words, bias)
        assert np.array_equal(c2, cols) and np.array_equal(v2, vals.astype(np.float32).astype(np.float64))
        deltas.append(delta)
    lens = np.diff(K.indptr)
    if case.name.startswith("F1_full"):
        # delta 1 everywhere except the step over the diagonal
        assert np.all(lens == m - 1) and all(np.count_nonzero(d != 1) <= 1 and d.max() <= 2 for d in deltas)
        return
    assert m % 16 in (1, 15)
    assert any(31 in d for d in deltas), "no delta of exactly 31"
    assert any(np.any(np.convolve(d == 16, np.ones(8), "valid") == 8) for d in deltas), "no chain of delta-16 steps"
    rows = [K.indices[K.indptr[r]:K.indptr[r + 1]].tolist() for r in range(m)]
    assert [] in rows                                      # only fillers
    assert [0] in rows and [m - 1] in rows                 # only column 0, only column m - 1
    last = 16 * (m // 16)
    assert any(r and min(r) >= last for r in rows[:5])     # only the partial last window


def test_f2_window_contents():
    cases = {c.name: c for top in pf.F2_MAX for c in pf.f2_variants(top)}
    for top, X in pf.F2_MAX.items():
        base = cases["F2_%s_in" % top]
        packed, b = pf.pack_gate(base)
        assert packed and base.mval.max() == X
        a = base.mval.astype(np.float32)
        assert np.array_equal(a.astype(np.float64), base.mval)        # exact fp32 values
        field, mant = pf.f32_field(a), a.view(np.uint32) & 0x7FFFFF
        assert np.any((field == b + 1) & (mant == 0)) and np.any((field == b + 1) & (mant == 0x7FFFFF))
        ehi = int(pf.f32_field(X))
        assert set(range(b + 1, ehi + 1)) <= set(field.tolist())      # every admitted binade
        if b > 0:
            assert ehi - b == 15                                       # the highest binade is code 15
        for v in ("below", "subnormal", "mc0", "m0c1"):
            if v == "below" and b == 0:
                assert "F2_%s_below" % top not in cases
                continue
            assert pf.pack_gate(cases["F2_%s_%s" % (top, v)])[0] is False, (top, v)
    sub = cases["F2_1_subnormal"].mval
    assert np.any((sub.astype(np.float32) != 0) & (pf.f32_field(sub) == 0))


def test_f3_imbalance_contents():
    for m in (27648, 27649):
        case, heavy, empty = pf.f3_imbalance(m)
        _, _, K = case.stored(True)
        lens = np.diff(K.indptr)
        assert np.all(lens[empty] == 0) and abs(empty.size / m - 0.6) < 0.01
        active = m - empty.size
        assert np.all(lens[heavy] == active - 1) and abs(heavy.size / m - 0.01) < 0.001
        rest = np.setdiff1d(np.arange(m), np.concatenate([heavy, empty]))
        assert 8 <= (lens[rest] - heavy.size).mean() <= 12
        assert pf.pack_gate(case)[0]


def test_f4_straddles_the_boundaries():
    for m in pf.F4_M:
        case = pf.f4_edges(m)
        _, _, K = case.stored(True)
        cols = set(K.indices.tolist())
        for bnd in (128, 2048, 4096):
            if bnd + 1 < m:
                assert {bnd - 1, bnd} <= cols
        assert m - 1 in cols
        nseg, W = pf.seg_plan(m)
        assert W % 128 == 0 and W <= pf.SEG_MAX and nseg * W >= m and (nseg - 1) * W < m + 128 * nseg


@pytest.mark.parametrize("case", [pf.f1_deltas(641), pf.f4_edges(129), pf.f5_small(17), pf.f5_empty(100)], ids=lambda c: c.name)
def test_bytes_per_pass_dense_equals_sparse(case):
    _, _, K = case.stored(True)
    for packed in (True, False):
        assert bytes_per_pass(K, packed) == bytes_per_pass(K.toarray(), packed)


def test_predicted_modes():
    K = pf.f5_empty(1000).stored(True)[2]
    assert pf.predict_mode(4, 1000, K, True, True) == 6          # all fillers: 63 words per row, far below m^2 / 2
    dense = pf.f1_full(161).stored(True)[2]
    assert pf.predict_mode(4, 161, dense, True, True) == 2       # a full matrix keeps the dense sweep
    assert pf.predict_mode(6, 27649, K, True, True) == 3         # the vector does not fit shared memory
