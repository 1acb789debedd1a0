"""Host-side conversion of MatrixBatchCLIPPER's inputs (clipper_b200.batch.matrices_to_csc), without a GPU: the CSC it
passes to clp_batch_solve_matrices must give the store set_matrix_data / set_sparse_matrix_data give."""
import numpy as np
import pytest
import scipy.sparse as sp

from clipper_b200.batch import matrices_to_csc


def _entries(colptr, rowidx, val):
    cols = np.repeat(np.arange(colptr.size - 1), np.diff(colptr))
    return list(zip(rowidx.tolist(), cols.tolist(), val.tolist()))


def _store_from_csc(m, cpM, riM, vM, cpC, riC, vC):
    """fp32 store bits (m x m, both triangles) and flags of clp_set_sparse_upper / the batched scatter: neutral -0.0,
    M entries as -|fp32(v)|, then the C entries equal to 1 clear the sign; flags 4 structure, 1 M < 0, 2 C not in {0, 1}"""
    S = np.full((m, m), -0.0, np.float32)
    flags = 0
    for (i, j, v) in _entries(cpM, riM, vM):
        if i < 0 or i >= j:
            flags |= 4; continue
        if v < 0.0:
            flags |= 1
        S[i, j] = S[j, i] = -abs(np.float32(v))
    for (i, j, v) in _entries(cpC, riC, vC):
        if i < 0 or i >= j:
            flags |= 4; continue
        if v == 0.0:
            continue
        if v != 1.0:
            flags |= 2
        S[i, j] = S[j, i] = abs(S[i, j])
    return S, flags


def _store_from_dense(M, Cm):
    """the same for set_matrix_data (encode_dense_panel_kernel): every upper pair stored as encode(M, C != 0)"""
    m = M.shape[0]
    S = np.full((m, m), -0.0, np.float32)
    flags = 0
    for i in range(m):
        for j in range(i + 1, m):
            mv, cv = M[i, j], Cm[i, j]
            if mv < 0.0:
                flags |= 1
            if cv != 0.0 and cv != 1.0:
                flags |= 2
            a = abs(np.float32(mv))
            S[i, j] = S[j, i] = a if cv != 0.0 else -a
    return S, flags


def test_dense_reads_the_strict_upper_triangle():
    M = np.array([[9.0, 0.5, 0.0], [7.0, 9.0, 0.25], [7.0, 7.0, 9.0]])
    Cm = np.array([[9.0, 1.0, 1.0], [7.0, 9.0, 0.0], [7.0, 7.0, 9.0]])
    m, cpM, riM, vM, cpC, riC, vC = matrices_to_csc(M, Cm)
    assert m == 3
    assert _entries(cpM, riM, vM) == [(0, 1, 0.5), (1, 2, 0.25)]
    assert _entries(cpC, riC, vC) == [(0, 1, 1.0), (0, 2, 1.0)]
    assert cpM.dtype == np.int64 and riM.dtype == np.int32 and vM.dtype == np.float64


def test_dense_keeps_c_values_and_nan_and_drops_negative_zero():
    M = np.zeros((4, 4)); Cm = np.zeros((4, 4))
    M[0, 1] = np.nan; M[0, 2] = -0.0; M[1, 3] = 0.75
    Cm[0, 1] = 0.5; Cm[0, 3] = np.nan; Cm[2, 3] = 1.0
    _, cpM, riM, vM, cpC, riC, vC = matrices_to_csc(M, Cm)
    eM = _entries(cpM, riM, vM)
    assert [(i, j) for i, j, _ in eM] == [(0, 1), (1, 3)] and np.isnan(eM[0][2]) and eM[1][2] == 0.75
    eC = _entries(cpC, riC, vC)
    assert [(i, j) for i, j, _ in eC] == [(0, 1), (0, 3), (2, 3)]
    assert eC[0][2] == 0.5 and np.isnan(eC[1][2]) and eC[2][2] == 1.0


def test_sparse_comes_out_sorted_with_lower_entries_kept():
    # rows of column 3 given out of order, one entry below the diagonal
    M = sp.csc_matrix((np.array([0.3, 0.1, 0.2]), np.array([2, 0, 3]), np.array([0, 0, 0, 0, 2, 3])), shape=(5, 5))
    Cm = sp.csr_matrix((np.array([1.0, 1.0]), (np.array([1, 0]), np.array([3, 3]))), shape=(5, 5))
    m, cpM, riM, vM, cpC, riC, vC = matrices_to_csc(M, Cm)
    assert m == 5
    assert _entries(cpM, riM, vM) == [(0, 3, 0.1), (2, 3, 0.3), (3, 4, 0.2)]
    L = sp.coo_matrix((np.array([0.4]), (np.array([4]), np.array([1]))), shape=(5, 5))
    _, cp2, ri2, v2, _, _, _ = matrices_to_csc(L, Cm)
    assert _entries(cp2, ri2, v2) == [(4, 1, 0.4)]   # passed through: the library refuses it
    assert _entries(cpC, riC, vC) == [(0, 3, 1.0), (1, 3, 1.0)]


def test_shapes_and_kinds_must_match():
    with pytest.raises(ValueError):
        matrices_to_csc(np.zeros((3, 3)), np.zeros((4, 4)))
    with pytest.raises(ValueError):
        matrices_to_csc(np.zeros((3, 4)), np.zeros((3, 4)))
    with pytest.raises(ValueError):
        matrices_to_csc(sp.csc_matrix((3, 3)), sp.csc_matrix((4, 4)))
    with pytest.raises(ValueError):
        matrices_to_csc(np.zeros((3, 3)), sp.csc_matrix((3, 3)))


@pytest.mark.parametrize("seed", range(6))
def test_csc_store_equals_dense_store(seed):
    """random dense (M, C): 0/1 constraints, sometimes invalid values (0.5, NaN, negative M); the store and the flags
    restated from the CSC equal those of set_matrix_data"""
    rng = np.random.default_rng(seed)
    m = int(rng.integers(2, 40))
    M = np.where(rng.random((m, m)) < 0.4, rng.random((m, m)), 0.0)
    M[rng.random((m, m)) < 0.05] = 1e-50            # non-zero double, zero in fp32
    M[rng.random((m, m)) < 0.05] = -0.0
    Cm = (rng.random((m, m)) < 0.5).astype(np.float64)
    if seed % 3 == 1:
        Cm[0, m - 1] = 0.5
    if seed % 3 == 2:
        Cm[0, 1] = np.nan
        M[0, m - 1] = -0.25
    S_csc, f_csc = _store_from_csc(*matrices_to_csc(M, Cm))
    S_dense, f_dense = _store_from_dense(M, Cm)
    assert S_csc.view(np.uint32).tolist() == S_dense.view(np.uint32).tolist()
    assert f_csc == f_dense
    # the single path reports structure, then M, then C: the first set bit in that order decides
    assert (f_csc & 1 != 0) == (seed % 3 == 2)
