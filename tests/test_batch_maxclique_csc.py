"""Host-side conversion of the graphs of maxclique_many to the strictly-upper CSC pattern of the C-ABI, and its
validation.  No GPU is needed."""
import numpy as np
import pytest
import scipy.sparse as sp


def _dense_from_csc(m, colptr, rowidx):
    A = np.zeros((m, m), dtype=bool)
    for c in range(m):
        for r in rowidx[colptr[c]:colptr[c + 1]]:
            A[r, c] = True
    return A


def _check(m, colptr, rowidx):
    assert colptr.dtype == np.int64 and rowidx.dtype == np.int32
    assert colptr.shape == (m + 1,) and colptr[0] == 0 and colptr[-1] == rowidx.size
    assert np.all(np.diff(colptr) >= 0)
    for c in range(m):
        rows = rowidx[colptr[c]:colptr[c + 1]]
        assert np.all(rows < c) and np.all(rows >= 0) and np.all(np.diff(rows) > 0)


@pytest.mark.parametrize("seed", range(5))
def test_dense_and_sparse_agree(built, seed):
    from clipper_b200.batch import graph_to_csc
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 70))
    G = rng.random((n, n)) * (rng.random((n, n)) < 0.3)
    G[rng.random((n, n)) < 0.05] = -1.5  # negative entries are edges too
    want = np.triu(G != 0, 1)
    m, cp, ri = graph_to_csc(G)
    _check(m, cp, ri)
    assert m == n and np.array_equal(_dense_from_csc(m, cp, ri), want)
    for fmt in (sp.csr_matrix, sp.csc_matrix, sp.coo_matrix):
        m2, cp2, ri2 = graph_to_csc(fmt(G))
        assert m2 == n and np.array_equal(cp2, cp) and np.array_equal(ri2, ri)


def test_only_the_upper_triangle_counts(built):
    from clipper_b200.batch import graph_to_csc
    G = np.zeros((4, 4))
    G[2, 0] = G[3, 1] = 1.0   # lower triangle: ignored
    np.fill_diagonal(G, 5.0)  # diagonal: ignored
    G[0, 3] = 2.0
    m, cp, ri = graph_to_csc(G)
    assert m == 4 and cp.tolist() == [0, 0, 0, 0, 1] and ri.tolist() == [0]
    # boolean and integer inputs, NaN is nonzero
    assert graph_to_csc(G != 0)[1].tolist() == cp.tolist()
    H = np.zeros((3, 3)); H[0, 1] = np.nan
    assert graph_to_csc(H)[2].tolist() == [0]


def test_sparse_explicit_zeros_and_duplicates(built):
    from clipper_b200.batch import graph_to_csc
    # an explicit zero is not an edge; duplicates that cancel are not an edge; duplicates that add up are one edge
    S = sp.coo_matrix((np.array([0.0, 1.0, -1.0, 0.5, 0.5]), (np.array([0, 0, 0, 1, 1]), np.array([1, 2, 2, 3, 3]))),
                      shape=(4, 4))
    m, cp, ri = graph_to_csc(S)
    assert m == 4 and cp.tolist() == [0, 0, 0, 0, 1] and ri.tolist() == [1]


def test_validation(built):
    from clipper_b200.batch import graph_to_csc
    with pytest.raises(ValueError):
        graph_to_csc(np.zeros((3, 4)))
    with pytest.raises(ValueError):
        graph_to_csc(np.zeros(5))
    with pytest.raises(ValueError):
        graph_to_csc(sp.csr_matrix((2, 3)))
    with pytest.raises(ValueError):
        graph_to_csc(np.zeros((0, 0)))
    m, cp, ri = graph_to_csc(np.zeros((1, 1)))
    assert m == 1 and cp.tolist() == [0, 0] and ri.size == 0
