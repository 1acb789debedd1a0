"""The numpy restatement of clp_correspondences (tests/knn_oracle.py) against scipy's kd-tree on tie-free data, against
the reference's loop written out in Python, and on hand-built cases with ties, NaN and empty clouds.  No GPU."""
import numpy as np
import pytest

import knn_oracle as ko


def _pair(rng, d, n1, n2):
    return rng.standard_normal((d, n1)), rng.standard_normal((d, n2))


@pytest.mark.parametrize("d", [3, 33])
@pytest.mark.parametrize("knn", [1, 5])
def test_agrees_with_ckdtree(d, knn):
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(10 + d + knn)
    D1, D2 = _pair(rng, d, 700, 900)
    dist, idx = cKDTree(D2.T).query(D1.T, k=knn)
    dist, idx = dist.reshape(700, knn), idx.reshape(700, knn)
    oi, osd = ko.neighbours(D1, D2, knn)
    assert np.array_equal(oi, idx)
    np.testing.assert_allclose(np.sqrt(osd), dist, rtol=1e-12, atol=0)
    # tie-free: consecutive neighbours and the radius are far apart relative to rounding
    assert np.all(np.diff(osd, axis=1) > 1e-9 * osd[:, 1:])
    r = float(np.median(dist))
    keep = dist <= r
    assert np.all(np.abs(dist - r) > 1e-9)
    A = ko.correspondences(D1, D2, knn, r, False)
    ii, rr = np.nonzero(keep)
    assert np.array_equal(A, np.stack([ii, idx[ii, rr]], axis=1))


@pytest.mark.parametrize("enforce", [False, True])
@pytest.mark.parametrize("knn", [1, 3, 7])
def test_matches_reference_loop(enforce, knn):
    rng = np.random.default_rng(knn)
    D1, D2 = _pair(rng, 3, 40, 30)
    for radius in (np.inf, 1.0, 0.5):
        assert np.array_equal(ko.correspondences(D1, D2, knn, radius, enforce),
                              ko.correspondences_loop(D1, D2, knn, radius, enforce))


def test_duplicate_points_prefer_lower_index():
    D2 = np.array([[1.0, 0.0, 1.0, 0.0]])        # columns 1 and 3 coincide, as do 0 and 2
    D1 = np.array([[0.0, 1.0]])
    A = ko.correspondences(D1, D2, 2, np.inf, False)
    assert A.tolist() == [[0, 1], [0, 3], [1, 0], [1, 2]]
    assert np.array_equal(A, ko.correspondences_loop(D1, D2, 2, np.inf, False))


def test_integer_lattice_ties():
    g = np.arange(4.0)
    P = np.array(np.meshgrid(g, g, g, indexing="ij")).reshape(3, -1)   # 64 points, many equal distances
    for knn in (1, 6, 27):
        for enforce in (False, True):
            A = ko.correspondences(P + 0.5, P, knn, np.inf, enforce)
            assert np.array_equal(A, ko.correspondences_loop(P + 0.5, P, knn, np.inf, enforce))
    # the query (0.5, 0.5, 0.5) has 8 candidates at sd 0.75: the 6 lowest indices of them win
    i0 = ko.neighbours(P[:, :1] + 0.5, P, 6)[0][0]
    eight = [j for j in range(64) if np.allclose(np.abs(P[:, j] - 0.5), 0.5)]
    assert i0.tolist() == sorted(eight)[:6]


def test_one_to_one_equal_sd_keeps_smallest_c0():
    D2 = np.array([[0.0, 10.0]])
    D1 = np.array([[1.0, -1.0, 1.0, 9.0, 11.0]])   # c0 0, 1, 2 all at sd 1 from c1 0; c0 3, 4 at sd 1 from c1 1
    A = ko.correspondences(D1, D2, 1, np.inf, True)
    assert A.tolist() == [[0, 0], [3, 1]]
    D1b = np.array([[2.0, 1.0, -1.0]])              # least sd wins over the order of pushes
    assert ko.correspondences(D1b, D2, 1, np.inf, True).tolist() == [[1, 0]]


def test_knn_above_n2_is_clamped():
    rng = np.random.default_rng(3)
    D1, D2 = _pair(rng, 2, 5, 3)
    A = ko.correspondences(D1, D2, 10, np.inf, False)
    assert A.shape == (15, 2)
    assert np.array_equal(A, ko.correspondences_loop(D1, D2, 10, np.inf, False))


def test_radius_zero_inf_nan():
    D1 = np.array([[0.0, 1.0, 2.0]])
    D2 = np.array([[1.0, 5.0]])
    assert ko.correspondences(D1, D2, 1, 0.0, False).tolist() == [[1, 0]]
    assert ko.correspondences(D1, D2, 2, np.inf, False).shape == (6, 2)
    assert ko.correspondences(D1, D2, 2, np.nan, False).shape == (0, 2)
    assert ko.correspondences(D1, D2, 2, np.nan, True).shape == (0, 2)
    # radius * radius as the reference computes it: a negative radius acts as its magnitude
    assert np.array_equal(ko.correspondences(D1, D2, 1, -1.0, False), ko.correspondences(D1, D2, 1, 1.0, False))


def test_nan_coordinates_are_never_neighbours():
    D2 = np.array([[0.0, np.nan, 2.0], [0.0, 0.0, 0.0]])
    D1 = np.array([[0.9, np.nan], [0.0, 0.0]])
    idx, sd = ko.neighbours(D1, D2, 3)
    assert idx[0].tolist() == [0, 2, -1]          # candidate 1 has a NaN coordinate
    assert idx[1].tolist() == [-1, -1, -1]        # so does query 1
    A = ko.correspondences(D1, D2, 3, np.inf, False)
    assert A.tolist() == [[0, 0], [0, 2]]
    assert np.array_equal(A, ko.correspondences_loop(D1, D2, 3, np.inf, False))


def test_empty_and_single_clouds():
    one = np.zeros((3, 1))
    none = np.zeros((3, 0))
    assert ko.correspondences(none, one, 1, np.inf, False).shape == (0, 2)
    assert ko.correspondences(one, none, 1, np.inf, True).shape == (0, 2)
    assert ko.correspondences(one, one, 4, np.inf, False).tolist() == [[0, 0]]
    assert ko.correspondences(one, one, 1, 0.0, True).tolist() == [[0, 0]]


def test_accumulation_order_is_sequential():
    # a value where (a + b) + c differs from a + (b + c): the restatement accumulates k = 0 .. d-1 in order
    D1 = np.array([[1.0], [2.0 ** -27], [2.0 ** -27], [2.0 ** -27], [2.0 ** -27]])
    D2 = np.zeros((5, 1))
    s = ko.squared_distances(D1, D2)[0, 0]
    assert s == 1.0                                # every 2^-54 is lost on its own
    assert s != 1.0 + 4 * 2.0 ** -54               # the small terms summed first would survive
    assert ko.correspondences_loop(D1, D2, 1, 1.0, False).tolist() == [[0, 0]]
    assert ko.correspondences(D1, D2, 1, 1.0, False).tolist() == [[0, 0]]
