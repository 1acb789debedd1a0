"""The argument checks of utils.distance_based_correspondences_many(_dev) raise TypeError or ValueError before the
library or a device is touched (no GPU needed): the library loader and the batch cache are replaced by functions that
fail the test if they are reached."""
import numpy as np
import pytest


@pytest.fixture
def env(monkeypatch):
    import torch
    import clipper_b200 as clipperpy
    from clipper_b200 import _capi, api

    def touched(*a, **k):
        raise AssertionError("the library was reached")

    monkeypatch.setattr(api, "_knn_batch", touched)
    monkeypatch.setattr(_capi, "load", touched)
    return torch, clipperpy.utils


def _batch(torch, B=2, d=3, n1=5, n2=6):
    """CPU tensors of a batch of the right dtype and shapes"""
    return torch.zeros((B, d, n1), dtype=torch.float64), torch.zeros((B, d, n2), dtype=torch.float64)


def test_dev_cpu_tensors(env):
    torch, u = env
    D1, D2 = _batch(torch)
    with pytest.raises(ValueError, match="CUDA"):
        u.distance_based_correspondences_many_dev(D1, D2, 1, 1.0, False)


def test_dev_dtypes(env):
    torch, u = env
    D1, D2 = _batch(torch)
    with pytest.raises(TypeError):
        u.distance_based_correspondences_many_dev(D1.float(), D2, 1, 1.0, False)
    with pytest.raises(TypeError):
        u.distance_based_correspondences_many_dev(D1, D2.to(torch.int32), 1, 1.0, False)
    with pytest.raises(TypeError):
        u.distance_based_correspondences_many_dev(D1.numpy(), D2, 1, 1.0, False)


def test_dev_ranks_and_shapes(env):
    torch, u = env
    D1, D2 = _batch(torch)
    for a, b in ((D1[0], D2[0]), (D1, D2[0]), (D1, D2[:, :2]), (D1, D2[:1]), (D1[:0], D2[:0])):
        with pytest.raises(ValueError):
            u.distance_based_correspondences_many_dev(a, b, 1, 1.0, False)


def test_dev_sizes_and_knn(env):
    torch, u = env
    D1, D2 = _batch(torch)
    for kw in (dict(n1=[6, 5]), dict(n2=[7, 1]), dict(n1=[-1, 5]), dict(n2=[3]), dict(n1=[1, 2, 3])):
        with pytest.raises(ValueError):
            u.distance_based_correspondences_many_dev(D1, D2, 1, 1.0, False, **kw)
    for knn in (0, -3):
        with pytest.raises(ValueError):
            u.distance_based_correspondences_many_dev(D1, D2, knn, 1.0, False)
    with pytest.raises(ValueError):   # d = 0
        u.distance_based_correspondences_many_dev(D1[:, :0], D2[:, :0], 1, 1.0, False)


def test_host_checks(env):
    _, u = env
    X = np.zeros((3, 4))
    assert u.distance_based_correspondences_many([], [], 1, 1.0, False) == []
    with pytest.raises(ValueError):   # lengths differ
        u.distance_based_correspondences_many([X, X], [X], 1, 1.0, False)
    with pytest.raises(TypeError):    # float32
        u.distance_based_correspondences_many([X.astype(np.float32)], [X], 1, 1.0, False)
    with pytest.raises(TypeError):    # a list, not an array
        u.distance_based_correspondences_many([X.tolist()], [X], 1, 1.0, False)
    with pytest.raises(ValueError):   # d differs within a pair and across pairs
        u.distance_based_correspondences_many([X], [np.zeros((2, 4))], 1, 1.0, False)
    with pytest.raises(ValueError):
        u.distance_based_correspondences_many([X, np.zeros((2, 4))], [X, np.zeros((2, 4))], 1, 1.0, False)
    with pytest.raises(ValueError):   # not 2-D
        u.distance_based_correspondences_many([np.zeros(3)], [X], 1, 1.0, False)
    with pytest.raises(ValueError):
        u.distance_based_correspondences_many([X], [X], 0, 1.0, False)
