"""The argument checks of utils.estimate_rigid_transform(_many)(_dev) raise TypeError or ValueError before the library
or a device is touched (no GPU needed): the library loader and the kept handle and batch are replaced by functions that
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
    monkeypatch.setattr(api, "_knn_handle", touched)
    monkeypatch.setattr(_capi, "load", touched)
    return torch, clipperpy.utils


def _host(d=3, n=5):
    return np.zeros((d, n)), np.zeros((d, n)), np.zeros((n, 2), np.int32)


def test_host_dtypes(env):
    _, u = env
    D1, D2, A = _host()
    with pytest.raises(TypeError):
        u.estimate_rigid_transform(D1.astype(np.float32), D2, A)
    with pytest.raises(TypeError):
        u.estimate_rigid_transform(D1, D2, A.astype(np.int64))
    with pytest.raises(TypeError):
        u.estimate_rigid_transform(D1, D2, A, rows=[0.5, 1.0])
    with pytest.raises(TypeError):
        u.estimate_rigid_transform_many([D1], [D2.astype(np.float32)], [A])


def test_host_shapes(env):
    _, u = env
    D1, D2, A = _host()
    for a, b, c in ((D1[0], D2, A), (D1, D2[:2], A), (D1, D2, A[:, :1]), (D1, D2, A.reshape(-1))):
        with pytest.raises(ValueError):
            u.estimate_rigid_transform(a, b, c)
    with pytest.raises(ValueError):
        u.estimate_rigid_transform(D1, D2, A, rows=[2 ** 31])
    with pytest.raises(ValueError):
        u.estimate_rigid_transform_many([D1, D1], [D2], [A, A])
    with pytest.raises(ValueError):
        u.estimate_rigid_transform_many([D1], [D2], [A], rows=[None, None])
    with pytest.raises(ValueError):
        u.estimate_rigid_transform_many([D1, D1[:2]], [D2, D2[:2]], [A, A])
    assert u.estimate_rigid_transform_many([], [], []) == ([], [])


def test_dev_types_and_devices(env):
    torch, u = env
    D1, D2 = torch.zeros((3, 5), dtype=torch.float64), torch.zeros((3, 5), dtype=torch.float64)
    A = torch.zeros((5, 2), dtype=torch.int32)
    with pytest.raises(TypeError):
        u.estimate_rigid_transform_dev(D1.float(), D2, A)
    with pytest.raises(TypeError):
        u.estimate_rigid_transform_dev(D1, D2, A.long())
    with pytest.raises(TypeError):
        u.estimate_rigid_transform_dev(D1.numpy(), D2, A)
    with pytest.raises(ValueError):
        u.estimate_rigid_transform_dev(D1[0], D2, A)
    with pytest.raises(ValueError):
        u.estimate_rigid_transform_dev(D1, D2, A[:, :1])
    with pytest.raises(ValueError, match="CUDA"):
        u.estimate_rigid_transform_dev(D1, D2, A)


def test_many_dev_checks(env):
    torch, u = env
    D1, D2 = torch.zeros((2, 3, 5), dtype=torch.float64), torch.zeros((2, 3, 5), dtype=torch.float64)
    A = torch.zeros((2, 5, 2), dtype=torch.int32)
    with pytest.raises(ValueError, match="CUDA"):
        u.estimate_rigid_transform_many_dev(D1, D2, A)
    with pytest.raises(ValueError):
        u.estimate_rigid_transform_many_dev(D1.numpy(), D2, A)
