"""The tensor checks of BatchCLIPPER.solve_many_dev / max_clique_many_dev and CLIPPER.score_pairwise_consistency_dev
raise TypeError or ValueError before the library or a device is touched (no GPU needed): the objects here have no
library handle, so any call that got that far would fail differently."""
import pytest


@pytest.fixture(scope="module")
def env():
    import torch
    import clipper_b200 as clipperpy
    b = object.__new__(clipperpy.BatchCLIPPER)
    b._device = 0
    b._invariant = clipperpy.invariants.EuclideanDistance(clipperpy.invariants.EuclideanDistanceParams())
    c = object.__new__(clipperpy.CLIPPER)
    c._device = 0
    c._invariant = b._invariant
    return torch, b, c


def _batch(torch, B=2, d=3, n1=5, n2=6, m=4):
    """CPU tensors of a batch of the right dtypes and shapes"""
    D1 = torch.zeros((B, d, n1), dtype=torch.float64)
    D2 = torch.zeros((B, d, n2), dtype=torch.float64)
    A = torch.zeros((B, m, 2), dtype=torch.int32)
    u0 = torch.zeros((B, m), dtype=torch.float64)
    return D1, D2, A, u0


def test_cpu_tensors(env):
    torch, b, c = env
    D1, D2, A, u0 = _batch(torch)
    with pytest.raises(ValueError, match="CUDA"):
        b.solve_many_dev(D1, D2, A, u0)
    with pytest.raises(ValueError, match="CUDA"):
        b.max_clique_many_dev(D1, D2, None)
    with pytest.raises(ValueError, match="CUDA"):
        c.score_pairwise_consistency_dev(D1[0], D2[0], A[0])


def test_dtypes(env):
    torch, b, c = env
    D1, D2, A, u0 = _batch(torch)
    with pytest.raises(TypeError):
        b.solve_many_dev(D1.float(), D2.float(), A, u0)
    with pytest.raises(TypeError):
        b.max_clique_many_dev(D1, D2, A.long())
    with pytest.raises(TypeError):
        b.solve_many_dev(D1.numpy(), D2, A, u0)
    with pytest.raises(TypeError):
        c.score_pairwise_consistency_dev(D1[0].float(), D2[0])
    with pytest.raises(TypeError):
        c.score_pairwise_consistency_dev(D1[0], D2[0], A[0].long())


def test_ranks_and_shapes(env):
    torch, b, c = env
    D1, D2, A, u0 = _batch(torch)
    with pytest.raises(ValueError):
        b.solve_many_dev(D1[0], D2[0], A, u0)
    with pytest.raises(ValueError):
        b.max_clique_many_dev(D1, D2, A[0])
    with pytest.raises(ValueError):  # d differs
        b.max_clique_many_dev(D1, D2[:, :2], A)
    with pytest.raises(ValueError):  # B differs
        b.max_clique_many_dev(D1, D2, A[:1])
    with pytest.raises(ValueError):
        c.score_pairwise_consistency_dev(D1, D2)


def test_sizes_beyond_padding(env):
    torch, b, c = env
    D1, D2, A, u0 = _batch(torch)
    for kw in (dict(n1=[5, 6]), dict(n2=[7, 1]), dict(m=[5, 4]), dict(n1=[0, 5]), dict(m=[4])):
        with pytest.raises(ValueError):
            b.max_clique_many_dev(D1, D2, A, **kw)
    with pytest.raises(ValueError):  # m needs A
        b.max_clique_many_dev(D1, D2, None, m=[1, 1])
    with pytest.raises(ValueError):  # u0 shorter than the problems
        b.solve_many_dev(D1, D2, A, u0[:, :3])
    with pytest.raises(ValueError):  # all-to-all: 5 x 6 associations, u0 holds 4
        b.solve_many_dev(D1, D2, None, u0)
