"""The persistent screened scoring kernel (score_tile_kernel_runs: fp32 storage, Euclidean d = 2, 3 and PointNormal)
against the unscreened kernel of an fp64-storage handle, which scores every pair in fp64 one tile per CTA: the fp32
store must be the fp32 rounding of the fp64 store bit for bit, with the same constraint matrix.  The sizes sit at the
edges of the kernel's work split: 1 to 33 rows, a 128-column tile and one past it, a 4096-column segment and one past
it, sizes with more work units than resident CTAs, and mode-3 (column-segmented) sizes.  A handle scored at a larger m and then at a smaller one must hold what a
fresh handle holds: no stale elements, counts or compact copy."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SIZES = [1, 2, 31, 33, 127, 128, 129, 255, 257, 1023, 1025, 4095, 4096, 4097]


@pytest.fixture(scope="module")
def clp(built):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import clipper_b200 as clipperpy
    return clipperpy


def _problem(kind, d, m, seed=7):
    """random associations over point sets with an inlier core, so that about a tenth of the pairs are kept"""
    rng = np.random.default_rng(seed + m)
    n = max(4, int(np.ceil(np.sqrt(m))) + 3)
    P = rng.uniform(-1.0, 1.0, (d, n))
    if kind == "pn":
        N = rng.normal(size=(3, n)); N /= np.linalg.norm(N, axis=0)
        Q = rng.normal(size=(3, n)); Q /= np.linalg.norm(Q, axis=0)
        D1 = np.vstack([P, N]); D2 = np.vstack([P + rng.normal(scale=0.01, size=P.shape), Q])
    else:
        D1 = P; D2 = P + rng.normal(scale=0.01, size=P.shape)
    A = np.stack([rng.integers(0, n, m), rng.integers(0, n, m)], axis=1).astype(np.int32)
    A[: m // 3, 1] = A[: m // 3, 0]  # a consistent core
    return np.asfortranarray(D1), np.asfortranarray(D2), np.asfortranarray(A)


def _invariant(clp, kind):
    if kind == "pn":
        ip = clp.invariants.PointNormalDistanceParams()
        ip.sigp, ip.epsp, ip.sign, ip.epsn = 0.5, 0.3, 0.5, 0.5
        return clp.invariants.PointNormalDistance(ip)
    ip = clp.invariants.EuclideanDistanceParams()
    ip.sigma, ip.epsilon = 0.05, 0.1
    return clp.invariants.EuclideanDistance(ip)


def _handle(clp, kind, storage, mode=None):
    c = clp.CLIPPER(_invariant(clp, kind), clp.Params(), storage=storage)
    if mode is not None:
        c.set_dense_mode(mode)
    return c


def _matrices(c):
    return c.get_affinity_matrix(), c.get_constraint_matrix()


def _assert_rounding_of(M32, C32, M64, C64):
    assert np.array_equal(C32, C64)
    assert np.array_equal(M32.astype(np.float32).view(np.uint32), M64.astype(np.float32).view(np.uint32))


@pytest.mark.parametrize("kind,d", [("eu", 2), ("eu", 3), ("pn", 3)])
@pytest.mark.parametrize("m", SIZES)
def test_screened_store_is_fp32_rounding_of_fp64(clp, kind, d, m):
    D1, D2, A = _problem(kind, d, m)
    c32 = _handle(clp, kind, 0); c32.score_pairwise_consistency(D1, D2, A)
    c64 = _handle(clp, kind, 1); c64.score_pairwise_consistency(D1, D2, A)
    _assert_rounding_of(*_matrices(c32), *_matrices(c64))
    assert c32.count_nonzeros() == c64.count_nonzeros()


@pytest.mark.parametrize("kind,d", [("eu", 3), ("pn", 3)])
def test_screened_store_column_segmented(clp, kind, d):
    """mode 3 cuts 4096-column segments: the per-(segment, row) counts of the scoring kernel feed the build"""
    m = 9000 if kind == "pn" else 27649
    D1, D2, A = _problem(kind, d, m)
    c32 = _handle(clp, kind, 0, mode=3); c32.score_pairwise_consistency(D1, D2, A)
    c64 = _handle(clp, kind, 1, mode=3); c64.score_pairwise_consistency(D1, D2, A)
    assert c32.count_nonzeros() == c64.count_nonzeros()
    if m <= 10000:
        _assert_rounding_of(*_matrices(c32), *_matrices(c64))


@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("mode,m", [(None, 8000), (3, 9000)])
def test_screened_store_more_units_than_ctas(clp, d, mode, m):
    """more work units than resident CTAs, so CTAs draw several units and reload the row side between row blocks; at
    m = 9000 mode 3 cuts 4608-column segments, so some runs of tiles cross a segment boundary"""
    D1, D2, A = _problem("eu", d, m)
    c32 = _handle(clp, "eu", 0, mode); c32.score_pairwise_consistency(D1, D2, A)
    c64 = _handle(clp, "eu", 1, mode); c64.score_pairwise_consistency(D1, D2, A)
    _assert_rounding_of(*_matrices(c32), *_matrices(c64))
    assert c32.count_nonzeros() == c64.count_nonzeros()


@pytest.mark.parametrize("kind,d", [("eu", 2), ("eu", 3), ("pn", 3)])
@pytest.mark.parametrize("m", [777, 4097])
def test_screened_two_shards_one_gpu(clp, kind, d, m):
    """row-block shards run the kernel without the mirror.  A shard's store cannot be read back (clp_get_dense needs the
    whole matrix), so every shard's kept upper-triangle entries of M and C are compared with the fp64 shard of the same
    rows, and their sums with one unsharded handle"""
    from clipper_b200 import distributed as cd
    D1, D2, A = _problem(kind, d, m)
    per_shard = []
    for storage in (0, 1):
        g = cd.ShardGroup(lambda: _invariant(clp, kind), clp.Params(), [0, 0], storage=storage, same_device=True)
        g.score_pairwise_consistency(D1, D2, A)
        per_shard.append([sh.count_nonzeros() for sh in g.shards])
    assert per_shard[0] == per_shard[1]
    one = _handle(clp, kind, 0); one.score_pairwise_consistency(D1, D2, A)
    assert tuple(map(sum, zip(*per_shard[0]))) == one.count_nonzeros()


@pytest.mark.parametrize("kind,d", [("eu", 3), ("pn", 3)])
@pytest.mark.parametrize("mode", [None, 3])
def test_rescored_smaller_matches_fresh(clp, kind, d, mode):
    big, small = _problem(kind, d, 4097), _problem(kind, d, 1025, seed=11)
    c = _handle(clp, kind, 0, mode); c.score_pairwise_consistency(*big)
    c.score_pairwise_consistency(*small)
    f = _handle(clp, kind, 0, mode); f.score_pairwise_consistency(*small)
    M, C = _matrices(c); Mf, Cf = _matrices(f)
    assert np.array_equal(M.view(np.uint64), Mf.view(np.uint64)) and np.array_equal(C, Cf)
    assert c.sparse_info() == f.sparse_info() and c.count_nonzeros() == f.count_nonzeros()
    u0 = np.full(1025, 0.5)
    c.solve(u0); f.solve(u0)
    sc, sf = c.get_solution(), f.get_solution()
    assert sc.u.tobytes() == sf.u.tobytes() and sc.nodes == sf.nodes
