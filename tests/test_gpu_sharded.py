"""Row-block-sharded solve (SURVEY 8e): G shards must give the same inlier set and the same
objective as one GPU.  `same_device` runs two shards (1 CTA/SM each) concurrently on cuda:0, so
the peer-memory exchange code path is exercised even on a single-GPU box; with >= 2 GPUs the
shards sit on different devices and the exchange crosses NVLink."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _single(clp, prob, cfg, storage):
    ip = clp.invariants.EuclideanDistanceParams(); ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params(), storage=storage)
    # the segmented full-matrix sweep (what a sharded handle runs for a dense matrix); the shards make their own
    # automatic choice, so their sums are grouped differently -> the 1e-10 bounds of the comparisons
    c.set_dense_mode(0)
    c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
    c.solve(prob["u0"])
    return c


def _group(clp, prob, cfg, devices, storage, same_device):
    from clipper_b200 import distributed as cd

    def mk():
        ip = clp.invariants.EuclideanDistanceParams(); ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
        return clp.invariants.EuclideanDistance(ip)
    g = cd.ShardGroup(mk, clp.Params(), devices, storage=storage, same_device=same_device)
    g.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
    return g


@pytest.mark.parametrize("storage", [0, 1])
@pytest.mark.parametrize("world,m", [(2, 1000), (2, 2500), (2, 777)])  # 3 shards x 122 regs do not fit one SM
def test_sharded_same_device_matches_segmented_single(built, world, m, storage):
    import clipper_b200 as clp
    from clipper_b200 import datagen
    prob = datagen.config_problem("c2", m); cfg = prob["cfg"]
    ref = _single(clp, prob, cfg, storage); s1 = ref.get_solution()
    g = _group(clp, prob, cfg, [0] * world, storage, same_device=True)
    assert g.count_nonzeros() == ref.count_nonzeros()
    for rep in range(2):  # second solve re-uses the connected peers and the running sequence numbers
        sols = g.solve(prob["u0"])
        for s in sols:
            assert s.nodes == s1.nodes
            # the shards use a different CTA count, hence a different (fixed) grouping of the fp64 reductions
            assert abs(s.score - s1.score) <= 1e-10 * abs(s1.score)
            assert s.ifinal == s1.ifinal and s.n_evals == s1.n_evals
            assert np.abs(s.u - s1.u).max() <= 1e-10
        # all ranks bit-identical among themselves
        assert all(s.u.tobytes() == sols[0].u.tobytes() and s.score == sols[0].score for s in sols)


def test_sharded_two_devices_matches_single(built):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import clipper_b200 as clp
    from clipper_b200 import datagen
    for m in (3000, 20000):
        prob = datagen.config_problem("c2", m); cfg = prob["cfg"]
        s1 = _single(clp, prob, cfg, 0).get_solution()
        g = _group(clp, prob, cfg, [0, 1], 0, same_device=False)
        sols = g.solve(prob["u0"])
        for s in sols:
            assert s.nodes == s1.nodes and abs(s.score - s1.score) <= 1e-10 * abs(s1.score)
            assert s.n_evals == s1.n_evals
