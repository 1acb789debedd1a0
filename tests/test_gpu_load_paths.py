"""Host paths of a matrix load on one handle that no other test reaches.

* A scoring call with an association index outside D1/D2 fails with CLP_ERR_INVALID on every sweep mode, storage type
  and entry point (host and device pointers): the dense sweeps read the flag right after the scoring launch, the
  compact build reads it with its totals.  The handle then holds no matrix, and a valid scoring call on it solves bit
  for bit like a fresh handle.
* Re-finalising a scored handle (grid knobs set to their defaults, the same sweep mode again) rebuilds the compact copy
  through the build's own counting pass instead of the scoring kernel's counts, and must give the same copy."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CLP_ERR_INVALID = 1


@pytest.fixture(scope="module")
def clp(built):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import clipper_b200 as clipperpy
    return clipperpy


def _handle(clp, cfg, storage=0, mode=None):
    ip = clp.invariants.EuclideanDistanceParams()
    ip.sigma, ip.epsilon = cfg["sigma"], cfg["epsilon"]
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(ip), clp.Params(), storage=storage)
    if mode is not None:
        c.set_dense_mode(mode)
    return c


def _score(c, prob, A, entry):
    """scores through clp_score_euclidean (entry "host") or clp_score_euclidean_dev (entry "dev")"""
    if entry == "host":
        c.score_pairwise_consistency(prob["D1"], prob["D2"], A)
        return
    import torch
    from clipper_b200 import _capi
    cfg, dev = prob["cfg"], torch.device("cuda:0")
    D1 = torch.from_numpy(np.ascontiguousarray(prob["D1"].T)).to(dev)  # (n, 3) row-major == (3, n) column-major
    D2 = torch.from_numpy(np.ascontiguousarray(prob["D2"].T)).to(dev)
    Ad = torch.from_numpy(np.ascontiguousarray(A.T)).to(dev)          # (2, m) row-major == (m, 2) column-major
    torch.cuda.synchronize()
    _capi.check(c.handle, _capi.load().clp_score_euclidean_dev(c.handle, D1.data_ptr(), 3, D1.shape[0], D2.data_ptr(),
                                                               D2.shape[0], Ad.data_ptr(), Ad.shape[1], cfg["sigma"],
                                                               cfg["epsilon"], 0.0))


def _outcome(c, u0):
    c.solve(u0)
    s = c.get_solution()
    return c.dense_mode(), c.sparse_info(), s.u.tobytes(), s.score, tuple(s.nodes), s.n_evals


@pytest.mark.parametrize("mode", [0, 2, 3, 4])
@pytest.mark.parametrize("storage", [0, 1], ids=["f32", "f64"])
@pytest.mark.parametrize("entry", ["host", "dev"])
def test_bad_association_index(clp, entry, storage, mode):
    from clipper_b200 import datagen
    prob = datagen.config_problem("c2", 1500)
    bad = np.array(prob["A"], dtype=np.int32, order="F")
    bad[700, 0] = prob["D1"].shape[1] + 5
    c = _handle(clp, prob["cfg"], storage, mode)
    with pytest.raises(clp.ClipperError, match="association index out of range of D1/D2") as err:
        _score(c, prob, bad, entry)
    assert err.value.code == CLP_ERR_INVALID
    with pytest.raises(clp.ClipperError, match="before any affinity matrix"):
        c.solve(prob["u0"])
    _score(c, prob, prob["A"], entry)
    fresh = _handle(clp, prob["cfg"], storage, mode)
    _score(fresh, prob, prob["A"], entry)
    assert _outcome(c, prob["u0"]) == _outcome(fresh, prob["u0"])


@pytest.mark.parametrize("mode", [4, 3])
@pytest.mark.parametrize("m", [3001, 9000])
def test_refinalise_after_scoring(clp, m, mode):
    """mode 4 takes the resident (packed) layout, mode 3 the column segments"""
    from clipper_b200 import datagen, _capi
    prob = datagen.config_problem("c2", m)
    c = _handle(clp, prob["cfg"], mode=mode)
    c.score_pairwise_consistency(prob["D1"], prob["D2"], prob["A"])
    want = _outcome(c, prob["u0"])
    assert want[0] == (6 if mode == 4 else 3)
    for what, refinalise in [("set_grid_cap(0)", lambda: c.set_grid_cap(0)),
                             ("clp_set_ctas_per_sm(3)",
                              lambda: _capi.check(c.handle, _capi.load().clp_set_ctas_per_sm(c.handle, C.c_int(3)))),
                             ("set_dense_mode(%d)" % mode, lambda: c.set_dense_mode(mode))]:
        refinalise()
        assert _outcome(c, prob["u0"]) == want, what
