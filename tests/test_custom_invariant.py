"""CUDA-source invariants without a GPU: the run-time compiler accepts the restated built-ins and the notebook's
invariant, rejects broken sources with a log, is linked into the library statically, and the CudaInvariant front-ends
exist and refuse host evaluation."""
import os
import subprocess
import sys

import numpy as np
import pytest

from test_gpu_custom_invariant import EUCLID_SRC, NOTEBOOK_SRC, PN_SRC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "clipper_b200", "lib")


@pytest.mark.parametrize("d", [3, 6])
def test_check_accepts_sources(built, d):
    import clipper_b200 as clipperpy
    for src in (EUCLID_SRC, NOTEBOOK_SRC) + ((PN_SRC,) if d == 6 else ()):
        assert clipperpy.invariants.check_cuda_invariant(src, d) is None
    assert clipperpy.invariants.check_cuda_invariant(EUCLID_SRC, 40) is None   # runtime dimension


def test_check_rejects_syntax_error(built):
    import clipper_b200 as clipperpy
    broken = EUCLID_SRC.replace("if (!(c < prm[1])) return 0.0;", "if (!(c < prm[1])) return 0.0", 1)
    line = broken.split("\n").index("  if (!(c < prm[1])) return 0.0") + 1
    with pytest.raises(clipperpy.ClipperError) as e:
        clipperpy.invariants.check_cuda_invariant(broken, 3)
    assert e.value.code == 1
    assert "invariant.cu(%d)" % line in str(e.value) or "invariant.cu(%d)" % (line + 1) in str(e.value), str(e.value)


def test_check_rejects_missing_definition(built):
    import clipper_b200 as clipperpy
    with pytest.raises(clipperpy.ClipperError):
        clipperpy.invariants.check_cuda_invariant("__device__ double other(double x) { return x; }\n", 3)
    with pytest.raises(clipperpy.ClipperError):
        clipperpy.invariants.check_cuda_invariant("", 3)
    with pytest.raises(clipperpy.ClipperError):
        clipperpy.invariants.check_cuda_invariant(EUCLID_SRC, 0)


def test_nvrtc_linked_statically(built):
    from clipper_b200 import _capi
    out = subprocess.run(["readelf", "-d", _capi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    needed = [l for l in out.splitlines() if "(NEEDED)" in l]
    assert needed and not any("nvrtc" in l or "nvptxcompiler" in l for l in needed), needed


def test_front_ends_exist_and_refuse_host_calls(built):
    import clipper_b200 as clipperpy
    inv = clipperpy.invariants.CudaInvariant(EUCLID_SRC, (0.01, 0.06, 0.0))
    assert isinstance(inv, clipperpy.invariants.PairwiseInvariant)
    assert inv.source() == EUCLID_SRC and inv.params() == (0.01, 0.06, 0.0)
    a = np.zeros(3)
    with pytest.raises(RuntimeError):
        inv(a, a, a, a)
    if LIB not in sys.path:
        sys.path.insert(0, LIB)
    import clipperpy as cp
    pinv = cp.invariants.CudaInvariant(EUCLID_SRC, [0.01, 0.06, 0.0])
    assert isinstance(pinv, cp.invariants.PairwiseInvariant)
    assert pinv.source() == EUCLID_SRC and pinv.params() == [0.01, 0.06, 0.0]
    with pytest.raises(RuntimeError):
        pinv(a, a, a, a)
    assert cp.invariants.CudaInvariant("x").params() == []
