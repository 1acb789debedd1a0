"""Which invariants BatchCLIPPER takes, checked before the library or a device is touched (no GPU needed)."""
import pytest


def test_batch_invariant_types():
    import clipper_b200 as clipperpy

    class HostInvariant(clipperpy.invariants.PairwiseInvariant):
        def __call__(self, ai, aj, bi, bj):
            return 1.0

    for inv in (object(), HostInvariant()):
        with pytest.raises(TypeError):
            clipperpy.BatchCLIPPER(inv, clipperpy.Params())


def test_custom_arguments():
    import clipper_b200 as clipperpy
    from clipper_b200.batch import _custom_args
    src, prm, n = _custom_args(clipperpy.invariants.CudaInvariant("// s", (0.5, 2.0)))
    assert src == b"// s" and n == 2 and list(prm) == [0.5, 2.0]
    src, prm, n = _custom_args(clipperpy.invariants.CudaInvariant("// s"))
    assert prm is None and n == 0
