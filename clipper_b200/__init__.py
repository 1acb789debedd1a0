"""clipper_b200 -- Hopper-native (H100) CLIPPER hot path (scorePairwiseConsistency + solve).

Python mirror of the reference's ``clipperpy`` module (reference bindings/python/py_clipper.cpp:116-232)
on top of the C-ABI in include/clipper_b200.h: same class / method / attribute names, same
argument meaning, numpy float64 / int32 in and out.  The compute runs in hand-written sm_90a
CUDA kernels (clipper_b200/csrc); there is no CPU fallback for the built-in invariants.

    import clipper_b200 as clipperpy
    iparams = clipperpy.invariants.EuclideanDistanceParams(); iparams.sigma = 0.015; iparams.epsilon = 0.05
    clipper = clipperpy.CLIPPER(clipperpy.invariants.EuclideanDistance(iparams), clipperpy.Params())
    clipper.score_pairwise_consistency(D1, D2, A)      # D: (d, n) float64, A: (m, 2) int32
    clipper.solve()
    Ain = clipper.get_selected_associations()
"""
from . import _capi
from ._capi import ClipperError, STORE_F32, STORE_F64
from .api import (CLIPPER, Params, Solution, Rounding, MCMethod, MCParams, SDPParams, invariants, utils, dsd,
                  __version__)
from .batch import BatchCLIPPER, MatrixBatchCLIPPER, maxclique_many

__all__ = ["CLIPPER", "Params", "Solution", "Rounding", "MCMethod", "MCParams", "SDPParams", "invariants", "utils",
           "dsd", "BatchCLIPPER", "MatrixBatchCLIPPER", "maxclique_many", "ClipperError", "STORE_F32", "STORE_F64", "__version__"]
