"""Host-side mirror of the reference's Python interface (``clipperpy``) over the C-ABI.

Names, argument meaning and defaults follow reference bindings/python/py_clipper.cpp:116-232:
  invariants.{Invariant, PairwiseInvariant, EuclideanDistanceParams, EuclideanDistance,
              PointNormalDistanceParams, PointNormalDistance}
  utils.{create_all_to_all, k2ij}      dsd.{solve, create_all_to_all, k2ij}
  utils.distance_based_correspondences(_dev) (additive: putative associations by exact kNN on the GPU)
  utils.distance_based_correspondences_many(_dev) (additive: the same for a batch of cloud pairs in one call)
  utils.estimate_rigid_transform(_many)(_dev) (additive: the rigid transform of selected associations on the GPU)
  Rounding, Params, Solution, MCParams, SDPParams, CLIPPER (11 methods)

Differences that are deliberate and additive:
  * ``CLIPPER(invariant, params, device=0, storage=STORE_F32)`` -- the two trailing keyword
    arguments select the GPU and the HBM storage type of the affinity matrix.
  * ``set_sparse_matrix_data`` exists (the reference forgot to bind it, SURVEY D8c).
  * ``dsd.solve`` is exported (the reference fills ``dsd`` with the utils by mistake, SURVEY D8b;
    both the mistaken names and the intended ``solve`` are present).
  * ``solve_as_maximum_clique(MCParams())`` runs on the GPU (clp_max_clique: KCORE, HEU, EXACT) instead of
    PMC; its Solution carries the call's statistics in ``mc_info``.  Without params this mirror still behaves
    like a build without PMC (warning, nothing selected), as it always did.  ``core_numbers()`` is additive.
  * ``solve_as_msrc_sdr(SDPParams())`` solves the semidefinite relaxation on the GPU (clp_sdp_solve: ADMM with a
    Jacobi eigensolver, m <= 128) instead of SCS; its Solution carries X, lambdas, evec1, thr and the call's
    statistics in ``sdp_info``.  Without params it still behaves like a reference build without SCS
    (sdp.cpp:298-302): a warning, nothing selected.
"""
import ctypes as C
import types

import numpy as np

from . import _capi
from ._capi import ClpParams, ClpSolution, ClipperError, STORE_F32, STORE_F64

__version__ = "0.2.4+b200.1"  # tracks the reference version the API mirrors (CMakeLists.txt:2)


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def _lp(a):
    return a.ctypes.data_as(C.POINTER(C.c_int64))


def _check_f64(x, name):
    # the reference binds D1, D2, u0, M, C as noconvert (py_clipper.cpp:216-231): float64 required
    if not isinstance(x, np.ndarray) or x.dtype != np.float64:
        raise TypeError("%s must be a numpy float64 array (noconvert, as in clipperpy)" % name)
    return x


# --------------------------------------------------------------------------------------------
# invariants  (reference include/clipper/invariants/*.h)
# --------------------------------------------------------------------------------------------
class Invariant:
    """reference invariants/abstract.h:37-40"""


class PairwiseInvariant(Invariant):
    """reference invariants/abstract.h:56-72.  Subclass and override __call__(ai, aj, bi, bj)
    for a custom invariant: it is evaluated on the host pair by pair, like the reference does
    for Python subclasses (trampolines.h:20-29), and the resulting matrix is uploaded."""

    def __call__(self, ai, aj, bi, bj):
        raise NotImplementedError("PairwiseInvariant.__call__ is pure virtual")


class EuclideanDistanceParams:
    """reference invariants/euclidean_distance.h:22-27"""

    def __init__(self):
        self.sigma = 0.01
        self.epsilon = 0.06
        self.mindist = 0.0

    def __repr__(self):
        return "<EuclideanDistanceParams : sigma=%g epsilon=%g mindist=%g>" % (self.sigma, self.epsilon, self.mindist)


class EuclideanDistance(PairwiseInvariant):
    """reference invariants/euclidean_distance.h:19-49; scored on the GPU (K1)."""

    def __init__(self, params):
        self._params = params

    def params(self):
        return self._params

    def __call__(self, ai, aj, bi, bj):
        raise RuntimeError("EuclideanDistance is evaluated inside the CUDA scoring kernel; "
                           "there is no host implementation in this package")


class PointNormalDistanceParams:
    """reference invariants/pointnormal_distance.h:25-31"""

    def __init__(self):
        self.sigp = 0.5
        self.epsp = 0.5
        self.sign = 0.10
        self.epsn = 0.35

    def __repr__(self):
        return "<PointNormalDistanceParams : sigp=%g epsp=%g sign=%g epsn=%g>" % (
            self.sigp, self.epsp, self.sign, self.epsn)


class PointNormalDistance(PairwiseInvariant):
    """reference invariants/pointnormal_distance.h:22-53; scored on the GPU (K1)."""

    def __init__(self, params):
        self._params = params

    def params(self):
        return self._params

    def __call__(self, ai, aj, bi, bj):
        raise RuntimeError("PointNormalDistance is evaluated inside the CUDA scoring kernel; "
                           "there is no host implementation in this package")


class CudaInvariant(PairwiseInvariant):
    """A custom pairwise invariant written in CUDA C++ and scored on the GPU (clp_score_custom).  ``source`` defines

        __device__ double clp_invariant(const double* ai, const double* aj, const double* bi, const double* bj,
                                        int d, const double* prm);

    ai, aj, bi, bj are the d coordinates of D1.col(A(i,0)), D1.col(A(j,0)), D2.col(A(i,1)), D2.col(A(j,1)); it is
    called with i < j, and ``prm`` holds ``params`` (at most 16 floats).  The source is compiled at run time (NVRTC)
    once per process and setting; a source that does not compile raises ClipperError with the compiler's log."""

    def __init__(self, source, params=()):
        self._source = str(source)
        self._params = tuple(float(x) for x in params)

    def source(self):
        return self._source

    def params(self):
        return self._params

    def __call__(self, ai, aj, bi, bj):
        raise RuntimeError("CudaInvariant is evaluated on the GPU only")


def check_cuda_invariant(source, d):
    """compile ``source`` for dimension d as CudaInvariant scoring would (no GPU needed): None, or ClipperError
    carrying the compiler's log"""
    log = C.create_string_buffer(1 << 16)
    rc = _capi.load().clp_invariant_check(str(source).encode(), int(d), log, len(log))
    if rc != _capi.OK:
        raise ClipperError(rc, log.value.decode(errors="replace"))


def jit_stats():
    """(run-time compilations of invariant sources in this process, their total milliseconds)"""
    n, ms = C.c_int64(), C.c_double()
    _capi.check(None, _capi.load().clp_jit_stats(C.byref(n), C.byref(ms)))
    return int(n.value), float(ms.value)


invariants = types.SimpleNamespace(
    Invariant=Invariant, PairwiseInvariant=PairwiseInvariant,
    EuclideanDistanceParams=EuclideanDistanceParams, EuclideanDistance=EuclideanDistance,
    PointNormalDistanceParams=PointNormalDistanceParams, PointNormalDistance=PointNormalDistance,
    CudaInvariant=CudaInvariant, check_cuda_invariant=check_cuda_invariant)


# --------------------------------------------------------------------------------------------
# utils / dsd
# --------------------------------------------------------------------------------------------
def _dev_matrix_dtype(device, mats, ndim):
    """the C-ABI dtype (IN_F32 / IN_F64) of CUDA tensors of equal shape and strides with ndim dimensions on device;
    TypeError / ValueError otherwise.  torch is imported here only: the rest of the package does not need it."""
    import torch
    for X in mats:
        if not isinstance(X, torch.Tensor):
            raise TypeError("expected a torch tensor, got %s" % type(X).__name__)
        if not X.is_cuda:
            raise ValueError("expected a CUDA tensor, got one on %s" % X.device)
        if X.device.index != device:
            raise ValueError("the tensor is on %s, the handle on cuda:%d" % (X.device, device))
    if any(X.dtype != mats[0].dtype for X in mats) or mats[0].dtype not in (torch.float32, torch.float64):
        raise TypeError("M and C must both be float32 or both float64, got %s" % ", ".join(str(X.dtype) for X in mats))
    if any(X.dim() != ndim for X in mats) or any(X.shape != mats[0].shape or X.stride() != mats[0].stride() for X in mats):
        raise ValueError("M and C must be %d-dimensional with equal shapes and strides" % ndim)
    rs, cs = mats[0].stride()[-2:]
    if not ((rs == 1 and cs >= 1) or (cs == 1 and rs >= 1)):
        raise ValueError("M and C need a unit stride along rows or columns, got strides %s" % (mats[0].stride(),))
    return _capi.IN_F32 if mats[0].dtype == torch.float32 else _capi.IN_F64


def _wait_for_torch(stream, device):
    """a handle on its own stream reads tensors torch may still be writing: synchronise torch's current stream"""
    if not stream:
        import torch
        torch.cuda.current_stream(device).synchronize()


def create_all_to_all(n1, n2):
    """reference utils.h:61-71 -> (n1*n2, 2) int32, column-major"""
    A = np.zeros((int(n1) * int(n2), 2), dtype=np.int32, order="F")
    _capi.load().clp_create_all_to_all(int(n1), int(n2), _ip(A))
    return A


_knn_handles = {}   # (device, on_device) -> a handle kept for clp_correspondences(_dev)


class _KnnHandle:
    def __init__(self, device):
        self._lib = _capi.load()
        self.h = C.c_void_p()
        rc = self._lib.clp_create(int(device), STORE_F32, C.byref(self.h))
        if rc != _capi.OK:
            msg = self._lib.clp_last_error(None)
            raise ClipperError(rc, msg.decode() if msg else "clp_create failed")

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self._lib.clp_destroy(self.h)
                self.h = None
        except Exception:
            pass


def _knn_handle(device, on_device):
    key = (int(device), bool(on_device))
    if key not in _knn_handles:
        _knn_handles[key] = _KnnHandle(device)
    return _knn_handles[key].h


def _knn_args(knn, d):
    knn, d = int(knn), int(d)
    if knn < 1 or d < 1:
        raise ValueError("knn and d must be >= 1, got knn=%d, d=%d" % (knn, d))
    return min(knn, 2 ** 31 - 1)


def _knn_rows(n1, n2, knn):
    """rows of the output buffer: n1 * min(knn, n2).  knn above the cap is left for the C-ABI to reject
    (CLP_ERR_UNSUPPORTED), so the buffer is sized for the cap, not for knn."""
    return n1 * min(knn, _capi.KNN_MAX_K, n2)


_CUDA_STREAM_LEGACY = 1   # cudaStreamLegacy


def distance_based_correspondences(D1, D2, knn, radius, enforce_1to1):
    """putative associations by exact k-nearest-neighbour matching on the GPU (device 0; clp_correspondences; the
    reference's benchmarks/bm_utils.cpp:147-232 for any d <= 64): D1 (d, n1) and D2 (d, n2) float64 -> (m, 2) int32.
    Column i of D1 goes to its min(knn, n2) nearest columns of D2 by squared distance (ties to the lower index), and
    (i, j) is kept when that distance is <= radius * radius.  Rows by i, then rank; with enforce_1to1 every j keeps its
    nearest i (ties to the smallest i), rows by j."""
    D1 = np.asfortranarray(_check_f64(D1, "D1"))
    D2 = np.asfortranarray(_check_f64(D2, "D2"))
    if D1.ndim != 2 or D2.ndim != 2 or D1.shape[0] != D2.shape[0]:
        raise ValueError("D1 and D2 must be (d, n1) and (d, n2)")
    (d, n1), n2 = D1.shape, D2.shape[1]
    knn = _knn_args(knn, d)
    cap = _knn_rows(n1, n2, knn)
    A = np.zeros(2 * max(cap, 1), dtype=np.int32)
    h = _knn_handle(0, False)
    m = C.c_int64()
    _capi.check(h, _capi.load().clp_correspondences(h, _dp(D1), d, n1, _dp(D2), n2, knn, float(radius),
                                                    int(bool(enforce_1to1)), _ip(A), cap, C.byref(m)))
    m = int(m.value)
    return np.asfortranarray(A[:2 * m].reshape(2, m).T)


def distance_based_correspondences_dev(D1, D2, knn, radius, enforce_1to1):
    """distance_based_correspondences of CUDA tensors D1 (d, n1), D2 (d, n2) float64 on their device and torch's current
    stream (clp_correspondences_dev) -> (m, 2) int32 CUDA tensor, column-major (strides (1, m)): the layout
    CLIPPER.score_pairwise_consistency_dev reads without a copy.  Tensors of another layout are copied on the device
    first.  Returns once m is known (the stream is synchronised)."""
    import torch
    for name, X in (("D1", D1), ("D2", D2)):
        if not isinstance(X, torch.Tensor) or X.dtype != torch.float64:
            raise TypeError("%s must be a torch.float64 tensor" % name)
        if not X.is_cuda:
            raise ValueError("%s must be a CUDA tensor, got one on %s" % (name, X.device))
    if D1.device != D2.device:
        raise ValueError("D1 and D2 must be on the same device, got %s and %s" % (D1.device, D2.device))
    if D1.dim() != 2 or D2.dim() != 2 or D1.shape[0] != D2.shape[0]:
        raise ValueError("D1 and D2 must be (d, n1) and (d, n2)")
    (d, n1), n2 = D1.shape, D2.shape[1]
    knn = _knn_args(knn, d)
    cap = _knn_rows(n1, n2, knn)
    device = D1.device.index
    P1, P2 = D1.t().contiguous(), D2.t().contiguous()   # column-major (d, n) is row-major (n, d)
    A = torch.empty(2 * max(cap, 1), dtype=torch.int32, device=D1.device)
    h = _knn_handle(device, True)
    lib = _capi.load()
    # torch's default stream reports the handle 0, which clp_set_stream reads as "a stream of the handle's own": name
    # the legacy default stream instead, so the kernels stay ordered after torch's work (the copies above included)
    stream = torch.cuda.current_stream(D1.device).cuda_stream or _CUDA_STREAM_LEGACY
    _capi.check(h, lib.clp_set_stream(h, C.c_void_p(stream)))
    m = C.c_int64()
    _capi.check(h, lib.clp_correspondences_dev(h, P1.data_ptr(), d, n1, P2.data_ptr(), n2, knn, float(radius),
                                               int(bool(enforce_1to1)), A.data_ptr(), cap, C.byref(m)))
    m = int(m.value)
    return A[:2 * m].view(2, m).t()


_knn_batches = {}   # (device, on_device) -> a batch kept for clp_batch_correspondences(_dev)


class _KnnBatch:
    def __init__(self, device):
        self._lib = _capi.load()
        self.b = C.c_void_p()
        rc = self._lib.clp_batch_create(int(device), C.byref(self.b))
        if rc != _capi.OK:
            msg = self._lib.clp_batch_last_error(None)
            raise ClipperError(rc, msg.decode() if msg else "clp_batch_create failed")

    def __del__(self):
        try:
            if getattr(self, "b", None):
                self._lib.clp_batch_destroy(self.b)
                self.b = None
        except Exception:
            pass

    def check(self, rc):
        if rc != _capi.OK:
            msg = self._lib.clp_batch_last_error(self.b)
            raise ClipperError(rc, msg.decode() if msg else "")


def _knn_batch(device, on_device):
    key = (int(device), bool(on_device))
    if key not in _knn_batches:
        _knn_batches[key] = _KnnBatch(device)
    return _knn_batches[key]


def distance_based_correspondences_many(D1s, D2s, knn, radius, enforce_1to1):
    """distance_based_correspondences of every pair (D1s[p], D2s[p]) in one batched call on the GPU (device 0;
    clp_batch_correspondences): lists of (d, n1[p]) and (d, n2[p]) float64 arrays, one d for all -> a list of (m[p], 2)
    int32 arrays, entry p exactly what distance_based_correspondences(D1s[p], D2s[p], ...) returns."""
    D1s, D2s = list(D1s), list(D2s)
    if len(D1s) != len(D2s):
        raise ValueError("D1s and D2s must have the same length, got %d and %d" % (len(D1s), len(D2s)))
    if not D1s:
        return []
    P1 = [np.asfortranarray(_check_f64(X, "D1s[%d]" % k)) for k, X in enumerate(D1s)]
    P2 = [np.asfortranarray(_check_f64(X, "D2s[%d]" % k)) for k, X in enumerate(D2s)]
    d = P1[0].shape[0] if P1[0].ndim == 2 else -1
    for k, (X, Y) in enumerate(zip(P1, P2)):
        if X.ndim != 2 or Y.ndim != 2 or X.shape[0] != d or Y.shape[0] != d:
            raise ValueError("pair %d: D1s and D2s must hold (d, n1) and (d, n2) arrays of one d" % k)
    knn = _knn_args(knn, d)
    nb = len(P1)
    n1 = [X.shape[1] for X in P1]
    n2 = [Y.shape[1] for Y in P2]
    cap = max(_knn_rows(a, b, knn) for a, b in zip(n1, n2))
    outs = [np.zeros(2 * max(cap, 1), dtype=np.int32) for _ in range(nb)]
    vp, i64 = C.c_void_p, C.c_int64
    m = (i64 * nb)()
    kb = _knn_batch(0, False)
    kb.check(_capi.load().clp_batch_correspondences(
        kb.b, nb, d, (vp * nb)(*[X.ctypes.data for X in P1]), (i64 * nb)(*n1), (vp * nb)(*[Y.ctypes.data for Y in P2]),
        (i64 * nb)(*n2), knn, float(radius), int(bool(enforce_1to1)), (vp * nb)(*[A.ctypes.data for A in outs]), cap, m))
    return [np.asfortranarray(A[:2 * int(mk)].reshape(2, int(mk)).T) for A, mk in zip(outs, m)]


def distance_based_correspondences_many_dev(D1, D2, knn, radius, enforce_1to1, n1=None, n2=None):
    """distance_based_correspondences of a batch of cloud pairs in GPU memory, in one call on torch's current stream
    (clp_batch_correspondences_dev).  D1 (B, d, n1_max) and D2 (B, d, n2_max): float64 CUDA tensors on one device, any
    strides (an ``expand`` along B shares one cloud); n1, n2: B sizes in [0, the padded dimension] (default: the padded
    dimensions); nothing past them is read.  Returns (A, m): A a (B, cap, 2) int32 tensor with strides (2 cap, 1, cap),
    cap = the largest n1[p] * min(knn, n2[p]), whose first m[p] rows of problem p are exactly what
    distance_based_correspondences_dev gives for (D1[p, :, :n1[p]], D2[p, :, :n2[p]]); m a list of B ints.  These are
    the A and m that BatchCLIPPER.solve_many_dev and max_clique_many_dev take without a copy -- except that there m[p] = 0
    means all-to-all and m[p] > 4096 is refused, so a problem without rows (or with too many) must be left out.
    Returns once m is known (the stream is synchronised)."""
    import torch
    for name, X in (("D1", D1), ("D2", D2)):
        if not isinstance(X, torch.Tensor) or X.dtype != torch.float64:
            raise TypeError("%s must be a torch.float64 tensor" % name)
    if D1.dim() != 3 or D2.dim() != 3 or D1.shape[:2] != D2.shape[:2] or D1.shape[0] == 0:
        raise ValueError("D1 and D2 must be (B, d, n1_max) and (B, d, n2_max) with B >= 1, got %s and %s"
                         % (tuple(D1.shape), tuple(D2.shape)))
    nb, d = int(D1.shape[0]), int(D1.shape[1])
    knn = _knn_args(knn, d)

    def sizes(x, pad, name):
        v = [int(pad)] * nb if x is None else [int(k) for k in x]
        if len(v) != nb or any(k < 0 or k > pad for k in v):
            raise ValueError("%s must hold B sizes in [0, %d]" % (name, pad))
        return v

    s1, s2 = sizes(n1, D1.shape[2], "n1"), sizes(n2, D2.shape[2], "n2")
    for name, X in (("D1", D1), ("D2", D2)):
        if not X.is_cuda:
            raise ValueError("%s must be a CUDA tensor, got one on %s" % (name, X.device))
    if D1.device != D2.device:
        raise ValueError("D1 and D2 must be on the same device, got %s and %s" % (D1.device, D2.device))
    cap = max(_knn_rows(a, b, knn) for a, b in zip(s1, s2))
    buf = torch.empty(2 * nb * max(cap, 1), dtype=torch.int32, device=D1.device)
    A = buf.as_strided((nb, cap, 2), (2 * cap, 1, cap))
    kb = _knn_batch(D1.device.index, True)
    lib = _capi.load()
    # as in distance_based_correspondences_dev: torch's default stream is named as the legacy default stream
    stream = torch.cuda.current_stream(D1.device).cuda_stream or _CUDA_STREAM_LEGACY
    kb.check(lib.clp_batch_set_stream(kb.b, C.c_void_p(stream)))
    i64 = C.c_int64
    m = (i64 * nb)()
    kb.check(lib.clp_batch_correspondences_dev(
        kb.b, nb, d, D1.data_ptr() or None, (i64 * 3)(*D1.stride()), (i64 * nb)(*s1), D2.data_ptr() or None,
        (i64 * 3)(*D2.stride()), (i64 * nb)(*s2), knn, float(radius), int(bool(enforce_1to1)), buf.data_ptr(),
        (i64 * 3)(2 * max(cap, 1), 1, max(cap, 1)), cap, m))
    return A, [int(x) for x in m]


class TransformInfo:
    """outcome of one rigid-transform estimate (clp_tf_info): status (TF_OK, TF_EMPTY, TF_DEGENERATE, TF_NONFINITE),
    k (pairs used), rmse, sv (singular values of H, descending, 3 entries), gap, t (wall-clock seconds), kernel_ms"""
    __slots__ = ("status", "k", "rmse", "sv", "gap", "t", "kernel_ms")

    def __init__(self, ci):
        self.status, self.k, self.rmse = int(ci.status), int(ci.k), float(ci.rmse)
        self.sv, self.gap = np.array(ci.sv[:], dtype=np.float64), float(ci.gap)
        self.t, self.kernel_ms = float(ci.t), float(ci.kernel_ms)

    def __repr__(self):
        return "<TransformInfo status=%d k=%d rmse=%g gap=%g>" % (self.status, self.k, self.rmse, self.gap)


def _tf_rows(rows, name):
    """(int32 array or None, k) of a rows argument: None is every row"""
    if rows is None:
        return None, 0
    r = np.ascontiguousarray(np.asarray(rows).reshape(-1))
    if r.size and not np.issubdtype(r.dtype, np.integer):
        raise TypeError("%s must hold integer row indices" % name)
    if r.size and (r.min() < -2 ** 31 or r.max() >= 2 ** 31):
        raise ValueError("%s holds row indices outside int32" % name)
    return np.ascontiguousarray(r, dtype=np.int32), int(r.size)


def _tf_host_problem(D1, D2, A, rows):
    """checked host arrays of one problem: (D1, D2, A or None, m, rows, k); an A without rows and rows None take
    k = 0 rows (empty, not all-to-all)"""
    D1 = np.asfortranarray(_check_f64(D1, "D1"))
    D2 = np.asfortranarray(_check_f64(D2, "D2"))
    if D1.ndim != 2 or D2.ndim != 2 or D1.shape[0] != D2.shape[0]:
        raise ValueError("D1 and D2 must be (d, n1) and (d, n2)")
    m = 0
    if A is not None:
        if not isinstance(A, np.ndarray) or A.dtype != np.int32:
            raise TypeError("A must be a numpy int32 array (m, 2)")
        if A.ndim != 2 or A.shape[1] != 2:
            raise ValueError("A must be (m, 2)")
        m = A.shape[0]
        A = np.asfortranarray(A)
    r, kk = _tf_rows(rows, "rows")
    if A is not None and m == 0 and r is None:
        r, kk = np.zeros(1, np.int32), 0   # an empty A is no pairs, not the all-to-all hypothesis
    return D1, D2, A, m, r, kk


def _tf_T(buf, d):
    """row-major (d+1, d+1) from the column-major buffer the C-ABI fills"""
    return np.ascontiguousarray(buf.reshape(d + 1, d + 1).T)


def estimate_rigid_transform(D1, D2, A, rows=None):
    """the proper rigid transform T ((d+1, d+1) float64, row-major, b ~ R a + t) that aligns the pairs (D1[:, A[r, 0]],
    D2[:, A[r, 1]]) of the rows r of A (device 0; clp_estimate_transform).  D1 (d, n1), D2 (d, n2) float64 with d 2 or
    3; A (m, 2) int32, e.g. CLIPPER.get_selected_associations(), or None for the all-to-all hypothesis (row r = (r //
    n2, r % n2)); rows: row indices of A (each counted once per listing) or None for every row.  An A without rows
    gives status TF_EMPTY.  Returns (T, TransformInfo)."""
    D1, D2, A, m, r, k = _tf_host_problem(D1, D2, A, rows)
    d = D1.shape[0]
    T = np.zeros((d + 1) ** 2 if d >= 1 else 1)
    info = _capi.ClpTfInfo()
    h = _knn_handle(0, False)   # the utils' kept handle: only its device, stream and error string are used
    _capi.check(h, _capi.load().clp_estimate_transform(
        h, D1.ctypes.data, d, D1.shape[1], D2.ctypes.data, D2.shape[1], A.ctypes.data if A is not None else None, m,
        r.ctypes.data if r is not None else None, k, T.ctypes.data, C.byref(info)))
    return _tf_T(T, d), TransformInfo(info)


def estimate_rigid_transform_many(D1s, D2s, As, rows=None):
    """estimate_rigid_transform of every problem (D1s[p], D2s[p], As[p], rows[p]) in one batched call on the GPU
    (device 0; clp_batch_estimate_transform), one d for all; rows None or a list whose entries may be None.  Problem p
    is bit for bit the single call.  Returns (list of T, list of TransformInfo)."""
    D1s, D2s, As = list(D1s), list(D2s), list(As)
    nb = len(D1s)
    if len(D2s) != nb or len(As) != nb:
        raise ValueError("D1s, D2s and As must have the same length, got %d, %d and %d" % (nb, len(D2s), len(As)))
    rows = [None] * nb if rows is None else list(rows)
    if len(rows) != nb:
        raise ValueError("rows must hold one entry per problem")
    if nb == 0:
        return [], []
    probs = [_tf_host_problem(X, Y, A, r) for X, Y, A, r in zip(D1s, D2s, As, rows)]
    d = probs[0][0].shape[0]
    if any(q[0].shape[0] != d for q in probs):
        raise ValueError("every problem must have the same d")
    Ts = [np.zeros((d + 1) ** 2 if d >= 1 else 1) for _ in range(nb)]
    infos = (_capi.ClpTfInfo * nb)()
    vp, i64 = C.c_void_p, C.c_int64
    ptr = lambda x: x.ctypes.data if x is not None else None  # noqa: E731
    kb = _knn_batch(0, False)   # the utils' kept batch: only its device, stream and error string are used
    kb.check(_capi.load().clp_batch_estimate_transform(
        kb.b, nb, d, (vp * nb)(*[q[0].ctypes.data for q in probs]), (i64 * nb)(*[q[0].shape[1] for q in probs]),
        (vp * nb)(*[q[1].ctypes.data for q in probs]), (i64 * nb)(*[q[1].shape[1] for q in probs]),
        (vp * nb)(*[ptr(q[2]) for q in probs]), (i64 * nb)(*[q[3] for q in probs]),
        (vp * nb)(*[ptr(q[4]) for q in probs]), (i64 * nb)(*[q[5] for q in probs]), (vp * nb)(*[T.ctypes.data for T in Ts]),
        infos))
    return [_tf_T(T, d) for T in Ts], [TransformInfo(infos[p]) for p in range(nb)]


def estimate_rigid_transform_dev(D1, D2, A, rows=None):
    """estimate_rigid_transform of CUDA tensors on their device and torch's current stream (clp_estimate_transform_dev):
    D1 (d, n1), D2 (d, n2) float64, A (m, 2) int32 CUDA tensor or None (all-to-all); rows a host sequence or None.
    Tensors of another layout than column-major are copied on the device first.  Returns (T, TransformInfo), T a (d+1,
    d+1) float64 CUDA tensor; bit for bit the host call's T."""
    import torch
    for name, X in (("D1", D1), ("D2", D2)):
        if not isinstance(X, torch.Tensor) or X.dtype != torch.float64:
            raise TypeError("%s must be a torch.float64 tensor" % name)
    if A is not None and (not isinstance(A, torch.Tensor) or A.dtype != torch.int32):
        raise TypeError("A must be a torch.int32 tensor or None")
    if D1.dim() != 2 or D2.dim() != 2 or D1.shape[0] != D2.shape[0]:
        raise ValueError("D1 and D2 must be (d, n1) and (d, n2)")
    if A is not None and (A.dim() != 2 or A.shape[1] != 2):
        raise ValueError("A must be (m, 2)")
    r, k = _tf_rows(rows, "rows")
    m = 0 if A is None else int(A.shape[0])
    if A is not None and m == 0 and r is None:
        r, k = np.zeros(1, np.int32), 0   # an empty A is no pairs, not the all-to-all hypothesis
    for name, X in (("D1", D1), ("D2", D2)) + ((("A", A),) if A is not None else ()):
        if not X.is_cuda or X.device != D1.device:
            raise ValueError("%s must be a CUDA tensor on D1's device, got one on %s" % (name, X.device))
    (d, n1), n2 = D1.shape, D2.shape[1]
    P1, P2 = D1.t().contiguous(), D2.t().contiguous()   # column-major (d, n) is row-major (n, d)
    PA = A.t().contiguous() if A is not None else None
    T = torch.empty((d + 1, d + 1), dtype=torch.float64, device=D1.device)
    h = _knn_handle(D1.device.index, True)
    lib = _capi.load()
    # as in distance_based_correspondences_dev: torch's default stream is named as the legacy default stream
    stream = torch.cuda.current_stream(D1.device).cuda_stream or _CUDA_STREAM_LEGACY
    _capi.check(h, lib.clp_set_stream(h, C.c_void_p(stream)))
    info = _capi.ClpTfInfo()
    # the C-ABI writes T column-major: T.t() of a row-major tensor
    _capi.check(h, lib.clp_estimate_transform_dev(
        h, P1.data_ptr() or None, d, n1, P2.data_ptr() or None, n2, PA.data_ptr() if PA is not None else None, m,
        r.ctypes.data if r is not None else None, k, T.data_ptr(), C.byref(info)))
    return T.t(), TransformInfo(info)


def estimate_rigid_transform_many_dev(D1, D2, A, rows=None, n1=None, n2=None, m=None):
    """estimate_rigid_transform of a batch in GPU memory, in one call on torch's current stream
    (clp_batch_estimate_transform_dev).  D1, D2, A, n1, n2 and m exactly as BatchCLIPPER.solve_many_dev takes them
    (A None or m[p] = 0: all-to-all); rows: None (every row) or B entries, each None or host row indices, e.g. [s.nodes
    for s in sols].  Returns (T, infos): T a (B, d+1, d+1) float64 CUDA tensor, row-major per problem, and B
    TransformInfo; problem p is bit for bit the single call."""
    import torch
    from .batch import _dev_points
    if not isinstance(D1, torch.Tensor) or not D1.is_cuda:
        raise ValueError("D1 must be a CUDA tensor")
    d, nb, pts, ms, keep = _dev_points(D1.device.index, D1, D2, A, n1, n2, m)  # keep: the host size arrays of pts
    rows = [None] * nb if rows is None else list(rows)
    if len(rows) != nb:
        raise ValueError("rows must hold one entry per problem")
    rk = [_tf_rows(r, "rows[%d]" % p) for p, r in enumerate(rows)]
    T = torch.empty((nb, d + 1, d + 1), dtype=torch.float64, device=D1.device)
    kb = _knn_batch(D1.device.index, True)
    lib = _capi.load()
    stream = torch.cuda.current_stream(D1.device).cuda_stream or _CUDA_STREAM_LEGACY
    kb.check(lib.clp_batch_set_stream(kb.b, C.c_void_p(stream)))
    infos = (_capi.ClpTfInfo * nb)()
    vp, i64 = C.c_void_p, C.c_int64
    kb.check(lib.clp_batch_estimate_transform_dev(
        kb.b, nb, d, C.byref(pts), (vp * nb)(*[r.ctypes.data if r is not None else None for r, _ in rk]),
        (i64 * nb)(*[k for _, k in rk]), T.data_ptr(), (i64 * 3)(*T.stride()), infos))
    return T, [TransformInfo(infos[p]) for p in range(nb)]


def k2ij(k, n):
    """reference utils.cpp:87-97"""
    i, j = C.c_uint64(), C.c_uint64()
    _capi.load().clp_k2ij(int(k), int(n), C.byref(i), C.byref(j))
    return int(i.value), int(j.value)


def find_indices_of_k_largest(x, k):
    """reference utils.cpp:33-55"""
    x = np.ascontiguousarray(x, dtype=np.float64)
    kk = min(max(int(k), 0), x.size)
    out = np.zeros(max(kk, 1), dtype=np.int32)
    n = _capi.load().clp_find_k_largest(_dp(x), x.size, int(k), _ip(out))
    return out[:n].copy()


def find_indices_where_above_threshold(x, thr):
    """reference utils.cpp:59-68"""
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = np.zeros(max(x.size, 1), dtype=np.int32)
    n = _capi.load().clp_find_above(_dp(x), x.size, float(thr), _ip(out))
    return out[:n].copy()


def dsd_solve(A, S=()):
    """reference dsd.cpp:274-327: exact densest edge-weighted subgraph of dense A restricted to S"""
    A = np.asfortranarray(_check_f64(A, "A"))
    n = A.shape[0]
    S = np.ascontiguousarray(np.asarray(S, dtype=np.int32))
    out = np.zeros(max(n, 1), dtype=np.int32)
    k = _capi.load().clp_dsd_dense(_dp(A), n, _ip(S) if S.size else None, int(S.size), _ip(out))
    if k < 0:
        raise ClipperError(_capi.OK + 4, "dsd.solve failed (%d)" % k)
    return out[:k].tolist()


utils = types.SimpleNamespace(create_all_to_all=create_all_to_all, k2ij=k2ij,
                              find_indices_of_k_largest=find_indices_of_k_largest,
                              find_indices_where_above_threshold=find_indices_where_above_threshold,
                              distance_based_correspondences=distance_based_correspondences,
                              distance_based_correspondences_dev=distance_based_correspondences_dev,
                              distance_based_correspondences_many=distance_based_correspondences_many,
                              distance_based_correspondences_many_dev=distance_based_correspondences_many_dev,
                              estimate_rigid_transform=estimate_rigid_transform,
                              estimate_rigid_transform_many=estimate_rigid_transform_many,
                              estimate_rigid_transform_dev=estimate_rigid_transform_dev,
                              estimate_rigid_transform_many_dev=estimate_rigid_transform_many_dev,
                              TransformInfo=TransformInfo, TF_OK=_capi.TF_OK, TF_EMPTY=_capi.TF_EMPTY,
                              TF_DEGENERATE=_capi.TF_DEGENERATE, TF_NONFINITE=_capi.TF_NONFINITE)
dsd = types.SimpleNamespace(solve=dsd_solve, create_all_to_all=create_all_to_all, k2ij=k2ij)


# --------------------------------------------------------------------------------------------
# Params / Solution
# --------------------------------------------------------------------------------------------
class Rounding:
    """reference clipper.h:49-59"""
    NONZERO = 0
    DSD = 1
    DSD_HEU = 2


class Params:
    """reference clipper.h:27-60 (same fields, same defaults)"""

    def __init__(self):
        p = ClpParams()
        _capi.load().clp_default_params(C.byref(p))
        for name, _ in ClpParams._fields_:
            setattr(self, name, getattr(p, name))
        self.rescale_u0 = bool(self.rescale_u0)

    def _pod(self):
        p = ClpParams()
        for name, _ in ClpParams._fields_:
            setattr(p, name, int(getattr(self, name)) if name in ("maxiniters", "maxoliters", "maxlsiters",
                                                                 "rescale_u0", "rounding") else getattr(self, name))
        return p

    def __repr__(self):
        return "<CLIPPER Parameters>"


class MCMethod:
    """reference maxclique.h:16 (same order)"""
    EXACT = 0
    HEU = 1
    KCORE = 2


class MCParams:
    """reference maxclique.h:18-24 (same fields and defaults; threads is not used by the GPU solver)"""

    def __init__(self):
        self.method = 0
        self.threads = 24
        self.time_limit = 3600
        self.verbose = False

    def __repr__(self):
        return "<CLIPPER Maximum Clique Parameters>"


class SDPParams:
    """reference sdp.h:39-52 (same fields and defaults).  max_iters, eps_abs, eps_rel and time_limit_secs steer the GPU
    relaxation; acceleration_interval, acceleration_lookback and eps_infeas are SCS settings and have no effect (the
    relaxation is always feasible and bounded)."""

    def __init__(self):
        self.verbose = False
        self.max_iters = 2000
        self.acceleration_interval = 10
        self.acceleration_lookback = 10
        self.eps_abs = 1e-3
        self.eps_rel = 1e-3
        self.eps_infeas = 1e-7
        self.time_limit_secs = 0

    def __repr__(self):
        return "<CLIPPER SDP Parameters>"


def sdp_params(p):
    """clp_sdp_params of an SDPParams"""
    out = _capi.ClpSdpParams()
    out.max_iters, out.eps_abs = int(p.max_iters), float(p.eps_abs)
    out.eps_rel, out.time_limit_s = float(p.eps_rel), float(p.time_limit_secs)
    return out


def sdp_solution(info, nodes, X, lambdas, evec1, m, u0):
    """Solution of solve_as_msrc_sdr (ref clipper.cpp:101-113): nodes, t, u = 0, score = -1, ifinal = 0, sdp_info"""
    s = Solution()
    s.t = info.t
    s.nodes = nodes[: info.n_nodes].tolist()
    s.u0 = u0
    s.u = np.zeros(m)
    s.score = -1
    s.kernel_ms = info.kernel_ms
    d = {name: getattr(info, name) for name, _ in _capi.ClpSdpInfo._fields_}
    d.update(X=np.array(X), lambdas=np.array(lambdas), evec1=np.array(evec1), pobj=-info.value, dobj=-info.bound)
    s.sdp_info = d
    return s


def sdp_summary(m, info):
    return ("sdp: n %d iters %d%s%s value %.9g bound %.9g rho %g sweeps %d nodes %d | kernel %.3f ms, eig+proj %.3f ms"
            % (m, info.iters, " converged" if info.converged else "", " (time limit)" if info.timed_out else "",
               info.value, info.bound, info.rho, info.n_sweeps, info.n_nodes, info.kernel_ms, info.proj_ms))


class Solution:
    """reference clipper.h:65-73 (+ device counters)"""

    def __init__(self):
        self.t = 0.0
        self.ifinal = 0
        self.nodes = []
        self.u0 = np.zeros(0)
        self.u = np.zeros(0)
        self.score = 0.0
        # additive diagnostics
        self.d_final = 0.0
        self.n_evals = 0
        self.n_matvec = 0
        self.n_inner = 0
        self.kernel_ms = 0.0
        self.prof_ms = (0.0, 0.0, 0.0)  # in-kernel split: dense passes, combine loops, exchange
        self.mc_info = None  # solve_as_maximum_clique: the clp_mc_info fields as a dict
        self.sdp_info = None  # solve_as_msrc_sdr: X, lambdas, evec1, thr, iters, pobj, dobj and the clp_sdp_info fields

    def __repr__(self):
        return "<CLIPPER Solution>"


# --------------------------------------------------------------------------------------------
# CLIPPER
# --------------------------------------------------------------------------------------------
class CLIPPER:
    """reference clipper.h:78-148 / py_clipper.cpp:197-232"""

    def __init__(self, invariant, params, device=0, storage=STORE_F32):
        self._lib = _capi.load()
        self._h = C.c_void_p()
        rc = self._lib.clp_create(int(device), int(storage), C.byref(self._h))
        if rc != _capi.OK:
            msg = self._lib.clp_last_error(None)
            raise ClipperError(rc, msg.decode() if msg else "clp_create failed")
        self._device = int(device)
        self._stream = None   # a caller's stream set with set_stream, else the handle's own
        self._invariant = invariant
        self._params = params
        self._parallelize = True
        self._soln = Solution()
        self._A_custom = None
        _capi.check(self._h, self._lib.clp_set_params(self._h, C.byref(params._pod())))

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self._lib.clp_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def __repr__(self):
        return "<CLIPPER>"

    # -- handle access for the low-level (device-pointer) entry points used by bench.py
    @property
    def handle(self):
        return self._h

    def set_stream(self, cuda_stream):
        _capi.check(self._h, self._lib.clp_set_stream(self._h, C.c_void_p(cuda_stream)))
        self._stream = cuda_stream or None

    def set_dense_mode(self, mode):
        """4 (default) auto; 6 compact rows + resident trial vector (m <= 27648); 3 compact rows, column segments;
        2 upper triangle read once, two-sided update; 0 segments; any other value raises ClipperError"""
        _capi.check(self._h, self._lib.clp_set_dense_mode(self._h, int(mode)))

    def set_grid_cap(self, n_ctas):
        """at most n_ctas CTAs in this object's persistent kernels (0 = every SM): lets several shards share one GPU"""
        _capi.check(self._h, self._lib.clp_set_grid_cap(self._h, int(n_ctas)))

    def dense_mode(self):
        """effective sweep mode of the current problem (sharded handles fall back from 2 to 0)"""
        a, b = C.c_int(), C.c_int()
        _capi.check(self._h, self._lib.clp_get_dense_mode(self._h, C.byref(a), C.byref(b)))
        return int(b.value)

    def sparse_info(self):
        """(entries kept by the compact-row copy, algorithmic bytes of one sparse pass)"""
        a, b = C.c_int64(), C.c_int64()
        _capi.check(self._h, self._lib.clp_sparse_info(self._h, C.byref(a), C.byref(b)))
        return int(a.value), int(b.value)

    def last_solve_sweeps(self):
        """how the line-search evaluations of the last solve read the matrix (clp_last_solve_sweeps): evaluations that
        swept the whole compact copy, rebuilt the restricted copy, swept only the restricted copy; entries and padding
        entries the restricted sweeps read; full sweeps after the first rebuild"""
        a = (C.c_int64 * 6)()
        _capi.check(self._h, self._lib.clp_last_solve_sweeps(self._h, a))
        return dict(zip(("full", "rebuild", "restricted", "entries", "padding", "fallback"), (int(x) for x in a)))

    def _sync_params(self):
        _capi.check(self._h, self._lib.clp_set_params(self._h, C.byref(self._params._pod())))

    # -- K1
    def score_pairwise_consistency(self, D1, D2, A=None):
        """reference clipper.cpp:21-65.  D1, D2: (d, n) float64; A: (m, 2) int32 or None/empty
        for the all-to-all hypothesis."""
        self._sync_params()
        D1 = np.asfortranarray(_check_f64(D1, "D1"))
        D2 = np.asfortranarray(_check_f64(D2, "D2"))
        if D1.ndim != 2 or D2.ndim != 2 or D1.shape[0] != D2.shape[0]:
            raise ValueError("D1 and D2 must be (d, n1) and (d, n2)")
        d, n1 = D1.shape
        n2 = D2.shape[1]
        if A is None or np.size(A) == 0:
            Ap, m = None, 0
        else:
            if not isinstance(A, np.ndarray) or A.dtype != np.int32 or A.ndim != 2 or A.shape[1] != 2:
                raise TypeError("A must be an (m, 2) numpy int32 array (noconvert, as in clipperpy)")
            A = np.asfortranarray(A)
            Ap, m = _ip(A), A.shape[0]
        inv = self._invariant
        self._A_custom = None
        if isinstance(inv, EuclideanDistance):
            p = inv.params()
            rc = self._lib.clp_score_euclidean(self._h, _dp(D1), d, n1, _dp(D2), n2, Ap, m,
                                               float(p.sigma), float(p.epsilon), float(p.mindist))
        elif isinstance(inv, PointNormalDistance):
            if d != 6:
                raise ValueError("PointNormalDistance expects 6 x n data (point; normal)")
            p = inv.params()
            rc = self._lib.clp_score_pointnormal(self._h, _dp(D1), n1, _dp(D2), n2, Ap, m,
                                                 float(p.sigp), float(p.epsp), float(p.sign), float(p.epsn))
        elif isinstance(inv, CudaInvariant):  # before the generic branch: a CudaInvariant is a PairwiseInvariant too
            prm = np.asarray(inv.params(), dtype=np.float64)
            rc = self._lib.clp_score_custom(self._h, inv.source().encode(), _dp(prm) if prm.size else None, prm.size,
                                            _dp(D1), d, n1, _dp(D2), n2, Ap, m)
        elif isinstance(inv, PairwiseInvariant):
            return self._score_custom(D1, D2, A if Ap is not None else None)
        else:
            raise TypeError("invariant must derive from invariants.PairwiseInvariant")
        _capi.check(self._h, rc)

    def score_pairwise_consistency_dev(self, D1, D2, A=None):
        """score_pairwise_consistency from CUDA tensors on the handle's device (clp_score_*_dev, clp_score_custom_dev):
        D1, D2: (d, n) float64; A: (m, 2) int32 or None for the all-to-all hypothesis.  Tensors whose layout differs
        from the column-major one the library reads are copied on the device first.  A PairwiseInvariant other than the
        built-ins and CudaInvariant runs on the host: TypeError.  Without a stream of the caller's, torch's current
        stream is synchronised first."""
        import torch
        inv = self._invariant
        if not isinstance(inv, (EuclideanDistance, PointNormalDistance, CudaInvariant)):
            raise TypeError("score_pairwise_consistency_dev scores with EuclideanDistance, PointNormalDistance or a "
                            "CudaInvariant; other invariants run on the host (score_pairwise_consistency)")
        given = [("D1", D1, torch.float64), ("D2", D2, torch.float64)] + ([("A", A, torch.int32)] if A is not None else [])
        for name, X, dt in given:
            if not isinstance(X, torch.Tensor) or X.dtype != dt:
                raise TypeError("%s must be a %s torch tensor" % (name, dt))
        if D1.dim() != 2 or D2.dim() != 2 or D1.shape[0] != D2.shape[0]:
            raise ValueError("D1 and D2 must be (d, n1) and (d, n2)")
        if A is not None and (A.dim() != 2 or A.shape[1] != 2):
            raise ValueError("A must be (m, 2)")
        for name, X, _ in given:
            if not X.is_cuda or X.device.index != self._device:
                raise ValueError("%s must be a CUDA tensor on cuda:%d, got one on %s" % (name, self._device, X.device))
        d, n1, n2 = D1.shape[0], D1.shape[1], D2.shape[1]
        if isinstance(inv, PointNormalDistance) and d != 6:
            raise ValueError("PointNormalDistance expects 6 x n data (point; normal)")
        self._sync_params()
        # column-major (d, n) and (m, 2): row-major (n, d) and (2, m); contiguous() copies only when the layout differs
        P1, P2 = D1.t().contiguous(), D2.t().contiguous()
        At = A.t().contiguous() if A is not None and A.shape[0] > 0 else None
        Ap, m = (At.data_ptr(), At.shape[1]) if At is not None else (None, 0)
        _wait_for_torch(self._stream, D1.device)
        self._A_custom = None
        if isinstance(inv, EuclideanDistance):
            p = inv.params()
            rc = self._lib.clp_score_euclidean_dev(self._h, P1.data_ptr(), d, n1, P2.data_ptr(), n2, Ap, m,
                                                   float(p.sigma), float(p.epsilon), float(p.mindist))
        elif isinstance(inv, PointNormalDistance):
            p = inv.params()
            rc = self._lib.clp_score_pointnormal_dev(self._h, P1.data_ptr(), n1, P2.data_ptr(), n2, Ap, m,
                                                     float(p.sigp), float(p.epsp), float(p.sign), float(p.epsn))
        else:
            prm = np.asarray(inv.params(), dtype=np.float64)
            rc = self._lib.clp_score_custom_dev(self._h, inv.source().encode(), _dp(prm) if prm.size else None, prm.size,
                                                P1.data_ptr(), d, n1, P2.data_ptr(), n2, Ap, m)
        _capi.check(self._h, rc)

    def _score_custom(self, D1, D2, A):
        """Custom-invariant host path (SURVEY D9): a user functor cannot run inside a CUDA kernel,
        so it is evaluated per pair on the host exactly like clipper.cpp:31-56 and the dense
        matrices are uploaded with clp_set_dense (C = pattern of M, clipper.cpp:63-64)."""
        if A is None:
            A = create_all_to_all(D1.shape[1], D2.shape[1])
        m = A.shape[0]
        M = np.zeros((m, m), dtype=np.float64, order="F")
        eps = self._params.affinityeps
        for i in range(m):
            for j in range(i + 1, m):
                if A[i, 0] == A[j, 0] or A[i, 1] == A[j, 1]:
                    continue
                scr = float(self._invariant(D1[:, A[i, 0]], D1[:, A[j, 0]], D2[:, A[i, 1]], D2[:, A[j, 1]]))
                if scr > eps:
                    M[i, j] = scr
        Cm = (M != 0).astype(np.float64, order="F")
        _capi.check(self._h, self._lib.clp_set_dense(self._h, _dp(M), _dp(Cm), m))
        self._A_custom = np.asfortranarray(A, dtype=np.int32)

    # -- K2..K6
    def solve(self, u0=None):
        """reference clipper.cpp:69-78,172-323"""
        self._sync_params()
        m = self._m()
        if m == 0:  # no matrix yet: let the library report it
            _capi.check(self._h, self._lib.clp_solve(self._h, None, None, None, None, None))
        if u0 is None or np.size(u0) == 0:
            u0p = None
        else:
            u0 = np.ascontiguousarray(_check_f64(u0, "u0")).reshape(-1)
            if u0.size != m:
                raise ValueError("u0 has %d entries, expected %d" % (u0.size, m))
            u0p = _dp(u0)
        s = ClpSolution()
        u = np.zeros(m, dtype=np.float64)
        u0_used = np.zeros(m, dtype=np.float64)
        nodes = np.zeros(max(m, 1), dtype=np.int32)
        _capi.check(self._h, self._lib.clp_solve(self._h, u0p, C.byref(s), _dp(u), _ip(nodes), _dp(u0_used)))
        out = Solution()
        out.t, out.ifinal, out.score = s.t, s.ifinal, s.score
        out.nodes = nodes[: s.n_nodes].tolist()
        out.u0, out.u = u0_used, u
        out.d_final, out.n_evals, out.n_matvec, out.n_inner, out.kernel_ms = (
            s.d_final, s.n_evals, s.n_matvec, s.n_inner, s.kernel_ms)
        out.prof_ms = (s.prof_matvec_ms, s.prof_combine_ms, s.prof_exchange_ms)
        self._soln = out

    def solve_as_maximum_clique(self, params=None):
        """reference clipper.cpp:82-97: maximum clique of the constraint graph on the GPU (clp_max_clique).
        params: MCParams (method EXACT / HEU / KCORE, time_limit in seconds, verbose); threads is not used.
        The solution holds the nodes ascending, u = 0, score = -1, and the call's statistics in mc_info.
        Called without params, this mirror keeps its earlier behaviour (a build without PMC: a warning, nothing
        selected, score = -1), so code written against it sees no change; pass MCParams() to run the solver."""
        if params is None:
            print("Warning: solve_as_maximum_clique() without MCParams selects nothing; "
                  "pass clipper_b200.MCParams() to run the GPU maximum-clique solver.")
            self._finish_unavailable()
            return
        m = self._m()
        nodes = np.zeros(max(m, 1), dtype=np.int32)
        info = _capi.ClpMcInfo()
        _capi.check(self._h, self._lib.clp_max_clique(self._h, int(params.method), float(params.time_limit),
                                                      _ip(nodes), C.byref(info)))
        if params.verbose:
            print("maxclique: n %d edges %d max core %d lb %d ub %d omega %d proven %d%s | adjacency %.3f ms, "
                  "peel %.3f ms, heuristic %.3f ms, search %.3f ms (%d branches)"
                  % (m, info.n_edges, info.max_core, info.lower_bound, info.upper_bound, info.n_nodes, info.proven,
                     " (time limit)" if info.timed_out else "", info.adjacency_ms, info.peel_ms, info.heuristic_ms,
                     info.search_ms, info.n_branches))
        s = Solution()
        s.t = info.t
        s.nodes = nodes[: info.n_nodes].tolist()
        s.u0 = self._soln.u0  # untouched, as in the reference
        s.u = np.zeros(m)
        s.score = -1
        s.kernel_ms = info.kernel_ms
        s.mc_info = {name: getattr(info, name) for name, _ in _capi.ClpMcInfo._fields_}
        self._soln = s

    def core_numbers(self):
        """core number of every vertex of the constraint graph (additive; clp_core_numbers)"""
        out = np.zeros(max(self._m(), 1), dtype=np.int32)
        _capi.check(self._h, self._lib.clp_core_numbers(self._h, _ip(out)))
        return out[: self._m()].copy()

    def solve_as_msrc_sdr(self, params=None):
        """reference clipper.cpp:101-113: the semidefinite relaxation of the handle's M and C on the GPU
        (clp_sdp_solve, m <= 128).  The solution holds the nodes ascending, u = 0, score = -1, and in sdp_info X,
        lambdas, evec1, thr, iters, pobj = -value, dobj = -bound and the clp_sdp_info fields.
        Called without params, this mirror keeps its earlier behaviour (a build without SCS: a warning, nothing
        selected, score = -1); pass SDPParams() to run the solver."""
        if params is None:
            print("Warning: clipper_b200 does not bundle SCS; SDR solver unavailable.")
            self._finish_unavailable()
            return
        m = self._m()
        k = max(m, 1)
        nodes, X = np.zeros(k, dtype=np.int32), np.zeros((k, k), order="F")
        lam, ev = np.zeros(k), np.zeros(k)
        info = _capi.ClpSdpInfo()
        _capi.check(self._h, self._lib.clp_sdp_solve(self._h, C.byref(sdp_params(params)), C.byref(info), _ip(nodes),
                                                     _dp(X), _dp(lam), _dp(ev)))
        self._soln = sdp_solution(info, nodes, X[:m, :m] if m else X[:0, :0], lam[:m], ev[:m], m, self._soln.u0)
        if params.verbose:
            print(sdp_summary(m, info))

    def _finish_unavailable(self):
        s = Solution()
        s.u = np.zeros(self._m())
        s.score = -1
        self._soln = s

    # -- getters / setters (K7)
    def _m(self):
        m = C.c_int64()
        _capi.check(self._h, self._lib.clp_num_associations(self._h, C.byref(m)))
        return int(m.value)

    def get_solution(self):
        return self._soln

    def get_initial_associations(self):
        if self._A_custom is not None:
            return self._A_custom.copy()
        A = np.zeros((self._m(), 2), dtype=np.int32, order="F")
        _capi.check(self._h, self._lib.clp_get_associations(self._h, _ip(A)))
        return A

    def get_selected_associations(self):
        """reference utils.cpp:101-108"""
        A = self.get_initial_associations()
        return A[np.asarray(self._soln.nodes, dtype=np.int64), :]

    def get_affinity_matrix(self):
        m = self._m()
        out = np.zeros((m, m), dtype=np.float64, order="F")
        _capi.check(self._h, self._lib.clp_get_dense(self._h, 0, _dp(out)))
        return out

    def get_constraint_matrix(self):
        m = self._m()
        out = np.zeros((m, m), dtype=np.float64, order="F")
        _capi.check(self._h, self._lib.clp_get_dense(self._h, 1, _dp(out)))
        return out

    def set_matrix_data(self, M, C_):
        """reference clipper.cpp:149-158"""
        M = np.asfortranarray(_check_f64(M, "M"))
        C_ = np.asfortranarray(_check_f64(C_, "C"))
        if M.shape != C_.shape or M.ndim != 2 or M.shape[0] != M.shape[1]:
            raise ValueError("M and C must be square and of equal shape")
        self._A_custom = None
        _capi.check(self._h, self._lib.clp_set_dense(self._h, _dp(M), _dp(C_), M.shape[0]))

    def set_matrix_data_dev(self, M, C_):
        """set_matrix_data from CUDA tensors already on the handle's device (clp_set_dense_dev): M and C are (m, m), both
        float32 or both float64, each with one unit stride (``.t()`` views and slices of larger tensors need no copy).
        Only the strict upper triangle is read; a float32 x is stored as the float64 (double)x would be.  Runs on the
        handle's stream (set_stream) and returns when the matrix is built.  Without a stream of the caller's, torch's
        current stream is synchronised first: the handle's own stream does not wait for the work that made M and C."""
        dtype = _dev_matrix_dtype(self._device, (M, C_), 2)
        if M.shape[0] != M.shape[1]:
            raise ValueError("M and C must be square, got %s" % (tuple(M.shape),))
        _wait_for_torch(self._stream, M.device)
        self._A_custom = None
        _capi.check(self._h, self._lib.clp_set_dense_dev(self._h, M.data_ptr(), C_.data_ptr(), M.shape[0], dtype,
                                                         M.stride(0), M.stride(1)))

    def set_sparse_matrix_data(self, M, C_):
        """reference clipper.cpp:162-166; M, C: scipy.sparse matrices, strictly upper triangular"""
        import scipy.sparse as sp
        Ms, Cs = sp.csc_matrix(M), sp.csc_matrix(C_)
        Ms.sort_indices(); Cs.sort_indices()
        m = Ms.shape[0]
        a = [np.ascontiguousarray(Ms.indptr, np.int64), np.ascontiguousarray(Ms.indices, np.int32),
             np.ascontiguousarray(Ms.data, np.float64), np.ascontiguousarray(Cs.indptr, np.int64),
             np.ascontiguousarray(Cs.indices, np.int32), np.ascontiguousarray(Cs.data, np.float64)]
        for k in (1, 2, 4, 5):
            if a[k].size == 0:
                a[k] = np.zeros(1, a[k].dtype)
        self._A_custom = None
        _capi.check(self._h, self._lib.clp_set_sparse_upper(self._h, m, _lp(a[0]), _ip(a[1]), _dp(a[2]),
                                                            _lp(a[3]), _ip(a[4]), _dp(a[5])))

    def set_parallelize(self, parallelize):
        """reference clipper.h:148 -- kept for source compatibility; the GPU path is always parallel."""
        self._parallelize = bool(parallelize)

    # -- additive: the exposed mat-vec and density counters
    def matvec(self, v, d):
        """y = Md v (clipper.cpp:219), plus the raw products Mhat v, Chat v"""
        m = self._m()
        v = np.ascontiguousarray(_check_f64(v, "v")).reshape(-1)
        y, Mv, Cv = np.zeros(m), np.zeros(m), np.zeros(m)
        _capi.check(self._h, self._lib.clp_matvec(self._h, _dp(v), float(d), _dp(y), _dp(Mv), _dp(Cv)))
        return y, Mv, Cv

    def count_nonzeros(self):
        a, b = C.c_int64(), C.c_int64()
        _capi.check(self._h, self._lib.clp_count_nonzeros(self._h, C.byref(a), C.byref(b)))
        return int(a.value), int(b.value)
