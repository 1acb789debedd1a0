"""Host-side mirror of the reference's Python interface (``clipperpy``) over the C-ABI.

Names, argument meaning and defaults follow reference bindings/python/py_clipper.cpp:116-232:
  invariants.{Invariant, PairwiseInvariant, EuclideanDistanceParams, EuclideanDistance,
              PointNormalDistanceParams, PointNormalDistance}
  utils.{create_all_to_all, k2ij}      dsd.{solve, create_all_to_all, k2ij}
  Rounding, Params, Solution, MCParams, SDPParams, CLIPPER (11 methods)

Differences that are deliberate and additive:
  * ``CLIPPER(invariant, params, device=0, storage=STORE_F32)`` -- the two trailing keyword
    arguments select the GPU and the HBM storage type of the affinity matrix.
  * ``set_sparse_matrix_data`` exists (the reference forgot to bind it, SURVEY D8c).
  * ``dsd.solve`` is exported (the reference fills ``dsd`` with the utils by mistake, SURVEY D8b;
    both the mistaken names and the intended ``solve`` are present).
  * ``solve_as_maximum_clique`` / ``solve_as_msrc_sdr`` behave like a reference build without
    PMC / SCS (maxclique.cpp:141-144, sdp.cpp:298-302): they print a warning and select nothing.
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


invariants = types.SimpleNamespace(
    Invariant=Invariant, PairwiseInvariant=PairwiseInvariant,
    EuclideanDistanceParams=EuclideanDistanceParams, EuclideanDistance=EuclideanDistance,
    PointNormalDistanceParams=PointNormalDistanceParams, PointNormalDistance=PointNormalDistance)


# --------------------------------------------------------------------------------------------
# utils / dsd
# --------------------------------------------------------------------------------------------
def create_all_to_all(n1, n2):
    """reference utils.h:61-71 -> (n1*n2, 2) int32, column-major"""
    A = np.zeros((int(n1) * int(n2), 2), dtype=np.int32, order="F")
    _capi.load().clp_create_all_to_all(int(n1), int(n2), _ip(A))
    return A


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
                              find_indices_where_above_threshold=find_indices_where_above_threshold)
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


class MCParams:
    """reference maxclique.h:18-24 (kept for source compatibility; PMC is not part of the hot path)"""

    def __init__(self):
        self.method = 0
        self.threads = 24
        self.time_limit = 3600
        self.verbose = False

    def __repr__(self):
        return "<CLIPPER Maximum Clique Parameters>"


class SDPParams:
    """reference sdp.h:39-52 (kept for source compatibility; SCS is not part of the hot path)"""

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
        elif isinstance(inv, PairwiseInvariant):
            return self._score_custom(D1, D2, A if Ap is not None else None)
        else:
            raise TypeError("invariant must derive from invariants.PairwiseInvariant")
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
        """reference clipper.cpp:82-97 with a build lacking PMC (maxclique.cpp:141-144)"""
        print("Warning: clipper_b200 does not bundle PMC; maximum-clique solver unavailable.")
        self._finish_unavailable()

    def solve_as_msrc_sdr(self, params=None):
        """reference clipper.cpp:101-113 with a build lacking SCS (sdp.cpp:298-302)"""
        print("Warning: clipper_b200 does not bundle SCS; SDR solver unavailable.")
        self._finish_unavailable()

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
