"""Batches of small problems in one launch (SURVEY.md section 8f rank 4) -- host mirror of clp_batch_* (include/clipper_b200.h).

The reference's own operating point is m <= 2048 associations per registration and its benchmark solves such problems
one after the other, each with a fresh clipper::CLIPPER (reference benchmarks/main.cpp:206-208, 254-270).  ``BatchCLIPPER``
takes the whole list: one CTA per problem scores the pairs, builds the compact copy and runs the solver, no device-wide
synchronisation anywhere; results per problem are those of ``CLIPPER.score_pairwise_consistency`` + ``solve``.
``BatchCLIPPER.max_clique_many`` and ``maxclique_many`` solve each problem of such a list as a maximum clique
(clp_batch_max_clique_*): per problem the answer of ``CLIPPER.solve_as_maximum_clique`` on an fp32 handle.  A
``BatchCLIPPER`` built with a ``CudaInvariant`` scores with the caller's CUDA source (clp_batch_*_custom): per problem
what an fp32 ``CLIPPER`` with the same invariant gives.  ``solve_many_dev`` and ``max_clique_many_dev`` take the point
clouds and associations as padded CUDA tensors (clp_batch_*_dev) and give what the host calls give for the same values.
``MatrixBatchCLIPPER`` solves problems whose (M, C) the caller gives (clp_batch_solve_matrices): per problem the
result of ``CLIPPER.set_sparse_matrix_data`` / ``set_matrix_data`` + ``solve`` on an fp32 handle.
"""
import ctypes as C

import numpy as np

from . import _capi
from .api import (CudaInvariant, EuclideanDistance, MCParams, PointNormalDistance, Params, Solution, _check_f64,
                  _dev_matrix_dtype, _wait_for_torch, sdp_params, sdp_solution)


class BatchCLIPPER:
    """invariant: EuclideanDistance (data 2 x n or 3 x n), PointNormalDistance (6 x n) or CudaInvariant (d x n, one d
    per call; compiled at run time once per source and d); params: Params (rounding NONZERO or DSD_HEU)"""

    def __init__(self, invariant, params=None, device=0):
        if not isinstance(invariant, (EuclideanDistance, PointNormalDistance, CudaInvariant)):
            raise TypeError("a batch scores with the built-in invariants (EuclideanDistance, PointNormalDistance) or a "
                            "CudaInvariant")
        self._lib = _capi.load()
        self._b = _new_batch(self._lib, device)
        self._device = int(device)
        self._stream = None   # a caller's stream set with set_stream, else the batch's own
        self._invariant = invariant
        self._params = params if params is not None else Params()

    def __del__(self):
        try:
            if getattr(self, "_b", None):
                self._lib.clp_batch_destroy(self._b)
                self._b = None
        except Exception:
            pass

    def _check(self, rc):
        if rc != _capi.OK:
            msg = self._lib.clp_batch_last_error(self._b)
            raise _capi.ClipperError(rc, msg.decode() if msg else "")

    def info(self):
        """(CTAs of the last launch, HBM scratch bytes, stored affinities i<j over all problems)"""
        a, b, c = C.c_int32(), C.c_int64(), C.c_int64()
        self._check(self._lib.clp_batch_info(self._b, C.byref(a), C.byref(b), C.byref(c)))
        return int(a.value), int(b.value), int(c.value)

    def set_stream(self, cuda_stream):
        """run on an existing CUDA stream (an int handle, e.g. torch.cuda.current_stream().cuda_stream); None or 0: the
        batch's own stream"""
        self._check(self._lib.clp_batch_set_stream(self._b, C.c_void_p(cuda_stream or None)))
        self._stream = cuda_stream or None

    def max_clique_many(self, problems, params=None):
        """problems: the dicts of solve_many (u0 is not needed); params: MCParams (method, time_limit for the whole
        call, verbose; threads is not used).  Scores every problem with the batch's invariant and affinityeps and
        returns one api.Solution per problem, as CLIPPER.solve_as_maximum_clique sets it (nodes ascending, u = 0,
        score = -1, mc_info) plus ``core``, the core numbers."""
        problems = list(problems)
        n = len(problems)
        if n == 0:
            return []
        params = params if params is not None else MCParams()
        self._check(self._lib.clp_batch_set_params(self._b, C.byref(self._params._pod())))
        d, pts, ms, keep = _point_problems(problems)  # keep: the arrays pts points into, alive during the call
        inv = self._invariant
        out, args = _mc_outputs(ms, params)
        if isinstance(inv, CudaInvariant):
            src, prm, nprm = _custom_args(inv)
            rc = self._lib.clp_batch_max_clique_custom(self._b, src, prm, nprm, n, int(d), *pts, *args)
        elif isinstance(inv, EuclideanDistance):
            q = inv.params()
            rc = self._lib.clp_batch_max_clique_euclidean(self._b, n, int(d), *pts, float(q.sigma), float(q.epsilon),
                                                          float(q.mindist), *args)
        else:
            if d != 6:
                raise ValueError("PointNormalDistance expects 6 x n data")
            q = inv.params()
            rc = self._lib.clp_batch_max_clique_pointnormal(self._b, n, *pts, float(q.sigp), float(q.epsp), float(q.sign),
                                                            float(q.epsn), *args)
        self._check(rc)
        return out()

    def solve_many(self, problems):
        """problems: sequence of dicts with D1 (d, n1) float64, D2 (d, n2) float64, A (m, 2) int32 or None (all-to-all)
        and u0 (m,) float64.  Returns the list of api.Solution in input order (``.kernel_ms`` = device time of the whole
        batch launch)."""
        problems = list(problems)
        n = len(problems)
        if n == 0:
            return []
        self._check(self._lib.clp_batch_set_params(self._b, C.byref(self._params._pod())))
        d, pts, ms, keep = _point_problems(problems)  # keep: the arrays pts points into, alive during the call
        vp = C.c_void_p
        u0p, up, np_ = (vp * n)(), (vp * n)(), (vp * n)()
        u0s, us, nodes = [], [], []
        for k, (p, mk) in enumerate(zip(problems, ms)):
            u0 = np.ascontiguousarray(_check_f64(p["u0"], "u0")).reshape(-1)
            if u0.size != mk:
                raise ValueError("problem %d: u0 has %d entries, expected %d" % (k, u0.size, mk))
            uk = np.zeros(mk, np.float64); nk = np.zeros(max(mk, 1), np.int32)
            u0s.append(u0); us.append(uk); nodes.append(nk)
            u0p[k], up[k], np_[k] = u0.ctypes.data, uk.ctypes.data, nk.ctypes.data
        sols = (_capi.ClpSolution * n)()
        inv = self._invariant
        if isinstance(inv, CudaInvariant):
            src, prm, nprm = _custom_args(inv)
            rc = self._lib.clp_batch_solve_custom(self._b, src, prm, nprm, n, int(d), *pts, u0p, sols, up, np_)
        elif isinstance(inv, EuclideanDistance):
            q = inv.params()
            rc = self._lib.clp_batch_solve_euclidean(self._b, n, int(d), *pts, u0p, float(q.sigma), float(q.epsilon),
                                                     float(q.mindist), sols, up, np_)
        else:
            if d != 6:
                raise ValueError("PointNormalDistance expects 6 x n data")
            q = inv.params()
            rc = self._lib.clp_batch_solve_pointnormal(self._b, n, *pts, u0p, float(q.sigp), float(q.epsp), float(q.sign),
                                                       float(q.epsn), sols, up, np_)
        self._check(rc)
        return _solutions(sols, n, u0s, us, nodes)

    def solve_many_dev(self, D1, D2, A, u0, n1=None, n2=None, m=None):
        """solve_many for problems already on the batch's device (clp_batch_solve_*_dev).  D1: (B, d, n1_max) and D2:
        (B, d, n2_max) float64 CUDA tensors, any strides (an ``expand`` along B shares one cloud); A: (B, m_max, 2) int32
        CUDA tensor, or None for the all-to-all hypothesis everywhere; u0: (B, k) float64 with unit column stride and k
        at least every problem's association count.  n1, n2, m: B sizes (default: the padded dimensions; m[p] = 0: all-to-
        all for problem p); nothing past them is read.  Returns one api.Solution per problem as solve_many fills it,
        except that .u and .u0 are device tensor views.  Runs on the batch's stream (set_stream); without a stream of the
        caller's, torch's current stream is synchronised first."""
        import torch
        d, nb, pts, ms, keep = _dev_points(self._device, D1, D2, A, n1, n2, m)  # keep: the host size arrays of pts
        inv = self._invariant
        if isinstance(inv, PointNormalDistance) and d != 6:
            raise ValueError("PointNormalDistance expects 6 x n data")
        if not isinstance(u0, torch.Tensor) or u0.dtype != torch.float64:
            raise TypeError("u0 must be a float64 torch tensor")
        if u0.dim() != 2 or u0.shape[0] != nb or u0.shape[1] < max(ms) or u0.stride(1) != 1:
            raise ValueError("u0 must be (B, k) with unit column stride and k >= every problem's association count (%d), "
                             "got shape %s" % (max(ms), tuple(u0.shape)))
        _on_device(self._device, (u0,))
        self._check(self._lib.clp_batch_set_params(self._b, C.byref(self._params._pod())))
        _wait_for_torch(self._stream, D1.device)
        u = torch.empty((nb, max(ms)), dtype=torch.float64, device=D1.device)
        nodes = [np.zeros(mk, np.int32) for mk in ms]
        np_ = (C.c_void_p * nb)(*[nk.ctypes.data for nk in nodes])
        sols = (_capi.ClpSolution * nb)()
        io = (u0.data_ptr(), u0.stride(0))
        out = (sols, u.data_ptr(), u.stride(0), np_)
        if isinstance(inv, CudaInvariant):
            src, prm, nprm = _custom_args(inv)
            rc = self._lib.clp_batch_solve_custom_dev(self._b, src, prm, nprm, nb, d, C.byref(pts), *io, *out)
        elif isinstance(inv, EuclideanDistance):
            q = inv.params()
            rc = self._lib.clp_batch_solve_euclidean_dev(self._b, nb, d, C.byref(pts), *io, float(q.sigma),
                                                         float(q.epsilon), float(q.mindist), *out)
        else:
            q = inv.params()
            rc = self._lib.clp_batch_solve_pointnormal_dev(self._b, nb, C.byref(pts), *io, float(q.sigp), float(q.epsp),
                                                           float(q.sign), float(q.epsn), *out)
        self._check(rc)
        return _solutions(sols, nb, [u0[k, :ms[k]] for k in range(nb)], [u[k, :ms[k]] for k in range(nb)], nodes)

    def max_clique_many_dev(self, D1, D2, A, n1=None, n2=None, m=None, params=None):
        """max_clique_many for problems already on the batch's device (clp_batch_max_clique_*_dev): D1, D2, A, n1, n2
        and m as solve_many_dev takes them.  Returns what max_clique_many returns."""
        d, nb, pts, ms, keep = _dev_points(self._device, D1, D2, A, n1, n2, m)  # keep: the host size arrays of pts
        inv = self._invariant
        if isinstance(inv, PointNormalDistance) and d != 6:
            raise ValueError("PointNormalDistance expects 6 x n data")
        params = params if params is not None else MCParams()
        self._check(self._lib.clp_batch_set_params(self._b, C.byref(self._params._pod())))
        _wait_for_torch(self._stream, D1.device)
        out, args = _mc_outputs(ms, params)
        if isinstance(inv, CudaInvariant):
            src, prm, nprm = _custom_args(inv)
            rc = self._lib.clp_batch_max_clique_custom_dev(self._b, src, prm, nprm, nb, d, C.byref(pts), *args)
        elif isinstance(inv, EuclideanDistance):
            q = inv.params()
            rc = self._lib.clp_batch_max_clique_euclidean_dev(self._b, nb, d, C.byref(pts), float(q.sigma),
                                                              float(q.epsilon), float(q.mindist), *args)
        else:
            q = inv.params()
            rc = self._lib.clp_batch_max_clique_pointnormal_dev(self._b, nb, C.byref(pts), float(q.sigp), float(q.epsp),
                                                                float(q.sign), float(q.epsn), *args)
        self._check(rc)
        return out()


def _on_device(device, tensors):
    """ValueError unless every tensor is a CUDA tensor on the batch's device"""
    for X in tensors:
        if not X.is_cuda:
            raise ValueError("expected a CUDA tensor, got one on %s" % X.device)
        if X.device.index != device:
            raise ValueError("the tensor is on %s, the batch on cuda:%d" % (X.device, device))


def _dev_points(device, D1, D2, A, n1, n2, m):
    """the point clouds and associations of a batch on the device as clp_points_dev describes them: D1 (B, d, n1_max)
    and D2 (B, d, n2_max) float64, A (B, m_max, 2) int32 or None, all CUDA tensors on the device; n1, n2, m: B sizes or
    None for the padded dimensions (A None: m = 0 everywhere, the all-to-all hypothesis).  Returns (d, B, the
    ClpPointsDev, every problem's association count, the host size arrays it points into).  TypeError / ValueError
    before the library or a device is touched."""
    import torch
    tensors = (("D1", D1), ("D2", D2)) + ((("A", A),) if A is not None else ())
    for name, X in tensors:
        if not isinstance(X, torch.Tensor):
            raise TypeError("%s must be a torch tensor, got %s" % (name, type(X).__name__))
    if D1.dtype != torch.float64 or D2.dtype != torch.float64:
        raise TypeError("D1 and D2 must be float64 (points are fp64 only), got %s and %s" % (D1.dtype, D2.dtype))
    if A is not None and A.dtype != torch.int32:
        raise TypeError("A must be int32, got %s" % A.dtype)
    if D1.dim() != 3 or D2.dim() != 3 or D1.shape[:2] != D2.shape[:2] or D1.shape[0] == 0:
        raise ValueError("D1 and D2 must be (B, d, n1_max) and (B, d, n2_max) with B >= 1, got %s and %s"
                         % (tuple(D1.shape), tuple(D2.shape)))
    nb, d = int(D1.shape[0]), int(D1.shape[1])
    if A is not None and (A.dim() != 3 or A.shape[0] != nb or A.shape[2] != 2):
        raise ValueError("A must be (B, m_max, 2), got %s" % (tuple(A.shape),))

    def sizes(x, pad, name, lo):
        v = [int(pad)] * nb if x is None else [int(k) for k in x]
        if len(v) != nb or any(k < lo or k > pad for k in v):
            raise ValueError("%s must hold B sizes in [%d, %d]" % (name, lo, pad))
        return v

    s1, s2 = sizes(n1, D1.shape[2], "n1", 1), sizes(n2, D2.shape[2], "n2", 1)
    if A is None:
        if m is not None and any(int(k) != 0 for k in m):
            raise ValueError("m needs A: without A every problem takes the all-to-all hypothesis")
        sm = [0] * nb
    else:
        sm = sizes(m, A.shape[1], "m", 0)
    _on_device(device, [X for _, X in tensors])
    keep = tuple((C.c_int64 * nb)(*v) for v in (s1, s2, sm))
    pts = _capi.ClpPointsDev(D1.data_ptr(), tuple(D1.stride()), D2.data_ptr(), tuple(D2.stride()),
                             A.data_ptr() if A is not None else None, tuple(A.stride()) if A is not None else (0, 0, 0),
                             *keep)
    ms = [k if k else a * b for k, a, b in zip(sm, s1, s2)]
    return d, nb, pts, ms, keep


def _custom_args(inv):
    """(source, parameter pointer, parameter count) of a CudaInvariant as clp_batch_*_custom take them"""
    prm = (C.c_double * max(len(inv.params()), 1))(*inv.params())
    return inv.source().encode(), (prm if inv.params() else None), len(inv.params())


def _solutions(sols, n, u0s, us, nodes):
    """api.Solution per problem from the clp_solution array of a batched solve"""
    out = []
    for k in range(n):
        s = sols[k]
        o = Solution()
        o.t, o.ifinal, o.score = s.t, s.ifinal, s.score
        o.nodes = nodes[k][: s.n_nodes].tolist()
        o.u0, o.u = u0s[k], us[k]
        o.d_final, o.n_evals, o.n_matvec, o.n_inner, o.kernel_ms = s.d_final, s.n_evals, s.n_matvec, s.n_inner, s.kernel_ms
        o.prof_ms = (s.prof_matvec_ms, s.prof_combine_ms, s.prof_exchange_ms)
        out.append(o)
    return out


def _new_batch(lib, device):
    """a new clp_batch handle on the device; ClipperError with the library's reason when it cannot be made"""
    b = C.c_void_p()
    rc = lib.clp_batch_create(int(device), C.byref(b))
    if rc != _capi.OK:
        msg = lib.clp_batch_last_error(None)
        raise _capi.ClipperError(rc, msg.decode() if msg else "clp_batch_create failed")
    return b


def _point_problems(problems):
    """the point clouds of scored problems (dicts with D1 (d, n1), D2 (d, n2) and A (m, 2) int32 or None) as the batch
    C-ABI takes them: (d, (D1, n1, D2, n2, A, m) pointer arrays, the m of every problem, the converted arrays the
    pointers point into).  A missing or empty A is the all-to-all hypothesis, passed as m = 0."""
    n = len(problems)
    vp = C.c_void_p
    D1p, D2p, Ap = (vp * n)(), (vp * n)(), (vp * n)()
    n1, n2, m = (C.c_int64 * n)(), (C.c_int64 * n)(), (C.c_int64 * n)()
    keep, ms = [], []
    d = None
    for k, p in enumerate(problems):
        D1 = np.asfortranarray(_check_f64(p["D1"], "D1")); D2 = np.asfortranarray(_check_f64(p["D2"], "D2"))
        if D1.ndim != 2 or D2.ndim != 2 or D1.shape[0] != D2.shape[0]:
            raise ValueError("D1 and D2 must be (d, n1) and (d, n2)")
        if d is None:
            d = D1.shape[0]
        elif d != D1.shape[0]:
            raise ValueError("all problems of a batch must have the same data dimension")
        A = p.get("A")
        if A is None or np.size(A) == 0:
            mk = D1.shape[1] * D2.shape[1]; Ak = None
        else:
            if not isinstance(A, np.ndarray) or A.dtype != np.int32 or A.ndim != 2 or A.shape[1] != 2:
                raise TypeError("A must be an (m, 2) numpy int32 array")
            Ak = np.asfortranarray(A); mk = Ak.shape[0]
        keep += [D1, D2, Ak]
        ms.append(mk)
        D1p[k], D2p[k] = D1.ctypes.data, D2.ctypes.data
        Ap[k] = Ak.ctypes.data if Ak is not None else None
        n1[k], n2[k], m[k] = D1.shape[1], D2.shape[1], (mk if Ak is not None else 0)
    return d, (D1p, n1, D2p, n2, Ap, m), ms, keep


def matrices_to_csc(M, C_):
    """(m, colptrM, rowidxM, valM, colptrC, rowidxC, valC) of one problem, in the form clp_set_sparse_upper and
    clp_batch_solve_matrices take (colptr int64, rowidx int32, val float64).
    Dense M and C (square arrays of equal shape) follow set_matrix_data: only the strict upper triangle is read; the
    entries of M that are non-zero (NaN included) and of C that are non-zero become CSC entries, with C's values kept as
    given so that the library checks them.  scipy sparse M and C follow set_sparse_matrix_data: CSC with sorted indices,
    entries on or below the diagonal passed through (the library refuses them)."""
    import scipy.sparse as sp
    if sp.issparse(M) != sp.issparse(C_):
        raise ValueError("M and C must both be dense arrays or both scipy sparse matrices")
    if sp.issparse(M):
        if M.shape != C_.shape or len(M.shape) != 2 or M.shape[0] != M.shape[1]:
            raise ValueError("M and C must be square and of equal shape, got %s and %s" % (M.shape, C_.shape))
        arrs = []
        for X in (M, C_):
            S = sp.csc_matrix(X, dtype=np.float64)   # shares the arrays of a float64 CSC input
            if not S.has_sorted_indices:
                S = S.copy(); S.sort_indices()         # never reorders the caller's matrix in place
            arrs += [np.ascontiguousarray(S.indptr, np.int64), np.ascontiguousarray(S.indices, np.int32),
                     np.ascontiguousarray(S.data, np.float64)]
        return (M.shape[0],) + tuple(arrs)
    Md = np.asarray(_check_f64(M, "M")); Cd = np.asarray(_check_f64(C_, "C"))
    if Md.shape != Cd.shape or Md.ndim != 2 or Md.shape[0] != Md.shape[1]:
        raise ValueError("M and C must be square and of equal shape, got %s and %s" % (Md.shape, Cd.shape))
    m = Md.shape[0]
    upper = np.triu(np.ones((m, m), bool), 1)
    arrs = []
    for X in (Md, Cd):
        cols, rows = np.nonzero((upper & (X != 0)).T)   # column-major order: rows ascending within a column
        colptr = np.zeros(m + 1, np.int64)
        np.cumsum(np.bincount(cols, minlength=m), out=colptr[1:])
        arrs += [colptr, rows.astype(np.int32), np.ascontiguousarray(X[rows, cols], np.float64)]
    return (m,) + tuple(arrs)


class MatrixBatchCLIPPER:
    """Many problems given as affinity and constraint matrices, solved in one launch (clp_batch_solve_matrices): the
    batched form of set_matrix_data / set_sparse_matrix_data + solve, for affinities that do not come from the built-in
    invariants (a custom PairwiseInvariant, another consistency measure, a matrix read back with get_affinity_matrix).
    params: Params (rounding NONZERO or DSD_HEU).  The handle keeps its device buffers between calls."""

    def __init__(self, params=None, device=0):
        self._lib = _capi.load()
        self._b = _new_batch(self._lib, device)
        self._device = int(device)
        self._stream = None   # a caller's stream set with set_stream, else the batch's own
        self._params = params if params is not None else Params()

    __del__ = BatchCLIPPER.__del__
    _check = BatchCLIPPER._check
    info = BatchCLIPPER.info

    def solve_many(self, problems):
        """problems: sequence of dicts with M and C (both square dense arrays or both scipy sparse matrices, m <= 4096,
        see matrices_to_csc) and u0 (m,) float64.  Returns the list of api.Solution in input order, as
        BatchCLIPPER.solve_many fills it."""
        problems = list(problems)
        n = len(problems)
        if n == 0:
            return []
        self._check(self._lib.clp_batch_set_params(self._b, C.byref(self._params._pod())))
        vp = C.c_void_p
        ptrs = [(vp * n)() for _ in range(6)]
        u0p, up, np_ = (vp * n)(), (vp * n)(), (vp * n)()
        m = (C.c_int64 * n)()
        keep, u0s, us, nodes = [], [], [], []
        for k, p in enumerate(problems):
            csc = matrices_to_csc(p["M"], p["C"])
            mk = csc[0]
            u0 = np.ascontiguousarray(_check_f64(p["u0"], "u0")).reshape(-1)
            if u0.size != mk:
                raise ValueError("problem %d: u0 has %d entries, expected %d" % (k, u0.size, mk))
            uk = np.zeros(mk, np.float64); nk = np.zeros(max(mk, 1), np.int32)
            keep.append(csc); u0s.append(u0); us.append(uk); nodes.append(nk)
            m[k] = mk
            for q in range(6):
                a = csc[1 + q]
                ptrs[q][k] = a.ctypes.data if a.size else None
            u0p[k], up[k], np_[k] = u0.ctypes.data, uk.ctypes.data, nk.ctypes.data
        sols = (_capi.ClpSolution * n)()
        self._check(self._lib.clp_batch_solve_matrices(self._b, n, m, *ptrs, u0p, sols, up, np_))
        return _solutions(sols, n, u0s, us, nodes)

    def sdr_many(self, problems, params):
        """Semidefinite relaxations of many problems in one launch (clp_batch_sdp_matrices): problems as solve_many
        takes them, without u0 (m <= 128 each); params: SDPParams, one set for the whole call (time_limit_secs bounds
        the call).  Returns one api.Solution per problem as CLIPPER.solve_as_msrc_sdr on an fp32 handle fills it."""
        problems = list(problems)
        n = len(problems)
        if n == 0:
            return []
        vp = C.c_void_p
        ptrs = [(vp * n)() for _ in range(6)]
        m = (C.c_int64 * n)()
        keep, outs = [], []
        outp = [(vp * n)() for _ in range(4)]
        for k, p in enumerate(problems):
            csc = matrices_to_csc(p["M"], p["C"])
            mk = csc[0]
            keep.append(csc)
            m[k] = mk
            for q in range(6):
                a = csc[1 + q]
                ptrs[q][k] = a.ctypes.data if a.size else None
            o = (np.zeros(max(mk, 1), np.int32), np.zeros((max(mk, 1), max(mk, 1)), order="F"), np.zeros(max(mk, 1)),
                 np.zeros(max(mk, 1)))
            outs.append(o)
            for q in range(4):
                outp[q][k] = o[q].ctypes.data
        infos = (_capi.ClpSdpInfo * n)()
        self._check(self._lib.clp_batch_sdp_matrices(self._b, n, m, *ptrs, C.byref(sdp_params(params)), infos, *outp))
        out = []
        for k in range(n):
            mk = int(m[k])
            nodes, X, lam, ev = outs[k]
            out.append(sdp_solution(infos[k], nodes, X[:mk, :mk], lam[:mk], ev[:mk], mk, np.zeros(0)))
        if params.verbose:
            print("sdp batch: %d problems, converged %d, timed out %d | kernel %.3f ms"
                  % (n, sum(infos[k].converged for k in range(n)), sum(infos[k].timed_out for k in range(n)),
                     infos[0].kernel_ms))
        return out

    set_stream = BatchCLIPPER.set_stream

    def solve_dense_dev(self, M, C_, u0, m=None):
        """Problems given as CUDA tensors on the batch's device (clp_batch_solve_dense_dev): M and C (B, m_max, m_max),
        both float32 or both float64, with a unit stride along rows or columns; problem p is the leading m[p] x m[p]
        block, of which only the strict upper triangle is read.  u0: (B, m_max) float64.  m: B sizes (default m_max
        each, at most 4096).  Returns one api.Solution per problem as solve_many fills it, except that .u and .u0 are
        device tensor views of length m[p].  Runs on the batch's stream (set_stream); without a stream of the caller's,
        torch's current stream is synchronised first."""
        import torch
        dtype = _dev_matrix_dtype(self._device, (M, C_), 3)
        nb, mm = M.shape[0], M.shape[1]
        if M.shape[2] != mm or nb == 0:
            raise ValueError("M and C must be (B, m_max, m_max) with B >= 1, got %s" % (tuple(M.shape),))
        if not isinstance(u0, torch.Tensor) or u0.dtype != torch.float64:
            raise TypeError("u0 must be a float64 torch tensor")
        if tuple(u0.shape) != (nb, mm) or not u0.is_cuda or u0.device.index != self._device or u0.stride(1) != 1:
            raise ValueError("u0 must be a (B, m_max) float64 CUDA tensor on the batch's device with unit column stride")
        ms = [mm] * nb if m is None else [int(x) for x in m]
        if len(ms) != nb or any(x < 1 or x > mm for x in ms):
            raise ValueError("m must hold B sizes in [1, m_max]")
        self._check(self._lib.clp_batch_set_params(self._b, C.byref(self._params._pod())))
        _wait_for_torch(self._stream, M.device)
        marr = (C.c_int64 * nb)(*ms)
        u = torch.empty((nb, mm), dtype=torch.float64, device=M.device)
        nodes = [np.zeros(max(mk, 1), np.int32) for mk in ms]
        np_ = (C.c_void_p * nb)(*[nk.ctypes.data for nk in nodes])
        sols = (_capi.ClpSolution * nb)()
        self._check(self._lib.clp_batch_solve_dense_dev(self._b, nb, marr, dtype, M.data_ptr(), C_.data_ptr(), M.stride(0),
                                                         M.stride(1), M.stride(2), u0.data_ptr(), u0.stride(0), sols,
                                                         u.data_ptr(), u.stride(0), np_))
        return _solutions(sols, nb, [u0[k, :ms[k]] for k in range(nb)], [u[k, :ms[k]] for k in range(nb)], nodes)


def _mc_outputs(ms, params):
    """output arrays of one batched maximum-clique call for problems of ms[p] vertices: the trailing C-ABI arguments
    (method, time limit, infos, nodes, cores) and a function that turns them into Solutions after the call"""
    n = len(ms)
    vp = C.c_void_p
    infos = (_capi.ClpMcInfo * n)()
    nodes = [np.zeros(max(mk, 1), np.int32) for mk in ms]
    cores = [np.zeros(max(mk, 1), np.int32) for mk in ms]
    nodep, corep = (vp * n)(), (vp * n)()
    for k in range(n):
        nodep[k], corep[k] = nodes[k].ctypes.data, cores[k].ctypes.data

    def finish():
        out = []
        for k in range(n):
            info = infos[k]
            s = Solution()
            s.t = info.t
            s.nodes = nodes[k][: info.n_nodes].tolist()
            s.u = np.zeros(ms[k])
            s.score = -1
            s.kernel_ms = info.kernel_ms
            s.mc_info = {name: getattr(info, name) for name, _ in _capi.ClpMcInfo._fields_}
            s.core = cores[k][: ms[k]].copy()
            out.append(s)
        if params.verbose and n:
            i0 = infos[0]
            print("maxclique batch: %d problems, proven %d, timed out %d | adjacency %.3f ms, peel %.3f ms, "
                  "heuristic %.3f ms, search %.3f ms, wall %.3f ms"
                  % (n, sum(infos[k].proven for k in range(n)), sum(infos[k].timed_out for k in range(n)),
                     i0.adjacency_ms, i0.peel_ms, i0.heuristic_ms, i0.search_ms, 1e3 * i0.t * n))
        return out

    args = (int(params.method), float(params.time_limit), infos, nodep, corep)
    return finish, args


def graph_to_csc(G):
    """The graph of a square dense array or scipy sparse matrix as the strictly-upper CSC pattern the C-ABI takes:
    (m, colptr int64 (m + 1), rowidx int32), rows ascending within a column.  Any nonzero entry above the diagonal is
    an edge (the rule of maxclique::solve); the diagonal and the lower triangle are ignored."""
    import scipy.sparse as sp
    if sp.issparse(G):
        if len(G.shape) != 2 or G.shape[0] != G.shape[1]:
            raise ValueError("a graph must be a square matrix, got shape %s" % (G.shape,))
        S = sp.csc_matrix(G, copy=True)
        S.sum_duplicates()
        U = sp.triu(S, k=1, format="csc")
        U.eliminate_zeros()
        U.sort_indices()
        m = G.shape[0]
        colptr, rowidx = U.indptr.astype(np.int64), U.indices.astype(np.int32)
    else:
        A = np.asarray(G)
        if A.ndim != 2 or A.shape[0] != A.shape[1]:
            raise ValueError("a graph must be a square matrix, got shape %s" % (A.shape,))
        m = A.shape[0]
        cols, rows = np.nonzero(np.triu(A != 0, 1).T)  # column-major order of the upper triangle
        colptr = np.zeros(m + 1, np.int64)
        np.cumsum(np.bincount(cols, minlength=m), out=colptr[1:])
        rowidx = rows.astype(np.int32)
    if m == 0:
        raise ValueError("a graph needs at least one vertex")
    return m, np.ascontiguousarray(colptr), np.ascontiguousarray(rowidx)


def maxclique_many(graphs, params=None, device=0):
    """Maximum clique of every graph of a list in one batched call (clp_batch_max_clique_graphs), the batched
    counterpart of maxclique::solve(A, params): graphs are square numpy arrays or scipy sparse matrices, any nonzero
    entry above the diagonal is an edge, m <= 4096 vertices each.  params: MCParams (default: EXACT, 3600 s for the
    whole call).  Returns one api.Solution per graph (nodes ascending, u = 0, score = -1, mc_info, core)."""
    graphs = list(graphs)
    n = len(graphs)
    if n == 0:
        return []
    params = params if params is not None else MCParams()
    csc = [graph_to_csc(G) for G in graphs]
    lib = _capi.load()
    b = _new_batch(lib, device)
    try:
        vp = C.c_void_p
        m = (C.c_int64 * n)(*[c[0] for c in csc])
        cpp, rip = (vp * n)(), (vp * n)()
        for k, (_, cp, ri) in enumerate(csc):
            cpp[k], rip[k] = cp.ctypes.data, (ri.ctypes.data if ri.size else None)
        out, args = _mc_outputs([c[0] for c in csc], params)
        rc = lib.clp_batch_max_clique_graphs(b, n, m, cpp, rip, *args)
        if rc != _capi.OK:
            msg = lib.clp_batch_last_error(b)
            raise _capi.ClipperError(rc, msg.decode() if msg else "")
        return out()
    finally:
        lib.clp_batch_destroy(b)
