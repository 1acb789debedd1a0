"""ctypes binding of the C-ABI in include/clipper_b200.h (libclipper_b200.so).

The library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a) and lives in
``clipper_b200/lib/``.  There is no fallback: if the shared object is missing, or no Hopper
GPU is usable, loading / handle creation raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libclipper_b200.so")

OK = 0
STORE_F32, STORE_F64 = 0, 1
IN_F32, IN_F64 = 0, 1
ROUND_NONZERO, ROUND_DSD, ROUND_DSD_HEU = 0, 1, 2

# every symbol include/clipper_b200.h declares (checked by tests/test_capi_symbols.py)
SYMBOLS = [
    "clp_create", "clp_destroy", "clp_last_error", "clp_default_params", "clp_set_params",
    "clp_get_params", "clp_set_stream", "clp_version",
    "clp_score_euclidean", "clp_score_pointnormal", "clp_score_euclidean_dev", "clp_score_pointnormal_dev",
    "clp_set_dense", "clp_set_sparse_upper", "clp_get_dense", "clp_num_associations",
    "clp_get_associations", "clp_count_nonzeros",
    "clp_solve", "clp_solve_dev", "clp_matvec", "clp_matvec_dev",
    "clp_k2ij", "clp_create_all_to_all", "clp_find_k_largest", "clp_find_above", "clp_dsd_dense",
    "clp_shard_config", "clp_shard_rows", "clp_shard_export", "clp_shard_import", "clp_shard_blob_bytes",
    "clp_set_ctas_per_sm", "clp_set_grid_cap", "clp_set_dense_mode", "clp_get_dense_mode", "clp_sparse_info",
    "clp_batch_create", "clp_batch_destroy", "clp_batch_last_error", "clp_batch_set_params",
    "clp_batch_solve_euclidean", "clp_batch_solve_pointnormal", "clp_batch_info",
    "clp_max_clique", "clp_core_numbers",
    "clp_batch_max_clique_euclidean", "clp_batch_max_clique_pointnormal", "clp_batch_max_clique_graphs",
    "clp_batch_solve_matrices", "clp_set_dense_dev", "clp_batch_set_stream", "clp_batch_solve_dense_dev",
    "clp_score_custom", "clp_score_custom_dev", "clp_invariant_check", "clp_jit_stats",
    "clp_batch_solve_custom", "clp_batch_max_clique_custom",
    "clp_batch_solve_euclidean_dev", "clp_batch_solve_pointnormal_dev", "clp_batch_solve_custom_dev",
    "clp_batch_max_clique_euclidean_dev", "clp_batch_max_clique_pointnormal_dev", "clp_batch_max_clique_custom_dev",
    "clp_sdp_default_params", "clp_sdp_solve", "clp_batch_sdp_matrices",
    "clp_correspondences", "clp_correspondences_dev",
]
INV_MAX_PARAMS = 16
MC_EXACT, MC_HEU, MC_KCORE = 0, 1, 2
SDP_MAX_M = 128
KNN_MAX_K, KNN_MAX_D = 32, 64


class ClpParams(C.Structure):
    """POD mirror of clipper::Params (reference include/clipper/clipper.h:27-60)."""
    _fields_ = [
        ("tol_u", C.c_double), ("tol_F", C.c_double), ("tol_Fop", C.c_double),
        ("maxiniters", C.c_int32), ("maxoliters", C.c_int32),
        ("beta", C.c_double), ("maxlsiters", C.c_int32),
        ("eps", C.c_double), ("affinityeps", C.c_double),
        ("rescale_u0", C.c_int32), ("rounding", C.c_int32),
    ]


class ClpSolution(C.Structure):
    """POD mirror of clipper::Solution (reference include/clipper/clipper.h:65-73) + counters."""
    _fields_ = [
        ("t", C.c_double), ("ifinal", C.c_int32), ("n_nodes", C.c_int32),
        ("score", C.c_double), ("d_final", C.c_double),
        ("n_evals", C.c_int64), ("n_matvec", C.c_int64), ("n_inner", C.c_int64),
        ("kernel_ms", C.c_double),
        ("prof_matvec_ms", C.c_double), ("prof_combine_ms", C.c_double), ("prof_exchange_ms", C.c_double),
    ]


class ClpMcInfo(C.Structure):
    """clp_mc_info: statistics of one clp_max_clique call."""
    _fields_ = [
        ("n_nodes", C.c_int32), ("max_core", C.c_int32), ("lower_bound", C.c_int32), ("upper_bound", C.c_int32),
        ("proven", C.c_int32), ("timed_out", C.c_int32), ("n_edges", C.c_int64), ("n_branches", C.c_int64),
        ("t", C.c_double), ("kernel_ms", C.c_double),
        ("adjacency_ms", C.c_double), ("peel_ms", C.c_double), ("heuristic_ms", C.c_double), ("search_ms", C.c_double),
    ]


class ClpSdpParams(C.Structure):
    """clp_sdp_params: parameters of the semidefinite relaxation (clp_sdp_solve, clp_batch_sdp_matrices)."""
    _fields_ = [("max_iters", C.c_int32), ("eps_abs", C.c_double), ("eps_rel", C.c_double), ("time_limit_s", C.c_double)]


class ClpSdpInfo(C.Structure):
    """clp_sdp_info: outcome and statistics of one relaxation."""
    _fields_ = [
        ("iters", C.c_int32), ("converged", C.c_int32), ("timed_out", C.c_int32), ("n_nodes", C.c_int32),
        ("value", C.c_double), ("bound", C.c_double), ("res_pri", C.c_double), ("res_dual", C.c_double),
        ("rho", C.c_double), ("thr", C.c_double), ("n_sweeps", C.c_int64),
        ("t", C.c_double), ("kernel_ms", C.c_double), ("proj_ms", C.c_double),
    ]


class ClpPointsDev(C.Structure):
    """clp_points_dev: point clouds and associations of a batch on the device (element strides), sizes on the host."""
    _fields_ = [
        ("D1", C.c_void_p), ("d1_strides", C.c_int64 * 3), ("D2", C.c_void_p), ("d2_strides", C.c_int64 * 3),
        ("A", C.c_void_p), ("a_strides", C.c_int64 * 3),
        ("n1", C.POINTER(C.c_int64)), ("n2", C.POINTER(C.c_int64)), ("m", C.POINTER(C.c_int64)),
    ]


class ClipperError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("clipper_b200 error %d: %s" % (code, msg))
        self.code = code


_lib = None


def load():
    """Load libclipper_b200.so and declare prototypes.  Raises if the library is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "clipper_b200: %s is missing -- run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  There is no CPU fallback." % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    dp, ip, lp = C.POINTER(C.c_double), C.POINTER(C.c_int32), C.POINTER(C.c_int64)
    i32, i64, dbl = C.c_int32, C.c_int64, C.c_double

    L.clp_create.argtypes = [C.c_int, C.c_int, C.POINTER(vp)]
    L.clp_destroy.argtypes = [vp]
    L.clp_last_error.argtypes = [vp]; L.clp_last_error.restype = C.c_char_p
    L.clp_version.restype = C.c_char_p
    L.clp_default_params.argtypes = [C.POINTER(ClpParams)]; L.clp_default_params.restype = None
    L.clp_set_params.argtypes = [vp, C.POINTER(ClpParams)]
    L.clp_get_params.argtypes = [vp, C.POINTER(ClpParams)]
    L.clp_set_stream.argtypes = [vp, vp]
    # host-pointer scoring takes typed pointers; *_dev variants take raw addresses (void*)
    L.clp_score_euclidean.argtypes = [vp, dp, i32, i64, dp, i64, ip, i64, dbl, dbl, dbl]
    L.clp_score_pointnormal.argtypes = [vp, dp, i64, dp, i64, ip, i64, dbl, dbl, dbl, dbl]
    L.clp_score_euclidean_dev.argtypes = [vp, vp, i32, i64, vp, i64, vp, i64, dbl, dbl, dbl]
    L.clp_score_pointnormal_dev.argtypes = [vp, vp, i64, vp, i64, vp, i64, dbl, dbl, dbl, dbl]
    L.clp_score_custom.argtypes = [vp, C.c_char_p, dp, i32, dp, i32, i64, dp, i64, ip, i64]
    L.clp_score_custom_dev.argtypes = [vp, C.c_char_p, dp, i32, vp, i32, i64, vp, i64, vp, i64]
    L.clp_invariant_check.argtypes = [C.c_char_p, i32, C.c_char_p, i64]
    L.clp_jit_stats.argtypes = [lp, dp]
    L.clp_set_dense.argtypes = [vp, dp, dp, i64]
    L.clp_set_dense_dev.argtypes = [vp, vp, vp, i64, C.c_int, i64, i64]
    L.clp_set_sparse_upper.argtypes = [vp, i64, lp, ip, dp, lp, ip, dp]
    L.clp_get_dense.argtypes = [vp, C.c_int, dp]
    L.clp_num_associations.argtypes = [vp, lp]
    L.clp_get_associations.argtypes = [vp, ip]
    L.clp_count_nonzeros.argtypes = [vp, lp, lp]
    L.clp_solve.argtypes = [vp, dp, C.POINTER(ClpSolution), dp, ip, dp]
    L.clp_solve_dev.argtypes = [vp, vp, C.POINTER(ClpSolution), vp, ip]
    L.clp_matvec.argtypes = [vp, dp, dbl, dp, dp, dp]
    L.clp_matvec_dev.argtypes = [vp, vp, dbl, vp, vp, vp, C.c_int, dp]
    L.clp_k2ij.argtypes = [C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.clp_k2ij.restype = None
    L.clp_create_all_to_all.argtypes = [i64, i64, ip]; L.clp_create_all_to_all.restype = None
    L.clp_find_k_largest.argtypes = [dp, i64, i32, ip]; L.clp_find_k_largest.restype = i32
    L.clp_find_above.argtypes = [dp, i64, dbl, ip]; L.clp_find_above.restype = i32
    L.clp_dsd_dense.argtypes = [dp, i64, ip, i32, ip]; L.clp_dsd_dense.restype = i32
    L.clp_shard_config.argtypes = [vp, C.c_int, C.c_int]
    L.clp_shard_blob_bytes.restype = i64
    L.clp_shard_export.argtypes = [vp, vp, i64, lp]
    L.clp_shard_import.argtypes = [vp, vp, i64, C.c_int]
    L.clp_shard_rows.argtypes = [i64, C.c_int, C.c_int, lp, lp]; L.clp_shard_rows.restype = None
    L.clp_set_ctas_per_sm.argtypes = [vp, C.c_int]
    L.clp_set_grid_cap.argtypes = [vp, C.c_int]
    L.clp_set_dense_mode.argtypes = [vp, C.c_int]
    L.clp_get_dense_mode.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.clp_sparse_info.argtypes = [vp, lp, lp]
    # batches of small problems: arrays of host pointers (void**) and sizes
    pp = C.POINTER(C.c_void_p)
    L.clp_batch_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.clp_batch_destroy.argtypes = [vp]
    L.clp_batch_last_error.argtypes = [vp]; L.clp_batch_last_error.restype = C.c_char_p
    L.clp_batch_set_params.argtypes = [vp, C.POINTER(ClpParams)]
    L.clp_batch_solve_euclidean.argtypes = [vp, i32, i32, pp, lp, pp, lp, pp, lp, pp, dbl, dbl, dbl,
                                            C.POINTER(ClpSolution), pp, pp]
    L.clp_batch_solve_pointnormal.argtypes = [vp, i32, pp, lp, pp, lp, pp, lp, pp, dbl, dbl, dbl, dbl,
                                              C.POINTER(ClpSolution), pp, pp]
    L.clp_batch_solve_matrices.argtypes = [vp, i32, lp, pp, pp, pp, pp, pp, pp, pp, C.POINTER(ClpSolution), pp, pp]
    L.clp_batch_set_stream.argtypes = [vp, vp]
    L.clp_batch_solve_dense_dev.argtypes = [vp, i32, lp, C.c_int, vp, vp, i64, i64, i64, vp, i64, C.POINTER(ClpSolution),
                                            vp, i64, pp]
    L.clp_batch_info.argtypes = [vp, ip, lp, lp]
    L.clp_max_clique.argtypes = [vp, C.c_int, dbl, ip, C.POINTER(ClpMcInfo)]
    L.clp_core_numbers.argtypes = [vp, ip]
    mip = C.POINTER(ClpMcInfo)
    L.clp_batch_max_clique_euclidean.argtypes = [vp, i32, i32, pp, lp, pp, lp, pp, lp, dbl, dbl, dbl, C.c_int, dbl,
                                                 mip, pp, pp]
    L.clp_batch_max_clique_pointnormal.argtypes = [vp, i32, pp, lp, pp, lp, pp, lp, dbl, dbl, dbl, dbl, C.c_int, dbl,
                                                   mip, pp, pp]
    L.clp_batch_max_clique_graphs.argtypes = [vp, i32, lp, pp, pp, C.c_int, dbl, mip, pp, pp]
    L.clp_batch_solve_custom.argtypes = [vp, C.c_char_p, dp, i32, i32, i32, pp, lp, pp, lp, pp, lp, pp,
                                         C.POINTER(ClpSolution), pp, pp]
    L.clp_batch_max_clique_custom.argtypes = [vp, C.c_char_p, dp, i32, i32, i32, pp, lp, pp, lp, pp, lp, C.c_int, dbl,
                                              mip, pp, pp]
    # batches on the device: clp_points_dev, device u0 / u (void*), host solutions and nodes
    ptp, sp = C.POINTER(ClpPointsDev), C.POINTER(ClpSolution)
    L.clp_batch_solve_euclidean_dev.argtypes = [vp, i32, i32, ptp, vp, i64, dbl, dbl, dbl, sp, vp, i64, pp]
    L.clp_batch_solve_pointnormal_dev.argtypes = [vp, i32, ptp, vp, i64, dbl, dbl, dbl, dbl, sp, vp, i64, pp]
    L.clp_batch_solve_custom_dev.argtypes = [vp, C.c_char_p, dp, i32, i32, i32, ptp, vp, i64, sp, vp, i64, pp]
    L.clp_batch_max_clique_euclidean_dev.argtypes = [vp, i32, i32, ptp, dbl, dbl, dbl, C.c_int, dbl, mip, pp, pp]
    L.clp_batch_max_clique_pointnormal_dev.argtypes = [vp, i32, ptp, dbl, dbl, dbl, dbl, C.c_int, dbl, mip, pp, pp]
    L.clp_batch_max_clique_custom_dev.argtypes = [vp, C.c_char_p, dp, i32, i32, i32, ptp, C.c_int, dbl, mip, pp, pp]
    L.clp_sdp_default_params.argtypes = [C.POINTER(ClpSdpParams)]; L.clp_sdp_default_params.restype = None
    L.clp_sdp_solve.argtypes = [vp, C.POINTER(ClpSdpParams), C.POINTER(ClpSdpInfo), ip, dp, dp, dp]
    L.clp_batch_sdp_matrices.argtypes = [vp, i32, lp, pp, pp, pp, pp, pp, pp, C.POINTER(ClpSdpParams),
                                         C.POINTER(ClpSdpInfo), pp, pp, pp, pp]
    L.clp_correspondences.argtypes = [vp, dp, i32, i64, dp, i64, i32, dbl, C.c_int, ip, i64, lp]
    L.clp_correspondences_dev.argtypes = [vp, vp, i32, i64, vp, i64, i32, dbl, C.c_int, vp, i64, lp]
    _lib = L
    return L


def check(h, rc):
    if rc != OK:
        msg = load().clp_last_error(h)
        raise ClipperError(rc, msg.decode() if msg else "")
