"""Fixtures restated from the reference's own tests / examples (values only, no code).

toy_problem()      reference test/affinity_test.cpp:33-48 and test/clipper_test.cpp:34-49
MTRUE_12           reference test/affinity_test.cpp:94-106 (12x12 0/1 literal "from MATLAB")
M20                reference test/sdp_test.cpp:17-37 == test/dsd_test.cpp:16-36 (20x20 weighted M)
DSD_NODES_20       reference test/dsd_test.cpp:15
planecloud()       reference examples/matlab/ex3_planecloud.m:18-33,79-86
"""
import numpy as np


def toy_problem():
    """4-point model, data = T_MD^-1 * model with T_MD = (Rz(pi/8), t=(5,3,0)), first 3 points."""
    model = np.array([[0, 0, 0], [2, 0, 0], [0, 3, 0], [2, 2, 0]], dtype=np.float64).T  # 3x4
    th = np.pi / 8
    R = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]], dtype=np.float64)
    t = np.array([5.0, 3.0, 0.0])
    data = R.T @ (model - t[:, None])  # inverse rigid transform
    return np.asfortranarray(model), np.asfortranarray(data[:, :3])


MTRUE_12 = np.array([
    [1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0],
    [0, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0],
    [0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 0, 0],
    [0, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1, 0],
    [1, 0, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0],
    [0, 0, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0],
    [0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 0, 0],
    [0, 0, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0],
    [1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0],
    [0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0],
    [0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 1, 0],
    [0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1]], dtype=np.float64)

# upper-triangle (i<j) non-zeros of the 20x20 literal; the matrix is symmetric with unit diagonal
_M20_UPPER = {
    (0, 18): 0.2964, (1, 13): 0.0138, (2, 11): 0.0016, (2, 18): 0.0747,
    (3, 5): 0.0555, (3, 6): 0.2547, (3, 13): 0.0102, (3, 15): 0.7715,
    (4, 5): 0.0063, (4, 7): 0.3846, (4, 9): 0.0003, (4, 10): 0.0014, (4, 15): 0.0063,
    (5, 12): 0.9927, (5, 15): 0.9722, (6, 8): 0.0023, (6, 11): 0.8775, (7, 8): 0.0001,
    (8, 9): 0.7914, (8, 13): 0.0617, (8, 16): 0.9938, (8, 19): 0.0007,
    (9, 12): 0.0001, (9, 13): 0.0091, (9, 15): 0.2503, (9, 16): 0.0222, (9, 17): 0.0549,
    (10, 19): 0.0008, (11, 18): 0.7007, (12, 14): 0.9978, (13, 17): 0.0003,
    (14, 15): 0.0012, (14, 19): 0.0074, (15, 16): 0.0026, (15, 17): 0.0217, (17, 18): 0.0007,
}


def m20():
    M = np.eye(20, dtype=np.float64)
    for (i, j), v in _M20_UPPER.items():
        M[i, j] = v; M[j, i] = v
    C = (M > 0).astype(np.float64)
    return M, C


DSD_NODES_20 = [3, 5, 12, 14, 15]


def bytes_per_pass(kept, packed, esize=4):
    """what one pass over the whole-row compact copy reads: entries (kept + one filler per empty 16-column window when
    packed), rows sorted by length, four per item padded to the longest, plus 20 bytes of descriptors per item.
    kept: the m x m boolean pattern of the stored off-diagonal entries, dense or scipy.sparse; esize: bytes of a stored
    value (a 6-byte entry of fp32 storage is the value and a 16-bit column index)"""
    import scipy.sparse as sp
    m = kept.shape[0]
    nwin = (m + 15) // 16
    if sp.issparse(kept):
        K = sp.csr_matrix(kept, dtype=bool); K.eliminate_zeros(); K.sort_indices()
        lens = np.diff(K.indptr).astype(np.int64)
        rows = np.repeat(np.arange(m, dtype=np.int64), lens)
        occ = np.bincount(np.unique(rows * nwin + K.indices // 16) // nwin, minlength=m)
    else:
        lens = kept.sum(1).astype(np.int64)
        occ = np.pad(kept, ((0, 0), (0, 16 * nwin - m))).reshape(m, nwin, 16).any(2).sum(1)
    if packed:
        lens = lens + (nwin - occ)
    rows_pad = -(-m // 32) * 32
    cls = np.zeros(rows_pad, np.int64)
    cls[:m] = (lens + 3) // 4
    stored = 16 * int(np.sort(cls)[::-1][0::4].sum())
    return (4 if packed else esize + 2) * stored + rows_pad // 4 * 20


def planecloud():
    """Plane normals of two LiDAR scans as 6xn point-normal data with zeroed points."""
    D1 = np.array([
        [0.99778409, -0.02919371, -0.05978833, 1.84071578],
        [0.00655776, -0.34994794, 0.93674619, 5.81443529],
        [0.03067185, 0.93082657, 0.36417186, -22.82330860],
        [-0.03095734, 0.91232313, 0.40829902, -24.11912204]], dtype=np.float64).T
    D2 = np.array([
        [-0.07169808126, 0.855164861, 0.513373592, -28.65209536],
        [0.99514624580, 0.078913239, 0.058793283, -21.00096958],
        [-0.00156293830, -0.344498312, 0.938785636, 5.98810865],
        [0.08368147539, -0.930524190, -0.356541920, 29.41486128]], dtype=np.float64).T
    DD1 = np.asfortranarray(np.vstack([np.zeros((3, 4)), D1[:3, :]]))
    DD2 = np.asfortranarray(np.vstack([np.zeros((3, 4)), D2[:3, :]]))
    Agt0 = np.array([[0, 3], [1, 2], [2, 1]], dtype=np.int32)  # 1-based [1 4;2 3;3 2]
    params = dict(sigp=0.5, epsp=0.5, sign=np.deg2rad(1.5), epsn=1.0)
    return DD1, DD2, Agt0, params
