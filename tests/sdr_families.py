"""Problem families of the semidefinite relaxation tests: dense (M, C) pairs, symmetric with unit diagonals.

Scored families are scored by the CPU oracle here; the GPU tests score them on a handle and read the matrices back, so
the relaxation on both sides starts from the matrices the kernel sees."""
import numpy as np

import fixtures as fx
from clipper_b200 import datagen

SCORED = {  # name: (kind, m, seed)
    "euclid64": ("euclidean", 64, 11),
    "euclid127": ("euclidean", 127, 12),
    "euclid128": ("euclidean", 128, 13),
    "pointnormal96": ("pointnormal", 96, 14),
}


def scored_problem(name):
    kind, m, seed = SCORED[name]
    if kind == "euclidean":
        return kind, datagen.euclidean_problem(m, 0.8, seed)
    return kind, datagen.pointnormal_problem(m, 0.8, seed)


def given(name):
    """Families given as matrices (clp_set_dense): name -> (M, C)."""
    if name == "m20":
        return fx.m20()
    if name == "toy":
        return fx.MTRUE_12.copy(), fx.MTRUE_12.copy()
    if name == "dense_odd":  # pairs with M = 0, C = 1 and with M > 0, C = 0
        p = datagen.weighted_matrix_problem(40, 0.3, 21, odd=0.3)
        M = p["M"].toarray(); C = p["C"].toarray()
        M = M + M.T + np.eye(40); C = C + C.T + np.eye(40)
        return M, C
    if name == "m1":
        return np.ones((1, 1)), np.ones((1, 1))
    if name == "m2":
        M = np.array([[1.0, 0.5], [0.5, 1.0]])
        return M, np.ones((2, 2))
    if name == "eye":  # every eigenvalue of W is equal in the first iteration
        return np.eye(16), np.ones((16, 16))
    if name == "two_cliques":  # the top eigenvalue of M is double
        M = np.eye(10)
        for S in ((0, 1, 2, 3), (5, 6, 7, 8)):
            for i in S:
                for j in S:
                    if i != j:
                        M[i, j] = 0.9
        return M, (M > 0).astype(np.float64)
    raise KeyError(name)


GIVEN = ["m20", "toy", "dense_odd", "m1", "m2", "eye", "two_cliques"]


def oracle_scored(name):
    """Scored family through the CPU oracle's scoring: (M, C)."""
    from oracle import clipper_oracle as orc
    kind, p = scored_problem(name)
    o = orc.Oracle()
    if kind == "euclidean":
        o.score_euclidean(p["D1"], p["D2"], p["A"])
    else:
        o.score_pointnormal(p["D1"], p["D2"], p["A"])
    return o.get_affinity_matrix(), o.get_constraint_matrix()
