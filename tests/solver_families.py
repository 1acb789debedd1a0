"""Solver cases whose every decision is robust, and a numpy restatement of findDenseClique that measures each margin.

restate() follows the oracle's operation order (oracle/clipper_oracle.c orc_solve, reference clipper.cpp:172-310), down
to the order of every sum, so that it reproduces the oracle bit for bit, and records, at every decision the solver takes, how far the compared quantities are from flipping it:
  - the line-search test deltaF < -eps and the stop tests deltau < tol_u, |deltaF| < tol_F;
  - the per-row tests Cbu_i > eps and u_i > eps of the initial d and of every penalty ramp;
  - the sign of every entry of the projection max(u + alpha gradF, 0);
  - round(F) against the nearest half-integer (and against the clamp to [0, m]) for DSD_HEU;
  - the gaps between consecutive entries of the sorted top round(F) + 1 entries of u (DSD_HEU keeps them in order),
    and the sign of every entry of u (NONZERO and DSD keep the support).
A comparison is robust when its operands are exact in every summation order (exact zeros of the projection and of the
inputs, NaN, sums of exact zeros) or when its margin exceeds 1e4 * gamma(K) times the absolute sum of its terms, where
gamma(k) = k u / (1 - k u), u = 2^-53 (Higham, section 3.1), K = 2 m + max row count + 8 covers the longest sum of the
objective, and 1e4 allows for the error carried along the trajectory.  The tests on F (line search, stop tests,
round(F)) use 4 gamma(K) times their absolute sums without that factor: with it no case under the default eps and tol_F
would be usable, and a carried error in u moves F and Fnew alike near a fixed point, though that is not proven here.
A case is usable only when every decision is robust.  The rule is a screen rather than a proof: it rejects every case
whose decisions lie within local rounding of their thresholds, which is what makes identical counts (ifinal, n_evals,
n_inner) and identical nodes a reasonable assertion across summation orders.

Every matrix here holds fp32-representable, non-negative weights and binary constraints, so fp32 and fp64 storage
store the same matrix and one oracle run is the reference for every door.  The scored problems (T8) are the exception:
their reference is the matrix each storage actually holds.
"""
import math

import numpy as np
import scipy.sparse as sp

U = 2.0 ** -53
CARRY = 1e4


def gamma(k):
    return k * U / (1.0 - k * U)


# ---- the restatement -----------------------------------------------------------------------------------------------
class Margins:
    """the worst decision seen: robust stays True while every comparison is exact or outside its bound"""

    def __init__(self):
        self.robust = True
        self.worst = None    # (ratio margin / bound, what, margin, bound)
        self.zero_candidates = 0

    def test(self, what, x, thr, bound):
        """comparisons x > thr (or x < thr) for arrays x with absolute rounding bounds; bound 0 or NaN operands are
        exact"""
        x = np.asarray(x, np.float64); bound = np.broadcast_to(np.asarray(bound, np.float64), x.shape)
        margin = np.abs(x - thr)
        ok = ~(margin <= bound) | (bound == 0) | np.isnan(x)
        return self._note(what, ok, margin, bound)

    def _note(self, what, ok, margin, bound):
        ok = np.asarray(ok, bool)
        if not ok.all():
            self.robust = False
            k = int(np.flatnonzero(~ok)[0])
            r = float(np.ravel(margin)[k] / np.ravel(bound)[k])
            if self.worst is None or r < self.worst[0]:
                self.worst = (r, what, float(np.ravel(margin)[k]), float(np.ravel(bound)[k]))
        return ok


def _seq(x):
    """left-to-right sum, as the oracle's loops add (np.sum adds pairwise)"""
    return float(np.cumsum(x)[-1]) if np.size(x) else 0.0


class _SeqMatVec:
    """y = S x with each row summed left to right in ascending column order: the order of the oracle's column sweep
    over the strict upper triangle (row i gathers its entries above the diagonal first, then receives those of the
    later columns in order)"""

    def __init__(self, S):
        S = sp.csr_matrix(S, dtype=np.float64, copy=True)
        S.sum_duplicates(); S.sort_indices()
        self.S = S
        self.len = np.diff(S.indptr)
        self.kmax = int(self.len.max()) if self.len.size else 0

    def __matmul__(self, x):
        S = self.S
        p = S.data * x[S.indices]
        y = np.zeros(S.shape[0])
        start = S.indptr[:-1]
        for t in range(self.kmax):
            rows = np.flatnonzero(self.len > t)
            y[rows] = y[rows] + p[start[rows] + t]
        return y


def _p(P, name):
    return P[name] if isinstance(P, dict) else getattr(P, name)


def restate(Mh, Ch, u0, P, dsd=None):
    """findDenseClique on the stored matrix (Mh, Ch: symmetric off-diagonal parts, scipy, fp64) from u0 with params P
    (dict or object with the Params fields).  dsd(support) -> nodes is called for Rounding::DSD.  Returns a dict with
    ifinal, n_evals, n_inner, d_final, score, u, nodes, trace (rows F, d used, inner steps) and margins."""
    Mh, Ch = sp.csr_matrix(Mh, dtype=np.float64), sp.csr_matrix(Ch, dtype=np.float64)
    aM, aC = abs(Mh), abs(Ch)
    Mh, Ch = _SeqMatVec(Mh), _SeqMatVec(Ch)
    m = Mh.S.shape[0]
    kmax = int(np.diff(((aM + aC) != 0).tocsr().indptr).max()) if m else 0
    GL = 4 * gamma(2 * m + kmax + 8)     # rounding of one evaluation, kernel and reference each
    G = CARRY * gamma(2 * m + kmax + 8)  # an entry of u, with the error carried along the trajectory
    eps, beta = float(_p(P, "eps")), float(_p(P, "beta"))
    tol_u, tol_F = float(_p(P, "tol_u")), float(_p(P, "tol_F"))
    maxol, maxin, maxls = int(_p(P, "maxoliters")), int(_p(P, "maxiniters")), int(_p(P, "maxlsiters"))
    rounding = int(_p(P, "rounding"))
    mg = Margins()
    u0 = np.asarray(u0, np.float64)
    n_evals = n_inner = 0

    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        if _p(P, "rescale_u0"):
            u = Mh @ u0 + u0
            su = aM @ np.abs(u0) + np.abs(u0)
        else:
            u = u0.copy()
            su = np.abs(u0)
        nrm = math.sqrt(_seq(u * u))
        u = u / nrm
        su = su / nrm

        def objective(v, d):
            """gradF and F of v under d (clipper.cpp:219-220) with the absolute sums of their terms"""
            S = _seq(v)
            Mv, Cv = Mh @ v, Ch @ v
            g = (((1 + d) * v - (d * 1.0) * S) + Mv) + Cv * d
            av = np.abs(v)
            gabs = (1 + abs(d)) * av + abs(d) * av.sum() + aM @ av + abs(d) * (aC @ av)
            return g, _seq(v * g), gabs, float(np.dot(av, gabs)), Mv, Cv

        def rows_pass(v, sv, Cv, what):
            """the per-row test Cbu_i > eps && u_i > eps, with its robustness"""
            S = _seq(v)
            cbu = (1.0 * S - Cv) - v
            av = np.abs(v)
            # Cbu_i sums the entries of u outside row i's constraint pattern: its local rounding, plus the carried error
            # of those entries only (the exact zeros of u carry none)
            carried = np.maximum((sv.sum() - aC @ sv) - sv, 0.0)
            okc = mg.test(what + " Cbu_i > eps", cbu, eps, GL * (av.sum() + aC @ av + av) + G * carried)
            passc, passu = cbu > eps, v > eps
            oku = (sv == 0) | ~(np.abs(v - eps) <= G * sv) | np.isnan(v)
            # the conjunction is decided when either side is robustly false or both are robust
            ok = (okc & ~passc) | (oku & ~passu) | (okc & oku)
            mg._note(what + " row", ok, np.abs(v - eps), G * sv + 1e-300)
            return passc & passu, cbu

        d = 0.0
        Cu = Ch @ u
        sel, cbu = rows_pass(u, su, Cu, "initial d")
        cnt = int(sel.sum())
        if cnt > 0:
            Mu = Mh @ u
            d = _seq((Mu[sel] + u[sel]) / cbu[sel]) / cnt   # mean, no abs (clipper.cpp:208)

        F = 0.0
        trace = []
        i = 0
        while i < maxol:
            g, F, gabs, Babs, _, _ = objective(u, d)
            d_used = d
            j = 0
            while j < maxin:
                alpha = 1.0
                Fnew = deltaF = 0.0
                k = 0
                while k < maxls:
                    w = u + alpha * g
                    mg.test("projection sign", w, 0.0, G * (su + alpha * gabs))
                    w = np.where(w < 0, 0.0, w)
                    sw_ = np.where(w == 0, 0.0, su + alpha * gabs)   # exact zeros stay exact
                    z = _seq(w * w)
                    if z > 0:
                        s = math.sqrt(z)
                        unew, sunew = w / s, sw_ / s
                    else:
                        if z == 0:
                            mg.zero_candidates += 1
                        unew, sunew = w, sw_
                    gn, Fnew, gabsn, Babsn, _, _ = objective(unew, d)
                    n_evals += 1
                    deltaF = Fnew - F
                    mg.test("line search deltaF < -eps", deltaF, -eps, GL * (Babs + Babsn))
                    if deltaF < -eps:
                        alpha = alpha * beta
                        k += 1
                    else:
                        break
                deltau = math.sqrt(_seq((unew - u) * (unew - u)))
                bu = G * (math.sqrt(float(np.dot(su, su))) + math.sqrt(float(np.dot(sunew, sunew))))
                bF = GL * (Babs + Babsn)
                stop_u, stop_F = deltau < tol_u, abs(deltaF) < tol_F
                oku = bool(not (abs(deltau - tol_u) <= bu) or bu == 0 or math.isnan(deltau))
                okF = bool(not (abs(abs(deltaF) - tol_F) <= bF) or bF == 0 or math.isnan(deltaF))
                if not ((oku and stop_u) or (okF and stop_F) or (oku and okF)):
                    mg._note("stop test deltau < tol_u || |deltaF| < tol_F", [False], [abs(abs(deltaF) - tol_F)], [bF])
                F, u, su, g, gabs, Babs = Fnew, unew, sunew, gn, gabsn, Babsn
                n_inner += 1
                j += 1
                if stop_u or stop_F:
                    break
            trace.append((F, d_used, j))
            Cu = Ch @ u
            sel, cbu = rows_pass(u, su, Cu, "penalty ramp")
            cnt = int(sel.sum())
            if cnt > 0:
                Mu = Mh @ u
                d += _seq(np.abs((Mu[sel] + u[sel]) / cbu[sel])) / cnt   # abs().mean() (clipper.cpp:274)
            else:
                break
            i += 1

        # rounding (clipper.cpp:287-310)
        if rounding == 2:
            r = round_half_away(F)
            omega = 0 if not (r >= 1) else min(int(r), m)
            if not math.isnan(F):
                bF = GL * Babs if maxol > 0 else 0.0
                if F > m + 0.5 + bF or F < 0.5 - bF:
                    pass                                   # the clamp decides
                else:
                    mg.test("round(F) vs half-integer", abs(F - math.floor(F) - 0.5), 0.0, bF)
            nodes = find_k_largest(u, omega)
            if omega > 0:
                top = np.argsort(-u, kind="stable")[: min(omega + 1, m)]
                gap = u[top[:-1]] - u[top[1:]]
                bound = G * (su[top[:-1]] + su[top[1:]])
                exact = (u[top[:-1]] == 0) & (u[top[1:]] == 0)
                mg._note("DSD_HEU order gap", exact | ~(gap <= bound), gap, bound)
        else:
            mg.test("support u_i > 0", u, 0.0, G * su)
            supp = np.flatnonzero(u > 0)
            if rounding == 0:
                nodes = supp.astype(np.int32)
            else:
                nodes = np.asarray(dsd(supp) if supp.size else [], np.int32)
    return dict(ifinal=i, n_evals=n_evals, n_inner=n_inner, d_final=d, score=F, u=u, nodes=np.asarray(nodes, np.int32),
                trace=np.array(trace, np.float64).reshape(-1, 3), margins=mg)


def round_half_away(x):
    return math.floor(abs(x) + 0.5) * (1 if x >= 0 else -1) if math.isfinite(x) else x


def find_k_largest(x, k):
    """the reference's bounded heap (utils.cpp:33-55), through the oracle's statement of it"""
    from oracle import clipper_oracle as orc
    return orc.find_k_largest(x, k) if k >= 1 else np.zeros(0, np.int32)


# ---- the cases -----------------------------------------------------------------------------------------------------
DEFAULTS = dict(tol_u=1e-8, tol_F=1e-9, tol_Fop=1e-10, maxiniters=200, maxoliters=1000, beta=0.25, maxlsiters=99,
                eps=1e-9, affinityeps=1e-4, rescale_u0=True, rounding=2)

# the parameter grid (overrides of the defaults)
GRID = {
    "defaults": {},
    "maxoliters0": dict(maxoliters=0),
    "maxoliters1": dict(maxoliters=1),
    "maxoliters2": dict(maxoliters=2),
    "maxiniters1": dict(maxiniters=1),
    "maxiniters3": dict(maxiniters=3),
    "maxlsiters1": dict(maxlsiters=1),
    "maxlsiters2": dict(maxlsiters=2),
    "beta0.5_eps1e-3": dict(beta=0.5, eps=1e-3),
    "tolu0_tolF1e-3": dict(tol_u=0.0, tol_F=1e-3),
    "tolu1e-2_tolF0": dict(tol_u=1e-2, tol_F=0.0),
    "eps0": dict(eps=0.0),
    "nonzero": dict(rounding=0),
    "dsd": dict(rounding=1),
}
# the parameters every door runs
DOOR_GRID = ("defaults", "maxlsiters1", "maxiniters3", "norescale")
GRID["norescale"] = dict(rescale_u0=False)
GRID["short"] = dict(maxoliters=1, maxiniters=3)
GRID["short1"] = dict(maxoliters=1, maxiniters=1)
GRID["short2"] = dict(maxoliters=2, maxiniters=1)
# scored problems: with the default tolerances their stop test |deltaF| < tol_F is decided by less than its rounding
# bound, so they run short trajectories whose every decision is robust
T8_GRID = ("short", "short2")


def params(name):
    P = dict(DEFAULTS)
    P.update(GRID[name])
    return P


def f32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


class Case:
    """a solver problem: Mh, Ch the symmetric off-diagonal parts of the matrix (fp32-representable weights, binary
    constraints), u0, and the family claim checked on the restatement's run with default parameters"""

    def __init__(self, name, family, Mh, Ch, u0, claim=None, grid=None):
        self.name, self.family = name, family
        self.Mh, self.Ch = sp.csr_matrix(Mh), sp.csr_matrix(Ch)
        self.Mh.eliminate_zeros(); self.Ch.eliminate_zeros()
        self.m = self.Mh.shape[0]
        self.u0 = np.asarray(u0, np.float64)
        self.claim = claim
        self.grid = grid   # the parameter sets the GPU file runs on this case (None: the door's own list)

    def dense(self):
        """(M, C) with unit diagonal, as set_matrix_data takes them"""
        I = np.eye(self.m)
        return np.asfortranarray(self.Mh.toarray() + I), np.asfortranarray(self.Ch.toarray() + I)

    def upper(self):
        """(M, C) strictly upper triangular scipy CSC, as set_sparse_matrix_data takes them"""
        return sp.triu(self.Mh, 1, format="csc"), sp.triu(self.Ch, 1, format="csc")

    def oracle(self, P, trace_cap=0):
        """the C oracle on this matrix"""
        from oracle import clipper_oracle as orc
        o = orc.Oracle(orc.default_params(**{k: (int(v) if isinstance(v, bool) else v) for k, v in P.items()}))
        if self.m <= 4096:
            o.set_matrix_data(*self.dense())
        else:
            Mu, Cu = self.upper()
            Mu.sort_indices(); Cu.sort_indices()
            o.set_sparse_upper(self.m, Mu.indptr, Mu.indices, Mu.data, Cu.indptr, Cu.indices, Cu.data)
        return o, o.solve(self.u0, trace_cap=trace_cap)

    def restate(self, P):
        from oracle import clipper_oracle as orc
        M = self.Mh
        return restate(self.Mh, self.Ch, self.u0, P,
                       dsd=lambda S: orc.dsd_solve((M + sp.eye(self.m)).toarray(), S))


def _pairs(m, i, j, w, c):
    """symmetric Mh, Ch from pairs i < j with weights w (rounded to fp32) and constraints c"""
    w, c = f32(w), (np.asarray(c) != 0).astype(np.float64)
    ii, jj = np.concatenate([i, j]), np.concatenate([j, i])
    Mh = sp.csr_matrix((np.concatenate([w, w]), (ii, jj)), shape=(m, m))
    Ch = sp.csr_matrix((np.concatenate([c, c]), (ii, jj)), shape=(m, m))
    return Mh, Ch


def _clique_pairs(nodes):
    a, b = np.triu_indices(len(nodes), 1)
    nodes = np.asarray(nodes)
    return nodes[a], nodes[b]


def _random_pairs(rng, nodes, density):
    nodes = np.asarray(nodes)
    a, b = np.triu_indices(nodes.size, 1)
    keep = rng.random(a.size) < density
    return nodes[a[keep]], nodes[b[keep]]


def planted(m, seed, k=None, density=None, scale=1.0, isolated=0):
    """a clique of k nodes with weights U[0.6, 1), random pairs U[0.05, 0.5) among the other non-isolated nodes"""
    rng = np.random.default_rng(seed)
    k = k if k is not None else max(2, min(m, m // 8))
    perm = rng.permutation(m)
    cl, rest = np.sort(perm[:k]), np.sort(perm[k:m - isolated])
    i1, j1 = _clique_pairs(cl)
    density = density if density is not None else min(0.1, 8.0 / max(m, 1))
    i2, j2 = _random_pairs(rng, np.concatenate([cl, rest]), density)
    key = set(zip(i1.tolist(), j1.tolist()))
    extra = np.array([(a, b) not in key for a, b in zip(i2.tolist(), j2.tolist())], bool)
    i2, j2 = i2[extra], j2[extra]
    i, j = np.concatenate([i1, i2]), np.concatenate([j1, j2])
    lo, hi = np.minimum(i, j), np.maximum(i, j)
    w = np.concatenate([rng.uniform(0.6, 1.0, i1.size), rng.uniform(0.05, 0.5, i2.size)]) * scale
    Mh, Ch = _pairs(m, lo, hi, w, np.ones(lo.size))
    return Mh, Ch, cl, np.sort(perm[m - isolated:]), rng.random(m) + 0.05


def _no_pairs(m):
    return sp.csr_matrix((m, m)), sp.csr_matrix((m, m))


def families():
    """every case, by name"""
    out = []
    rng = np.random.default_rng(20261018)

    # T1 edgeless: C = I, with (M > 0, C = 0) weights; the ramp drives u to a zero candidate
    m, r1 = 24, np.random.default_rng(1)
    i, j = _random_pairs(r1, np.arange(m), 0.2)
    Mh, _ = _pairs(m, i, j, r1.uniform(0.05, 1.0, i.size), np.zeros(i.size))
    out.append(Case("T1_edgeless", "T1", Mh, sp.csr_matrix((m, m)), 1.0 + 0.2 * r1.random(m),
                    claim=("a zero candidate occurs", lambda c, r: r["margins"].zero_candidates > 0)))
    Mh, Ch = _no_pairs(24)
    out.append(Case("T1_empty", "T1", Mh, Ch, rng.random(24) + 0.05,
                    claim=("one node survives", lambda c, r: r["nodes"].size == 1)))

    # T2 complete graph: d stays 0, the ramp breaks after the first outer iteration
    for m in (24, 33):
        i, j = _clique_pairs(np.arange(m))
        Mh, Ch = _pairs(m, i, j, rng.uniform(0.5, 1.0, i.size), np.ones(i.size))
        out.append(Case("T2_complete_m%d" % m, "T2", Mh, Ch, rng.random(m) + 0.05,
                        claim=("d = 0, ramp breaks at once", lambda c, r: r["d_final"] == 0.0 and r["ifinal"] == 0)))

    # T3 isolated nodes beside a planted clique
    Mh, Ch, cl, iso, u0 = planted(48, 3, k=10, density=0.15, isolated=8)
    out.append(Case("T3_isolated", "T3", Mh, Ch, u0,
                    claim=("isolated rows are empty and end at 0",
                           lambda c, r, iso=iso: iso.size == 8 and c.Mh[iso].nnz == 0 and c.Ch[iso].nnz == 0
                           and np.all(r["u"][iso] == 0))))

    # T4 two disjoint cliques of equal size; u0 favours the first
    m, k = 40, 8
    perm = rng.permutation(m)
    A, B = np.sort(perm[:k]), np.sort(perm[k:2 * k])
    i1, j1 = _clique_pairs(A); i2, j2 = _clique_pairs(B)
    Mh, Ch = _pairs(m, np.concatenate([i1, i2]), np.concatenate([j1, j2]), rng.uniform(0.8, 1.0, 2 * i1.size),
                    np.ones(2 * i1.size))
    u0 = rng.uniform(0.2, 0.3, m); u0[A] += 0.3
    out.append(Case("T4_two_cliques", "T4", Mh, Ch, u0,
                    claim=("the favoured clique wins", lambda c, r, A=A: r["nodes"].size > 0
                           and set(r["nodes"].tolist()) <= set(A.tolist()))))

    # T5 mixed entries: (M = 0, C = 1) and (M > 0, C = 0) beside plain ones
    m = 80
    Mh, Ch, cl, _, u0 = planted(m, 5, k=9, density=0.12)
    U_ = sp.triu(Mh, 1).tocoo()
    sel = np.random.default_rng(6).random(U_.nnz)
    clset = set(cl.tolist())
    inside = np.array([a in clset and b in clset for a, b in zip(U_.row, U_.col)])
    w = np.where((sel < 0.15) & ~inside, 0.0, U_.data)
    c = np.where((sel > 0.85) & ~inside, 0.0, 1.0)
    Mh, Ch = _pairs(m, U_.row, U_.col, w, c)
    out.append(Case("T5_mixed", "T5", Mh, Ch, u0,
                    claim=("both odd kinds present", lambda c, r: (c.Ch - (c.Mh != 0).multiply(c.Ch)).nnz > 0
                           and ((c.Mh != 0) - (c.Mh != 0).multiply(c.Ch)).nnz > 0)))

    # T6 extreme weights
    m = 48
    i, j = _clique_pairs(np.arange(m))   # complete, so that d stays 0 and no penalty drowns the tiny affinities
    Mh, Ch = _pairs(m, i, j, rng.uniform(0.5, 1.0, i.size) * 2.0 ** -100, np.ones(i.size))
    out.append(Case("T6_tiny", "T6", Mh, Ch, rng.random(m) + 0.05,
                    claim=("weights near 2^-100", lambda c, r: 0 < c.Mh.data.max() < 2.0 ** -98)))
    # weights near 1e10 make F > 2^31; the tolerances mean nothing at that scale, so one short outer iteration
    Mh, Ch, _, _, u0 = planted(64, 8, k=8, scale=1e10)
    out.append(Case("T6_huge", "T6", Mh, Ch, u0,
                    claim=("F > 2^31 keeps all m nodes", lambda c, r: r["score"] > 2.0 ** 31 and r["nodes"].size == c.m),
                    grid=("short",)))

    # T7 sizes
    for m in (1, 2, 31, 32, 33, 127, 128, 129, 4096):
        # a small clique at m = 4096: with m // 8 members the gaps of the DSD_HEU order fall below their bound
        Mh, Ch, _, _, u0 = planted(m, 100 + m + (1000 if m in (127, 128) else 0), k=24 if m == 4096 else None)
        out.append(Case("T7_m%d" % m, "T7", Mh, Ch, u0, claim=("size", lambda c, r, m=m: c.m == m)))

    # u0 edges on a planted problem
    Mh, Ch, cl, _, u0 = planted(33, 9, k=6, density=0.2)
    z = u0.copy(); z[::3] = 0.0
    out.append(Case("U_zeros_norescale", "U", Mh, Ch, z, claim=("zeros in u0", lambda c, r: np.any(c.u0 == 0)),
                    grid=("norescale", "defaults")))
    one = np.zeros(33); one[cl[0]] = 1.0
    out.append(Case("U_single", "U", Mh, Ch, one, claim=("one non-zero", lambda c, r: np.count_nonzero(c.u0) == 1),
                    grid=("defaults", "norescale")))
    neg = u0.copy(); neg[1::4] = -neg[1::4]
    out.append(Case("U_negative", "U", Mh, Ch, neg, claim=("negative entries", lambda c, r: np.any(c.u0 < 0)),
                    grid=("defaults", "norescale")))
    out.append(Case("U_zero", "U", Mh, Ch, np.zeros(33),
                    claim=("u0 = 0 gives NaN and no node", lambda c, r: np.all(np.isnan(r["u"])) and r["nodes"].size == 0
                           and math.isnan(r["score"])), grid=("defaults", "maxiniters3", "nonzero")))
    return {c.name: c for c in out}


def big_case():
    """m = 27 649: one past the resident solver's limit, so mode 6 hands over to the segmented solver; few outer
    iterations keep it short"""
    Mh, Ch, _, _, u0 = planted(27649, 27649, k=24, density=6.0 / 27649)
    return Case("T9_m27649", "T9", Mh, Ch, u0, claim=("past the resident limit", lambda c, r: c.m == 27649),
                grid=("short", "short1", "short2"))


SCORED = (("c2", 100), ("c2", 3001), ("c3", 700))


def scored_case(name, m, f32_store):
    """T8: the matrix the oracle scores for datagen's problem; with f32_store the weights rounded to fp32 (what an fp32
    handle stores, up to the scoring kernel's last-bit differences, which the GPU test reads back instead)"""
    from clipper_b200 import datagen
    from oracle import clipper_oracle as orc
    prob = datagen.config_problem(name, m); cfg = prob["cfg"]
    o = orc.Oracle()
    if cfg["kind"] == "euclidean":
        o.score_euclidean(prob["D1"], prob["D2"], prob["A"], sigma=cfg["sigma"], epsilon=cfg["epsilon"])
    else:
        o.score_pointnormal(prob["D1"], prob["D2"], prob["A"], sigp=cfg["sigp"], epsp=cfg["epsp"], sign=cfg["sign"],
                            epsn=cfg["epsn"])
    M = o.get_affinity_matrix(); np.fill_diagonal(M, 0.0)
    Cm = o.get_constraint_matrix(); np.fill_diagonal(Cm, 0.0)
    if f32_store:
        M = f32(M)
    return Case("T8_%s_m%d" % (name, m), "T8", sp.csr_matrix(M), sp.csr_matrix(Cm), prob["u0"],
                claim=("scored", lambda c, r: c.Mh.nnz > 0))


# the parameter sets of the full grid on the default door and the solver_kernel door.  eps = 0 is in none: on every
# family here some comparison with eps = 0 is an exact tie in exact arithmetic (Cbu_i = 0 on a clique row, deltaF = 0
# at a fixed point), so its outcome depends on the summation order.
FULL_GRID = tuple(n for n in GRID if n not in ("dsd", "eps0", "short", "short1", "short2"))

# (case, parameter set) pairs left out, with the decision that is not robust
EXCLUDE = {
    ("T7_m129", "norescale"): "the stop test |deltaF| < tol_F of an inner step is decided by less than its bound",
}


def grid_for(case, names):
    """the parameter sets of `names` a case runs (its own grid when it has one), without the excluded pairs"""
    names = case.grid if case.grid else names
    return [g for g in names if (case.name, g) not in EXCLUDE]
