"""Matrix families that aim at the edges of the compact copies (DESIGN.md section 2), and host restatements of the rules
that decide how a matrix is stored: the packed gate (pack_window), the packed row encoding (fillers + 5-bit column
deltas), the column segmentation of the segmented sweep (make_plan) and the bytes one pass reads.

Every builder is deterministic and returns a Case: the strict upper triangle as pair lists (i < j) with the affinity
and the constraint value of each pair.  tests/test_packed_families.py checks on the CPU that each family contains what
it claims; tests/test_gpu_exact_products.py runs the kernels on them.
"""
import numpy as np
import scipy.sparse as sp

WIN = 16          # columns per packed window (kWinCols)
SEG_MAX = 4096    # kSegMax
RES_MAX_M = 27648  # kResMaxM: largest m of the resident (whole-row) layout


class Case:
    def __init__(self, name, m, i, j, mval, cval):
        i, j = np.asarray(i, np.int64), np.asarray(j, np.int64)
        assert np.all(i < j) and (i.size == 0 or j.max() < m)
        key = i * m + j
        assert np.unique(key).size == key.size, name
        self.name, self.m = name, int(m)
        self.i, self.j = i, j
        self.mval, self.cval = np.asarray(mval, np.float64), np.asarray(cval, np.float64)

    def upper(self):
        """(M, C) strictly upper triangular, scipy CSR (explicit M entries only where M != 0, C entries where C != 0)"""
        m = self.m
        km, kc = self.mval != 0, self.cval != 0
        M = sp.csr_matrix((self.mval[km], (self.i[km], self.j[km])), shape=(m, m))
        C = sp.csr_matrix((self.cval[kc], (self.i[kc], self.j[kc])), shape=(m, m))
        return M, C

    def dense_upper(self):
        M = np.zeros((self.m, self.m), order="F"); C = np.zeros((self.m, self.m), order="F")
        M[self.i, self.j] = self.mval; C[self.i, self.j] = self.cval
        return M, C

    def stored(self, f32):
        """(Mhat, Chat): the symmetric off-diagonal parts of the matrix the library stores, CSR fp64.  fp32 storage keeps
        |float32(M)|; an entry is kept when its stored affinity or its constraint bit is non-zero."""
        a = np.abs(self.mval.astype(np.float32).astype(np.float64)) if f32 else np.abs(self.mval)
        keep = (a != 0) | (self.cval != 0)
        i, j, a, c = self.i[keep], self.j[keep], a[keep], (self.cval[keep] != 0).astype(np.float64)
        m = self.m
        M = sp.csr_matrix((np.concatenate([a, a]), (np.concatenate([i, j]), np.concatenate([j, i]))), shape=(m, m))
        C = sp.csr_matrix((np.concatenate([c, c]), (np.concatenate([i, j]), np.concatenate([j, i]))), shape=(m, m))
        M.eliminate_zeros(); C.eliminate_zeros()
        return M, C, kept_pattern(m, i, j)

    def with_entry(self, name, i, j, mval, cval):
        return Case(name, self.m, np.append(self.i, i), np.append(self.j, j), np.append(self.mval, mval), np.append(self.cval, cval))

    def with_c0(self, name, k):
        """pair k keeps its affinity but loses its constraint bit: an (M > 0, C = 0) entry"""
        c = self.cval.copy(); c[k] = 0.0
        return Case(name, self.m, self.i, self.j, self.mval, c)

    def free_pair(self):
        """the first pair (0, j) the case does not use"""
        used = set(self.j[self.i == 0].tolist())
        j = next(j for j in range(1, self.m) if j not in used)
        return 0, j


def kept_pattern(m, i, j):
    """boolean CSR of the stored off-diagonal pattern (both triangles)"""
    r, c = np.concatenate([i, j]), np.concatenate([j, i])
    K = sp.csr_matrix((np.ones(r.size, bool), (r, c)), shape=(m, m))
    K.sort_indices()
    return K


def f32_field(x):
    """fp32 exponent field of float64 values (after rounding to fp32)"""
    return (np.asarray(x, np.float64).astype(np.float32).view(np.uint32) >> 23) & 0xFF


def f32_from(field, mant):
    return (np.asarray((np.asarray(field, np.uint32) << 23) | np.asarray(mant, np.uint32), np.uint32)
            .view(np.float32).astype(np.float64))


# ---- rule 1: the packed gate (pack_window in clp_sparse.cuh, with the plain test of the counting pass) -------------
def pack_gate(case):
    """(packed, bias) for fp32 storage of the case: plain (every kept entry has M > 0 and C = 1) and every kept exponent
    field at least b + 1, b = max(E_max - 15, 0); a matrix without kept entries is packed (all fillers)"""
    a = np.abs(case.mval.astype(np.float32))
    keep = (a != 0) | (case.cval != 0)
    if not keep.any():
        return True, 0
    plain = bool(np.all((a[keep] > 0) & (case.cval[keep] != 0)))
    E = f32_field(a[keep])
    b = max(int(E.max()) - 15, 0)
    return plain and bool(E.min() >= b + 1), b


# ---- rule 2: one packed row ------------------------------------------------------------------------------------------
def pack_row(cols, vals, m, bias):
    """words of one packed row: a filler (code 0) at the first column of every empty 16-column window, then per entry
    [31:27] delta - 1 | [26:23] exponent field - bias | [22:0] mantissa; the first delta counts from column -1"""
    cols = np.asarray(cols, np.int64)
    nwin = (m + WIN - 1) // WIN
    occ = np.zeros(nwin, bool); occ[cols // WIN] = True
    fill = np.flatnonzero(~occ) * WIN
    allc = np.concatenate([cols, fill])
    bits = np.concatenate([np.asarray(vals, np.float64).astype(np.float32).view(np.uint32), np.zeros(fill.size, np.uint32)])
    order = np.argsort(allc, kind="stable")
    allc, bits = allc[order], bits[order]
    delta = np.diff(np.concatenate([[-1], allc]))
    assert np.all((delta >= 1) & (delta <= 31)), "a delta does not fit 5 bits"
    code = np.where(bits != 0, (bits >> 23).astype(np.int64) - bias, 0)
    assert np.all((bits == 0) | ((code >= 1) & (code <= 15))), "an exponent outside the window"
    words = ((delta - 1).astype(np.uint32) << 27) | (code.astype(np.uint32) << 23) | (bits & 0x7FFFFF)
    return words, delta


def unpack_row(words, bias):
    """(columns, values) of the entries of a packed row (fillers dropped)"""
    words = np.asarray(words, np.uint32)
    field = (words >> 27).astype(np.int64)
    cols = np.cumsum(np.where(field == 31, 0, field + 1)) - 1
    code = (words >> 23) & 0xF
    real = code != 0
    bits = ((code.astype(np.uint32) + np.uint32(bias)) << 23) | (words & 0x7FFFFF)
    return cols[real], bits[real].view(np.float32).astype(np.float64)


# ---- the segmented layout (make_plan) and the bytes of one pass --------------------------------------------------------
def seg_plan(m):
    """(NSEG, W) of the column segmentation; depends on m only"""
    cols128 = (m + 127) // 128
    sgmax = next(c for c in (8, 4, 2, 1) if c <= max(1, cols128))
    nseg_min = -(-m // SEG_MAX)
    nseg = sgmax * max(1, -(-nseg_min // sgmax))
    W = max(128, -(-(-(-m // nseg)) // 128) * 128)
    nseg = max(sgmax, -(-(-(-m // W)) // sgmax) * sgmax)
    return nseg, W


def seg_bytes_per_pass(K, esize):
    """sparse_info()'s byte count of the segmented layout (mode 3): per column segment, slices sorted by length and
    padded four at a time, (esize + 2) bytes per stored entry, 20 bytes of descriptors per item and segment"""
    m = K.shape[0]
    nseg, W = seg_plan(m)
    rows_pad = -(-m // 32) * 32
    lens = np.diff(K.indptr)
    rows = np.repeat(np.arange(m, dtype=np.int64), lens)
    cnt = np.bincount(rows * nseg + K.indices // W, minlength=m * nseg).reshape(m, nseg)
    stored = 0
    for s in range(nseg):
        cls = np.zeros(rows_pad, np.int64)
        cls[:m] = (cnt[:, s] + 3) // 4
        stored += 16 * int(np.sort(cls)[::-1][0::4].sum())
    return (esize + 2) * stored + rows_pad // 4 * nseg * 20, stored


def predict_mode(requested, m, K, f32, packed):
    """the sweep mode finalize_matrix picks on one GPU.  Auto (4) takes the compact copy when it reads less than 0.8 x
    the upper triangle, whole rows when the trial vector fits shared memory (m <= 27648)"""
    if requested in (0, 2):
        return requested
    resident = m <= RES_MAX_M
    if requested == 3 or requested == 6:
        return 6 if (requested == 6 and resident) else 3
    esize = 4 if f32 else 8
    if resident:
        from fixtures import bytes_per_pass
        eb = 4 if packed else esize + 2
        stored = (bytes_per_pass(K, packed, esize) - (-(-m // 32) * 32) // 4 * 20) // eb
    else:
        eb = esize + 2
        stored = seg_bytes_per_pass(K, esize)[1]
    if stored * eb < 0.8 * 0.5 * esize * float(m) * float(m):
        return 6 if resident else 3
    return 2


# ---- the families -------------------------------------------------------------------------------------------------------
def _vals(rng, n):
    return rng.uniform(0.05, 1.0, n)


def f1_deltas(m, seed=11):
    """F1: rows of the first half connect only to chosen columns of the second half (h = first half, a multiple of 16):
    row 1 to columns 16w and 16w + 31 of every other window (a delta of exactly 31 after the fillers), row 2 to column
    16w + 15 of every window (a chain of delta-16 steps), row 3 to column m - 1 only, row 4 to the first column of the
    partial last window only, row 0 to column m - 3 only (so row m - 3 holds only column 0).  All other rows of the first
    half are empty, as is every second-half row nobody connects to."""
    assert m % WIN in (1, 15)
    rng = np.random.default_rng(seed)
    h = WIN * ((m // 2) // WIN)
    pairs = []
    w = h // WIN
    while WIN * w + 31 < m - WIN:
        pairs += [(1, WIN * w), (1, WIN * w + 31)]; w += 2
    w = h // WIN
    while WIN * w + 15 < m - 32:
        pairs.append((2, WIN * w + 15)); w += 1
    pairs += [(3, m - 1), (4, WIN * (m // WIN)), (0, m - 3)]
    pairs = sorted(set(pairs))
    i, j = np.array(pairs).T
    return Case("F1_deltas_m%d" % m, m, i, j, _vals(rng, i.size), np.ones(i.size))


def f1_full(m, seed=12):
    """F1: every row full (delta 1 throughout, the longest length class)"""
    rng = np.random.default_rng(seed)
    i, j = np.triu_indices(m, 1)
    return Case("F1_full_m%d" % m, m, i, j, _vals(rng, i.size), np.ones(i.size))


F2_MAX = {"1": 1.0, "2m": 2.0 - 2.0 ** -23, "2p20": 2.0 ** 20, "2m115": 2.0 ** -115}


def f2_window(top, m=300, seed=21):
    """F2: exact fp32 values whose largest is F2_MAX[top].  Every in-window binade appears; the lowest admitted binade
    (code 1) with mantissa 0 and with all mantissa bits set; the highest binade (code 15 when the bias is > 0) up to the
    largest value"""
    rng = np.random.default_rng(seed)
    X = F2_MAX[top]
    ehi = int(f32_field(X)); b = max(ehi - 15, 0); lo = b + 1
    xmant = int(np.array(X, np.float32).view(np.uint32)) & 0x7FFFFF
    iu, ju = np.triu_indices(m, 1)
    pick = np.flatnonzero(rng.random(iu.size) < 0.08)
    n = pick.size
    field = rng.integers(lo, ehi + 1, n)
    mant = rng.integers(0, 1 << 23, n)
    mant = np.where(field == ehi, np.minimum(mant, xmant), mant)     # nothing above the largest value
    field[0], mant[0] = ehi, xmant                                    # the largest value itself
    field[1:9], mant[1:9] = lo, 0                                     # lowest binade, minimal mantissa
    field[9:17], mant[9:17] = lo, 0x7FFFFF                            # lowest binade, all mantissa bits set
    field[17:25], mant[17:25] = ehi, rng.integers(0, xmant + 1, 8)    # highest binade
    return Case("F2_%s_in" % top, m, iu[pick], ju[pick], f32_from(field, mant), np.ones(n))


def f2_variants(top):
    """F2 in-window case and its fall-back variants: one value a binade below the window (when the window does not start
    at the smallest normal), one fp32 subnormal (2^-130), one (M > 0, C = 0) entry, one (M = 0, C = 1) entry"""
    base = f2_window(top)
    ehi = int(f32_field(F2_MAX[top])); b = max(ehi - 15, 0)
    i0, j0 = base.free_pair()
    out = [base]
    if b >= 1:
        out.append(base.with_entry("F2_%s_below" % top, i0, j0, float(f32_from(b, 0x2AAAAA)), 1.0))
    out.append(base.with_entry("F2_%s_subnormal" % top, i0, j0, 2.0 ** -130, 1.0))
    out.append(base.with_c0("F2_%s_mc0" % top, 30))
    out.append(base.with_entry("F2_%s_m0c1" % top, i0, j0, 0.0, 1.0))
    return out


def f3_imbalance(m, seed=31):
    """F3: about 1 % heavy rows (connected to every non-empty row), about 60 % empty rows, the rest about 10 entries"""
    rng = np.random.default_rng(seed)
    perm = rng.permutation(m)
    nh, ne = m // 100, (6 * m) // 10
    heavy, rest = perm[:nh], perm[nh + ne:]
    active = np.concatenate([heavy, rest])
    a = np.repeat(heavy, active.size); b = np.tile(active, heavy.size)
    ra = np.repeat(rest, 5); rb = rest[rng.integers(0, rest.size, ra.size)]
    a, b = np.concatenate([a, ra]), np.concatenate([b, rb])
    keep = a != b
    lo, hi = np.minimum(a[keep], b[keep]), np.maximum(a[keep], b[keep])
    key = np.unique(lo.astype(np.int64) * m + hi)
    i, j = key // m, key % m
    return Case("F3_m%d" % m, m, i, j, _vals(rng, i.size), np.ones(i.size)), heavy, perm[nh:nh + ne]


F4_M = (127, 128, 129, 2047, 2048, 2049, 4095, 4096, 4097, 8193)


def f4_edges(m, seed=41):
    """F4: random rows (about 60 entries each, 10 % for small m) plus entries on both sides of columns 127/128,
    2047/2048 and 4095/4096 (the tile, stripe and segment boundaries) and in the last column"""
    rng = np.random.default_rng(seed + m)
    per = min(60, max(1, m // 10))
    a = np.repeat(np.arange(m), per // 2 + 1); b = rng.integers(0, m, a.size)
    edge = [c for bnd in (128, 2048, 4096) for c in (bnd - 2, bnd - 1, bnd, bnd + 1) if c < m] + [m - 1]
    ea = np.array([r for c in edge for r in (0, 1, c // 2, c - 1, c - 2) if 0 <= r < c] +
                  [c for c in edge for r in (c + 1, m - 1) if c < r < m], np.int64)
    eb = np.array([c for c in edge for r in (0, 1, c // 2, c - 1, c - 2) if 0 <= r < c] +
                  [r for c in edge for r in (c + 1, m - 1) if c < r < m], np.int64)
    a, b = np.concatenate([a, ea]), np.concatenate([b, eb])
    keep = a != b
    lo, hi = np.minimum(a[keep], b[keep]), np.maximum(a[keep], b[keep])
    key = np.unique(lo.astype(np.int64) * m + hi)
    i, j = key // m, key % m
    return Case("F4_m%d" % m, m, i, j, _vals(rng, i.size), np.ones(i.size))


def f5_small(m, seed=51):
    """F5: tiny problems, about half of the pairs kept"""
    rng = np.random.default_rng(seed + m)
    iu, ju = np.triu_indices(m, 1)
    pick = rng.random(iu.size) < 0.5
    return Case("F5_m%d" % m, m, iu[pick], ju[pick], _vals(rng, int(pick.sum())), np.ones(int(pick.sum())))


def f5_empty(m=1000):
    """F5: no off-diagonal entry at all"""
    return Case("F5_empty_m%d" % m, m, [], [], [], [])


def pair_cases():
    """every pair-list case of the families F1, F2, F4, F5 (F3 is built on its own: it is large)"""
    out = [f1_deltas(641), f1_deltas(655), f1_full(161)]
    for top in F2_MAX:
        out += f2_variants(top)
    out += [f4_edges(m) for m in F4_M]
    out += [f5_small(m) for m in (1, 2, 3, 17)] + [f5_empty()]
    return out
