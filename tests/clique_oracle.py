"""CPU restatement of the maximum-clique semantics of clp_max_clique (tests only).

The graph is given as a boolean adjacency (symmetric, zero diagonal) or as a list of Python-int bitsets.
  core_numbers_bz(adj)    Batagelj-Zaversnik bucket peeling (O(n + E) sequential)
  core_numbers_level(adj) level-synchronous peeling on a dense boolean matrix (numpy; fast for large n)
  heu(adj, core)          the deterministic greedy heuristic (seed v: K = {v}, P = N(v), repeatedly add the u in P of
                          highest core number, ties to the lowest index; the largest K, ties to the smallest seed)
  exact(adj, budget)      bitset branch-and-bound with a greedy colouring bound (MCQ / BBMC); returns (clique, proven)
"""
import numpy as np


def bitsets(adj):
    """rows of a boolean matrix as Python ints (bit j of row i = edge {i, j})"""
    A = np.asarray(adj, dtype=bool)
    n = A.shape[0]
    out = []
    packed = np.packbits(A, axis=1, bitorder="little")
    for i in range(n):
        out.append(int.from_bytes(packed[i].tobytes(), "little"))
    return out


def graph_from_constraint(C):
    """C (dense, any diagonal): edge {i, j}, i != j, iff C[i, j] != 0 -- the pattern of C without its diagonal"""
    A = np.asarray(C) != 0
    A = A.copy()
    np.fill_diagonal(A, False)
    return A


def core_numbers_bz(adj):
    A = np.asarray(adj, dtype=bool)
    n = A.shape[0]
    nbrs = [np.flatnonzero(A[i]).tolist() for i in range(n)]
    deg = [len(x) for x in nbrs]
    md = max(deg) if n else 0
    bins = [0] * (md + 1)
    for d in deg:
        bins[d] += 1
    start = 0
    for d in range(md + 1):
        bins[d], start = start, start + bins[d]
    pos = [0] * n
    vert = [0] * n
    for v in range(n):
        pos[v] = bins[deg[v]]
        vert[pos[v]] = v
        bins[deg[v]] += 1
    for d in range(md, 0, -1):
        bins[d] = bins[d - 1]
    if md >= 0 and n:
        bins[0] = 0
    for i in range(n):
        v = vert[i]
        for u in nbrs[v]:
            if deg[u] > deg[v]:
                du, pu = deg[u], pos[u]
                pw = bins[du]
                w = vert[pw]
                if u != w:
                    pos[u], vert[pu] = pw, w
                    pos[w], vert[pw] = pu, u
                bins[du] += 1
                deg[u] -= 1
    return np.array(deg, dtype=np.int64)


def core_numbers_level(adj):
    """same core numbers by level-synchronous peeling (every vertex of degree <= k leaves, k rises when none does)"""
    A = np.asarray(adj, dtype=bool)
    n = A.shape[0]
    deg = A.sum(1).astype(np.int64)
    alive = np.ones(n, dtype=bool)
    core = np.zeros(n, dtype=np.int64)
    k = 0
    while alive.any():
        f = alive & (deg <= k)
        if not f.any():
            k = int(deg[alive].min())
            continue
        core[f] = k
        alive &= ~f
        deg -= A[f].sum(0)
    return core


def heu(adj, core):
    """the greedy heuristic; returns the clique (ascending)"""
    A = np.asarray(adj, dtype=bool)
    n = A.shape[0]
    if n == 0:
        return []
    core = np.asarray(core)
    # relabel so that "highest core, lowest index" is the lowest label: the pick is then the lowest set bit
    perm = np.lexsort((np.arange(n), -core))  # perm[label] = vertex
    label = np.empty(n, dtype=np.int64)
    label[perm] = np.arange(n)
    B = bitsets(A[np.ix_(perm, perm)])
    best_size, best_seed, best_K = 0, n, None
    for v in sorted(range(n), key=lambda x: (-core[x], x)):
        if core[v] + 1 < best_size:
            continue
        K = [v]
        P = B[label[v]]
        while P:
            if len(K) + P.bit_count() < best_size or (len(K) + P.bit_count() == best_size and v > best_seed):
                K = None
                break
            low = (P & -P).bit_length() - 1
            K.append(int(perm[low]))
            P &= B[low]
        if K is None:
            continue
        if len(K) > best_size or (len(K) == best_size and v < best_seed):
            best_size, best_seed, best_K = len(K), v, K
    return sorted(best_K)


def heu_plain(adj, core):
    """literal restatement of the heuristic, every seed, no pruning (small graphs)"""
    A = np.asarray(adj, dtype=bool)
    n = A.shape[0]
    best = None
    for v in range(n):
        K = [v]
        P = set(np.flatnonzero(A[v]).tolist())
        while P:
            u = min(P, key=lambda x: (-core[x], x))
            K.append(u)
            P &= set(np.flatnonzero(A[u]).tolist())
        if best is None or len(K) > len(best):
            best = K
    return sorted(best) if best is not None else []


def exact(adj, budget=2_000_000, lb_clique=None):
    """maximum clique by MCQ-style branch-and-bound on Python-int bitsets.
    Returns (clique ascending, proven): proven is False when more than `budget` nodes were expanded."""
    A = np.asarray(adj, dtype=bool)
    n = A.shape[0]
    if n == 0:
        return [], True
    # initial order: degeneracy-like, high degree first helps the colouring bound
    order = np.argsort(-A.sum(1), kind="stable")
    B = bitsets(A[np.ix_(order, order)])
    best = [list(lb_clique) if lb_clique else [int(order[0])]]
    best_lab = [None]
    nodes = [0]

    def colour_sort(P):
        out = []  # (vertex label, colour) ascending colour
        U = P
        col = 0
        while U:
            col += 1
            Q = U
            while Q:
                low = Q & -Q
                v = low.bit_length() - 1
                U &= ~low
                Q &= ~low & ~B[v]
                out.append((v, col))
        return out

    class Budget(Exception):
        pass

    def expand(K, P):
        nodes[0] += 1
        if nodes[0] > budget:
            raise Budget()
        lst = colour_sort(P)
        for v, c in reversed(lst):
            if len(K) + c <= len(best[0]):
                return
            NP = P & B[v]
            K.append(v)
            if NP == 0:
                if len(K) > len(best[0]):
                    best[0] = [int(order[x]) for x in K]
            else:
                expand(K, NP)
            K.pop()
            P &= ~(1 << v)

    import sys
    old = sys.getrecursionlimit()
    sys.setrecursionlimit(max(old, 4 * n + 100))
    try:
        expand([], (1 << n) - 1)
        proven = True
    except Budget:
        proven = False
    finally:
        sys.setrecursionlimit(old)
    return sorted(best[0]), proven


def is_clique(adj, nodes):
    A = np.asarray(adj, dtype=bool)
    nodes = list(nodes)
    if len(set(nodes)) != len(nodes):
        return False
    sub = A[np.ix_(nodes, nodes)]
    return bool((sub | np.eye(len(nodes), dtype=bool)).all())


def brute_omega(adj):
    """clique number by enumeration (n <= 18)"""
    A = np.asarray(adj, dtype=bool)
    n = A.shape[0]
    nb = [sum(1 << j for j in np.flatnonzero(A[i])) for i in range(n)]
    best = 0
    for s in range(1 << n):
        c = s.bit_count()
        if c <= best:
            continue
        ok = True
        t = s
        while t:
            low = t & -t
            v = low.bit_length() - 1
            if (s & ~low) & ~nb[v]:
                ok = False
                break
            t &= ~low
        if ok:
            best = c
    return best
