"""The CPU restatement of the maximum-clique semantics (tests/clique_oracle.py) against brute force, networkx and a
literal restatement of the heuristic, and the graph families against what they claim to contain.  No GPU."""
import numpy as np
import pytest

import clique_families as cf
import clique_oracle as co


def _small_graphs():
    rng = np.random.default_rng(3)
    out = []
    for n in (1, 2, 5, 9, 13, 18):
        for p in (0.0, 0.3, 0.6, 0.9, 1.0):
            out.append(cf._sym(rng.random((n, n)) < p))
    out += [cf.moon_moser(3), cf.disjoint_cliques(3, 4), cf.star(10), cf.complete(7)]
    return out


def test_exact_equals_brute_force():
    for A in _small_graphs():
        K, proven = co.exact(A)
        assert proven and co.is_clique(A, K)
        assert len(K) == (co.brute_omega(A) if A.shape[0] else 0)


def test_core_numbers_two_ways():
    rng = np.random.default_rng(4)
    for n in (1, 2, 17, 64, 150):
        for p in (0.0, 0.05, 0.3, 0.8):
            A = cf._sym(rng.random((n, n)) < p)
            assert np.array_equal(co.core_numbers_bz(A), co.core_numbers_level(A))


def test_against_networkx():
    nx = pytest.importorskip("networkx")
    rng = np.random.default_rng(5)
    for n in (3, 20, 60, 120):
        for p in (0.1, 0.5, 0.8):
            A = cf._sym(rng.random((n, n)) < p)
            G = nx.from_numpy_array(A.astype(int))
            G.remove_edges_from(nx.selfloop_edges(G))
            core = nx.core_number(G)
            assert co.core_numbers_bz(A).tolist() == [core[i] for i in range(n)]
            _, w = nx.max_weight_clique(G, weight=None)
            K, proven = co.exact(A)
            assert proven and len(K) == w


def test_heuristic_equals_literal_statement():
    rng = np.random.default_rng(6)
    graphs = _small_graphs() + [cf._sym(rng.random((n, n)) < p) for n in (40, 90) for p in (0.2, 0.6, 0.9)]
    for A in graphs:
        if A.shape[0] == 0:
            continue
        core = co.core_numbers_bz(A)
        assert co.heu(A, core) == co.heu_plain(A, core)


def test_heuristic_ties():
    # edgeless: every seed gives a singleton, the smallest seed wins; star: the hub and the smallest leaf
    assert co.heu(np.zeros((6, 6), bool), np.zeros(6, int)) == [0]
    A = cf.star(9)
    assert co.heu(A, co.core_numbers_bz(A)) == [0, 1]
    A = cf.disjoint_cliques(3, 4)  # three equal cliques: the one of seed 0
    assert co.heu(A, co.core_numbers_bz(A)) == [0, 1, 2, 3]


def test_families_contain_what_they_claim():
    for fam in cf.graph_families():
        A = cf.adjacency(fam)
        assert np.array_equal(A, A.T) and not A.diagonal().any()
        claim = fam["claim"]
        if "clique" in claim:
            assert co.is_clique(A, claim["clique"]), fam["name"]
        if "omega" in claim:
            K, proven = co.exact(A, budget=200_000)
            assert proven and len(K) == claim["omega"], fam["name"]
        M, C = fam["M"], fam["C"]
        assert (np.triu(M, 1) >= 0).all() and set(np.unique(C).tolist()) <= {0.0, 1.0}
    names = [f["name"] for f in cf.graph_families()]
    assert len(names) == len(set(names))
    # the (M=0, C=1) edges and (M>0, C=0) non-edges are really there
    weird = [f for f in cf.graph_families() if f["name"].startswith("weird")][0]
    up = np.triu(np.ones_like(weird["C"], dtype=bool), 1)
    assert ((weird["M"] == 0) & (weird["C"] == 1) & up).any()
    assert ((weird["M"] > 0) & (weird["C"] == 0) & up).any()
    # cliques that straddle word boundaries
    s = [f for f in cf.graph_families() if f["name"] == "straddle_wide_130"][0]["claim"]["clique"]
    assert len({v // 32 for v in s}) == 3
