"""Batched maximum clique (clp_batch_max_clique_*, BatchCLIPPER.max_clique_many, maxclique_many) against the CPU
restatement in tests/clique_oracle.py and against single fp32 handles (clp_max_clique) holding the same graphs.
Run with  pytest -m gpu  on an H100.

  core numbers, n_edges, KCORE and HEU nodes: identical to the oracle and to the single path
  EXACT: a valid clique, sorted, no smaller than HEU; where the oracle proves omega, that size and proven = 1, and the
         nodes of the single path wherever both runs are proven
"""
import ctypes as C

import numpy as np
import pytest

import clique_families as cf
import clique_oracle as co
import fixtures as fx

pytestmark = pytest.mark.gpu

EXACT_LIMIT = 20.0  # seconds for a whole batch call, and per single-handle EXACT call (test_gpu_maxclique.py)
HARD_LIMIT = 5.0
ORACLE_BUDGET = 300_000
FAMILIES = cf.graph_families()

_cache = {}


def _oracle(fam):
    if fam["name"] not in _cache:
        A = cf.adjacency(fam)
        core = co.core_numbers_level(A)
        h = co.heu(A, core)
        K, proven = co.exact(A, budget=ORACLE_BUDGET, lb_clique=h)
        _cache[fam["name"]] = dict(A=A, core=core, heu=h, K=K, proven=proven)
    return _cache[fam["name"]]


@pytest.fixture(scope="module")
def clp(built):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import clipper_b200 as clipperpy
    return clipperpy


def _mc(clp, method, time_limit=EXACT_LIMIT):
    p = clp.MCParams()
    p.method, p.time_limit = method, time_limit
    return p


def _single(c, clp, method, time_limit=EXACT_LIMIT):
    c.solve_as_maximum_clique(_mc(clp, method, time_limit))
    s = c.get_solution()
    return s.nodes, s.mc_info


def _single_graph(clp, fam, method, time_limit=EXACT_LIMIT):
    c = clp.CLIPPER(clp.invariants.EuclideanDistance(clp.invariants.EuclideanDistanceParams()), clp.Params())
    c.set_matrix_data(fam["M"], fam["C"])
    return _single(c, clp, method, time_limit)


def _check_common(o, s, name):
    A = o["A"]
    assert s.core.tolist() == o["core"].tolist(), name
    mc = int(o["core"].max())
    i = s.mc_info
    assert i["max_core"] == mc and i["upper_bound"] == mc + 1 and i["n_edges"] == int(A.sum()) // 2, (name, i)
    assert s.score == -1 and s.ifinal == 0 and not s.u.any() and s.u.shape == (A.shape[0],)


def test_graph_families_kcore_heu(clp):
    graphs = [f["C"] for f in FAMILIES]
    kc = clp.maxclique_many(graphs, _mc(clp, clp.MCMethod.KCORE))
    heu = clp.maxclique_many(graphs, _mc(clp, clp.MCMethod.HEU))
    assert len(kc) == len(heu) == len(FAMILIES)
    for fam, sk, sh in zip(FAMILIES, kc, heu):
        o = _oracle(fam)
        _check_common(o, sk, fam["name"])
        _check_common(o, sh, fam["name"])
        assert sk.nodes == np.flatnonzero(o["core"] >= o["core"].max()).tolist(), fam["name"]
        assert sh.nodes == o["heu"] and sh.mc_info["lower_bound"] == len(o["heu"]), fam["name"]
        assert sh.mc_info["proven"] == int(len(o["heu"]) == o["core"].max() + 1)


def test_graph_families_exact(clp):
    # the time limits of test_gpu_maxclique.py: the families the oracle proves in one call under EXACT_LIMIT, the
    # others in one call under HARD_LIMIT.  In one call with the proven ones, the long tasks of G(500, 0.9) would hold
    # every search worker until the limit (the draw order interleaves the problems; a task runs to its end).
    easy = [f for f in FAMILIES if _oracle(f)["proven"]]
    hard = [f for f in FAMILIES if not _oracle(f)["proven"]]
    fams = easy + hard
    sols = (clp.maxclique_many([f["C"] for f in easy], _mc(clp, clp.MCMethod.EXACT, EXACT_LIMIT)) +
            clp.maxclique_many([f["C"] for f in hard], _mc(clp, clp.MCMethod.EXACT, HARD_LIMIT)))
    compared = 0
    for fam, s in zip(fams, sols):
        o = _oracle(fam)
        _check_common(o, s, fam["name"])
        i = s.mc_info
        assert co.is_clique(o["A"], s.nodes) and s.nodes == sorted(s.nodes) and i["n_nodes"] == len(s.nodes)
        assert len(s.nodes) >= len(o["heu"]) and i["lower_bound"] == len(o["heu"]), fam["name"]
        if o["proven"]:
            assert len(s.nodes) == len(o["K"]) and i["proven"] == 1 and i["timed_out"] == 0, (fam["name"], i)
            nodes1, info1 = _single_graph(clp, fam, clp.MCMethod.EXACT)
            assert info1["proven"] == 1
            assert s.nodes == nodes1, fam["name"]
            compared += 1
        else:
            assert i["proven"] == 1 or i["timed_out"] == 1, (fam["name"], i)
    assert compared >= 50


def test_time_limit_zero(clp):
    fams = [f for f in FAMILIES if f["C"].shape[0] <= 200]
    sols = clp.maxclique_many([f["C"] for f in fams], _mc(clp, clp.MCMethod.EXACT, 0))
    for fam, s in zip(fams, sols):
        o = _oracle(fam)
        i = s.mc_info
        assert s.nodes == o["heu"] and i["n_branches"] == 0 and i["timed_out"] == 0, fam["name"]
        assert i["proven"] == int(i["lower_bound"] == i["upper_bound"]), fam["name"]


def test_hard_problem_does_not_starve_small_ones(clp):
    hard = [f for f in FAMILIES if f["name"] == "gnp_n500_p0.9"][0]
    small = [f for f in FAMILIES if f["C"].shape[0] <= 65]
    fams = small[: len(small) // 2] + [hard] + small[len(small) // 2:]
    sols = clp.maxclique_many([f["C"] for f in fams], _mc(clp, clp.MCMethod.EXACT, 2.0))
    for fam, s in zip(fams, sols):
        o = _oracle(fam)
        i = s.mc_info
        assert co.is_clique(o["A"], s.nodes) and len(s.nodes) >= len(o["heu"]), fam["name"]
        if fam is hard:
            print("gnp_n500_p0.9 in a 2 s batch:", i)
            assert i["proven"] == 1 or i["timed_out"] == 1
        else:
            assert o["proven"], fam["name"]
            assert len(s.nodes) == len(o["K"]) and i["proven"] == 1 and i["timed_out"] == 0, (fam["name"], i)


def test_reproducible_and_order_free(clp):
    fams = [f for f in FAMILIES if f["C"].shape[0] <= 200 and f["name"] != "gnp_n200_p0.9"]
    p = _mc(clp, clp.MCMethod.EXACT, EXACT_LIMIT)
    first = clp.maxclique_many([f["C"] for f in fams], p)
    again = clp.maxclique_many([f["C"] for f in fams], p)
    perm = np.random.default_rng(3).permutation(len(fams))
    shuffled = clp.maxclique_many([fams[k]["C"] for k in perm], p)
    back = [None] * len(fams)
    for j, k in enumerate(perm):
        back[k] = shuffled[j]
    nproven = 0
    for fam, a, b, c in zip(fams, first, again, back):
        if a.mc_info["proven"] and b.mc_info["proven"] and c.mc_info["proven"]:
            assert a.nodes == b.nodes == c.nodes, fam["name"]
            nproven += 1
    assert nproven >= len(fams) - 2


# ---- scored problems against single handles scored on the same inputs ---------------------------------------------
def _euclid(clp, sigma, epsilon):
    ip = clp.invariants.EuclideanDistanceParams()
    ip.sigma, ip.epsilon = sigma, epsilon
    return clp.invariants.EuclideanDistance(ip)


def _compact(prob, m):
    """the first m associations of a datagen problem, with only the points they touch"""
    A = prob["A"][:m]
    used1, inv1 = np.unique(A[:, 0], return_inverse=True)
    used2, inv2 = np.unique(A[:, 1], return_inverse=True)
    return dict(D1=np.asfortranarray(prob["D1"][:, used1]), D2=np.asfortranarray(prob["D2"][:, used2]),
                A=np.asfortranarray(np.stack([inv1, inv2], axis=1).astype(np.int32)))


def _compare_scored(clp, make_single, batch, probs, exact_limit):
    methods = (clp.MCMethod.KCORE, clp.MCMethod.HEU, clp.MCMethod.EXACT)
    got = {mth: batch.max_clique_many(probs, _mc(clp, mth, exact_limit)) for mth in methods}
    both_proven = 0
    for k, p in enumerate(probs):
        c = make_single()
        c.score_pairwise_consistency(p["D1"], p["D2"], p.get("A"))
        core = c.core_numbers()
        for mth in methods:
            s = got[mth][k]
            nodes1, info1 = _single(c, clp, mth, exact_limit)
            assert s.core.tolist() == core.tolist(), (k, mth)
            for key in ("n_edges", "max_core", "upper_bound", "lower_bound"):
                assert s.mc_info[key] == info1[key], (k, mth, key, s.mc_info, info1)
            if mth != clp.MCMethod.EXACT:
                assert s.nodes == nodes1, (k, mth)
            else:
                assert len(s.nodes) >= s.mc_info["lower_bound"] and s.nodes == sorted(s.nodes)
                if s.mc_info["proven"] and info1["proven"]:
                    assert s.nodes == nodes1, k
                    both_proven += 1
    return both_proven


def test_scored_euclidean_against_single(clp):
    from clipper_b200 import datagen
    sigma, eps = 0.015, 0.05
    base = datagen.euclidean_problem(2048, 0.9, 4242)
    probs = [_compact(base, m) for m in (1, 2, 4)]
    model, data = fx.toy_problem()
    probs.append(dict(D1=model, D2=data, A=None))  # the toy, all-to-all: m = 12
    for k, m in enumerate((64, 65, 333, 1000, 2048)):
        probs.append(_compact(datagen.euclidean_problem(m, 0.9, 4300 + k), m))
    b = clp.BatchCLIPPER(_euclid(clp, sigma, eps), clp.Params())
    n = _compare_scored(clp, lambda: clp.CLIPPER(_euclid(clp, sigma, eps), clp.Params()), b, probs, EXACT_LIMIT)
    print("euclidean: %d of %d EXACT answers proven on both paths" % (n, len(probs)))
    assert n >= 4  # at least m = 1, 2, 4 and the toy


def test_scored_c2_parameters_m4096(clp):
    from clipper_b200 import datagen
    prob = datagen.config_problem("c2", m=4096)
    cfg = prob["cfg"]
    probs = [_compact(prob, 4096)]
    b = clp.BatchCLIPPER(_euclid(clp, cfg["sigma"], cfg["epsilon"]), clp.Params())
    n = _compare_scored(clp, lambda: clp.CLIPPER(_euclid(clp, cfg["sigma"], cfg["epsilon"]), clp.Params()), b, probs,
                        HARD_LIMIT)
    print("c2 parameters at m = 4096: EXACT proven on both paths:", n)


def test_scored_pointnormal_against_single(clp):
    from clipper_b200 import datagen
    probs, cfg = [], None
    for m in (200, 2000):
        prob = datagen.config_problem("c3", m=m)
        cfg = prob["cfg"]
        probs.append(dict(D1=prob["D1"], D2=prob["D2"], A=prob["A"]))

    def inv():
        ip = clp.invariants.PointNormalDistanceParams()
        ip.sigp, ip.epsp, ip.sign, ip.epsn = cfg["sigp"], cfg["epsp"], cfg["sign"], cfg["epsn"]
        return clp.invariants.PointNormalDistance(ip)

    b = clp.BatchCLIPPER(inv(), clp.Params())
    n = _compare_scored(clp, lambda: clp.CLIPPER(inv(), clp.Params()), b, probs, EXACT_LIMIT)
    print("pointnormal: EXACT proven on both paths:", n)


# ---- errors ---------------------------------------------------------------------------------------------------------
def _graphs_call(clp, colptrs, rowidxs, ms, method=0):
    from clipper_b200 import _capi
    L = _capi.load()
    b = C.c_void_p()
    assert L.clp_batch_create(0, C.byref(b)) == 0
    try:
        n = len(ms)
        vp = C.c_void_p
        cpp, rip = (vp * n)(), (vp * n)()
        keep = []
        for k in range(n):
            cp = np.ascontiguousarray(colptrs[k], np.int64); ri = np.ascontiguousarray(rowidxs[k], np.int32)
            keep += [cp, ri]
            cpp[k], rip[k] = cp.ctypes.data, ri.ctypes.data
        infos = (_capi.ClpMcInfo * n)()
        nodes = [np.zeros(max(m, 1), np.int32) for m in ms]
        nodep = (vp * n)(*[x.ctypes.data for x in nodes])
        rc = L.clp_batch_max_clique_graphs(b, n, (C.c_int64 * n)(*ms), cpp, rip, method, 1.0, infos, nodep, None)
        return rc, L.clp_batch_last_error(b), infos, nodes
    finally:
        L.clp_batch_destroy(b)


def test_errors(clp):
    with pytest.raises(clp.ClipperError) as e:
        clp.maxclique_many([np.zeros((3, 3)), np.zeros((4097, 4097), np.float32)], _mc(clp, clp.MCMethod.HEU))
    assert e.value.code == 1
    with pytest.raises(clp.ClipperError) as e:
        clp.maxclique_many([np.ones((3, 3))], _mc(clp, 7))
    assert e.value.code == 1
    # the smallest valid call works through the C-ABI: a triangle
    rc, _, infos, nodes = _graphs_call(clp, [[0, 0, 1, 3]], [[0, 0, 1]], [3])
    assert rc == 0 and infos[0].n_nodes == 3 and nodes[0].tolist() == [0, 1, 2]
    for cp, ri in (([0, 0, 1, 2], [0, 2]),      # row == column
                   ([0, 0, 1, 2], [0, 3]),      # row > column (and out of range)
                   ([0, 0, 1, 2], [0, -1]),     # negative row
                   ([0, 1, 1, 1], [0])):        # an entry in column 0
        rc, msg, _, _ = _graphs_call(clp, [cp], [ri], [3])
        assert rc == 1 and b"strictly upper" in msg, (cp, ri, msg)
    rc, msg, _, _ = _graphs_call(clp, [[0, 0, 1, 3]], [[0, 0, 1]], [3], method=5)
    assert rc == 1
    # association indices out of range of D1 / D2
    from clipper_b200 import datagen
    p = _compact(datagen.euclidean_problem(100, 0.9, 11), 100)
    bad = dict(p)
    bad["A"] = p["A"].copy(order="F")
    bad["A"][7, 0] = p["D1"].shape[1]
    b = clp.BatchCLIPPER(_euclid(clp, 0.015, 0.05), clp.Params())
    with pytest.raises(clp.ClipperError) as e:
        b.max_clique_many([p, bad], _mc(clp, clp.MCMethod.HEU))
    assert e.value.code == 1
    bad["A"][7, 0] = -1
    with pytest.raises(clp.ClipperError) as e:
        b.max_clique_many([bad], _mc(clp, clp.MCMethod.EXACT))
    assert e.value.code == 1
    assert b.max_clique_many([p], _mc(clp, clp.MCMethod.HEU))[0].nodes  # the handle still works


def test_single_vertex_and_edgeless(clp):
    sols = clp.maxclique_many([np.zeros((1, 1)), np.zeros((5, 5))], _mc(clp, clp.MCMethod.KCORE))
    assert sols[0].nodes == [0] and sols[1].nodes == [0, 1, 2, 3, 4]
    for mth in (clp.MCMethod.HEU, clp.MCMethod.EXACT):
        sols = clp.maxclique_many([np.zeros((1, 1)), np.zeros((5, 5))], _mc(clp, mth))
        assert sols[0].nodes == [0] and sols[1].nodes == [0] and all(s.mc_info["proven"] == 1 for s in sols)
