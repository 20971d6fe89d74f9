"""SCC decomposition and fair-cycle search on the device (include/tlag.h: tlag_scc, tlag_fair_cycles).

The device results are compared with a numpy/scipy restatement: SCCs from
`scipy.sparse.csgraph.connected_components(connection="strong")`, Emerson-Lei written out over them.  Without a GPU, that
restatement is itself checked against a brute force on tiny graphs: a state lies on a fair cycle iff some strongly
connected set of states holding it satisfies every fairness condition and holds a state with each required bit clear.
"""
import itertools

import numpy as np
import pytest
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import breadth_first_order, connected_components

NO = 0xFFFFFFFF


# ---------------------------------------------------------------- host restatement
def _kept(n, src, dst, vmask, emask):
    keep = src != dst
    if emask is not None:
        keep &= emask.astype(bool)
    if vmask is not None:
        keep &= vmask[src] & vmask[dst]
    return src[keep], dst[keep], keep


def ref_scc(n, src, dst, vmask=None, emask=None):
    """component label per state (-1 outside the mask)"""
    vm = np.ones(n, bool) if vmask is None else vmask.astype(bool)
    s, d, _ = _kept(n, src, dst, vm, emask)
    a = csr_matrix((np.ones(s.size, np.int8), (s, d)), shape=(n, n))
    _, lab = connected_components(a, directed=True, connection="strong")
    lab = lab.astype(np.int64)
    lab[~vm] = -1
    return lab


def canon(lab, none):
    """relabel each component by its smallest state; states labelled `none` -> -1"""
    lab = np.asarray(lab).astype(np.int64)
    out = np.full(lab.size, -1, np.int64)
    inside = lab != none
    idx = np.nonzero(inside)[0]
    if idx.size:
        _, first, inv = np.unique(lab[idx], return_index=True, return_inverse=True)
        out[idx] = idx[first][inv]      # idx ascends: a label's first occurrence is its smallest state
    return out


def _bits(fairness):
    return [(1 << en, 1 << act) for k, en, act in fairness if k == "WF"], \
           [(1 << en, 1 << act) for k, en, act in fairness if k == "SF"]


def ref_fair(n, src, dst, elab=None, slab=None, vmask=None, emask=None, fairness=(), need_clear=0, seeds=None):
    """-> (accepted SCC label per state, -1 elsewhere; witness or None)"""
    vm = np.ones(n, bool) if vmask is None else vmask.astype(bool)
    slab = np.zeros(n, np.uint32) if slab is None else np.asarray(slab, np.uint32)
    elab = np.zeros(src.size, np.uint32) if elab is None else np.asarray(elab, np.uint32)
    wf, sf = _bits(fairness)
    alive = vm.copy()
    while True:
        lab = ref_scc(n, src, dst, alive, emask)
        ids = np.where(alive, lab, 0)
        s_or = np.zeros(n, np.uint32)
        s_and = np.full(n, 0xFFFFFFFF, np.uint32)
        np.bitwise_or.at(s_or, ids[alive], slab[alive])
        np.bitwise_and.at(s_and, ids[alive], slab[alive])
        _, _, keep = _kept(n, src, dst, alive, emask)
        inner = keep & (lab[src] == lab[dst])
        e_or = np.zeros(n, np.uint32)
        np.bitwise_or.at(e_or, lab[src[inner]], elab[inner])
        so, sa, eo = s_or[ids], s_and[ids], e_or[ids]
        drop = (sa & need_clear) != 0
        for en, act in wf:
            drop |= ((sa & en) != 0) & ((eo & act) == 0)
        sf_drop = np.zeros(n, bool)
        for en, act in sf:
            sf_drop |= ((so & en) != 0) & ((eo & act) == 0) & ((slab & en) != 0)
        drop &= alive
        sf_drop &= alive
        alive &= ~(drop | sf_drop)
        if not (sf_drop & ~drop).any():
            break
    acc = np.where(alive, lab, -1)
    cand = alive.copy()
    if seeds is not None:
        s, d, _ = _kept(n, src, dst, vm, emask)
        sd = np.nonzero(np.asarray(seeds).astype(bool) & vm)[0]
        # one extra vertex n with an edge to every seed: what it reaches is what the seeds reach
        a = csr_matrix((np.ones(s.size + sd.size, np.int8), (np.r_[s, np.full(sd.size, n)], np.r_[d, sd])),
                       shape=(n + 1, n + 1))
        reach = np.zeros(n + 1, bool)
        reach[breadth_first_order(a, n, directed=True, return_predecessors=False)] = True
        cand &= reach[:n]
    w = np.nonzero(cand)[0]
    return acc, (int(w[0]) if w.size else None)


def brute_fair(n, src, dst, elab, slab, vmask, emask, fairness, need_clear, seeds):
    """states on a fair, accepting cycle, from every strongly connected set of states (tiny graphs only)"""
    wf, sf = _bits(fairness)
    s, d, keep = _kept(n, src, dst, vmask.astype(bool), emask)
    el = np.asarray(elab, np.uint32)[keep]
    on = np.zeros(n, bool)
    for r in range(1, n + 1):
        for sub in itertools.combinations([v for v in range(n) if vmask[v]], r):
            S = set(sub)
            inside = np.array([a in S and b in S for a, b in zip(s.tolist(), d.tolist())], bool)
            if r > 1:
                sub_lab = ref_scc(n, s[inside], d[inside], np.isin(np.arange(n), sub))
                if len(set(sub_lab[list(sub)].tolist())) != 1:
                    continue
            so = np.bitwise_or.reduce(slab[list(sub)])
            sa = np.bitwise_and.reduce(slab[list(sub)])
            eo = int(np.bitwise_or.reduce(el[inside])) if inside.any() else 0
            ok = (sa & need_clear) == 0
            ok &= all(not ((sa & en) and not (eo & act)) for en, act in wf)
            ok &= all(not ((so & en) and not (eo & act)) for en, act in sf)
            if ok:
                on[list(sub)] = True
    witness = None
    if seeds is not None:
        a = csr_matrix((np.ones(s.size, np.int8), (s, d)), shape=(n, n))
        reach = np.zeros(n, bool)
        for v in np.nonzero(np.asarray(seeds).astype(bool) & vmask.astype(bool))[0]:
            reach[breadth_first_order(a, v, directed=True, return_predecessors=False)] = True
        w = np.nonzero(on & reach)[0]
    else:
        w = np.nonzero(on)[0]
    if w.size:
        witness = int(w[0])
    return on, witness


def random_case(rng, n, m, n_bits=3):
    src = rng.integers(0, n, m).astype(np.uint32)
    dst = rng.integers(0, n, m).astype(np.uint32)
    elab = rng.integers(0, 1 << n_bits, m).astype(np.uint32)
    slab = rng.integers(0, 1 << n_bits, n).astype(np.uint32)
    vmask = (rng.random(n) < 0.85).astype(np.uint8)
    emask = (rng.random(m) < 0.85).astype(np.uint8)
    fairness = [(("WF", "SF")[int(rng.integers(2))], int(rng.integers(n_bits)), int(rng.integers(n_bits)))
                for _ in range(int(rng.integers(0, 3)))]
    need = int(rng.integers(0, 1 << n_bits)) if rng.random() < 0.5 else 0
    seeds = (rng.random(n) < 0.3).astype(np.uint8) if rng.random() < 0.5 else None
    return dict(src=src, dst=dst, elab=elab, slab=slab, vmask=vmask, emask=emask, fairness=fairness, need_clear=need,
                seeds=seeds)


# ---------------------------------------------------------------- CPU: the restatement against the brute force
def test_reference_matches_brute_force():
    rng = np.random.default_rng(7)
    for _ in range(150):
        n = int(rng.integers(1, 8))
        c = random_case(rng, n, int(rng.integers(0, 3 * n + 1)))
        acc, w = ref_fair(n, c["src"], c["dst"], c["elab"], c["slab"], c["vmask"], c["emask"], c["fairness"],
                          c["need_clear"], c["seeds"])
        on, bw = brute_fair(n, c["src"], c["dst"], c["elab"], c["slab"], c["vmask"], c["emask"], c["fairness"],
                            c["need_clear"], c["seeds"])
        assert np.array_equal(acc >= 0, on), c
        assert w == bw, c


def test_reference_small_cases():
    # 0 -> 1 -> 2 -> 0, 2 -> 3; edge 1->2 carries action bit 0; states 0, 1 have ENABLED bit 0
    src = np.array([0, 1, 2, 2], np.uint32)
    dst = np.array([1, 2, 0, 3], np.uint32)
    elab = np.array([0, 1, 0, 0], np.uint32)
    slab = np.array([1, 1, 0, 0], np.uint32)
    assert canon(ref_scc(4, src, dst), -1).tolist() == [0, 0, 0, 3]
    # WF holds on the cycle (it takes the action) and on {3} (stutters with the action disabled)
    acc, w = ref_fair(4, src, dst, elab, slab, fairness=[("WF", 0, 0)])
    assert (acc >= 0).tolist() == [True, True, True, True] and w == 0
    # without the action edge, the cycle is still WF-fair (state 2 disables it), not SF-fair: SF drops 0 and 1
    acc, _ = ref_fair(4, src, dst, np.zeros(4, np.uint32), slab, fairness=[("SF", 0, 0)])
    assert (acc >= 0).tolist() == [False, False, True, True]
    # <>[]Y with Y = bit 1 everywhere but state 3: only {3} holds a ~Y state
    acc, w = ref_fair(4, src, dst, slab=np.array([2, 2, 2, 0], np.uint32), need_clear=2)
    assert (acc >= 0).tolist() == [False, False, False, True] and w == 3


# ---------------------------------------------------------------- GPU
def _graphs():
    rng = np.random.default_rng(11)
    n = 50_000
    yield "singletons", n, *_dag(rng, n, 4 * n)
    yield "no_edges", n, np.zeros(0, np.uint32), np.zeros(0, np.uint32)
    ring = np.arange(n, dtype=np.uint32)
    yield "giant", n, np.r_[ring, rng.integers(0, n, 2 * n).astype(np.uint32)], \
        np.r_[(ring + 1) % n, rng.integers(0, n, 2 * n).astype(np.uint32)]
    # paths, one numbered forwards, one backwards, one shuffled
    L = 100_000
    perm = rng.permutation(L).astype(np.uint32)
    yield "chains", 3 * L, np.r_[np.arange(L - 1), 2 * L - 1 - np.arange(L - 1), 2 * L + perm[:-1]].astype(np.uint32), \
        np.r_[np.arange(1, L), 2 * L - 2 - np.arange(L - 1), 2 * L + perm[1:]].astype(np.uint32)
    # many small cycles of lengths 1..8, chained into a DAG of cycles, vertices shuffled
    lens = rng.integers(1, 9, 20_000)
    n2 = int(lens.sum())
    starts = np.r_[0, np.cumsum(lens)[:-1]]
    cyc_src = np.arange(n2)
    cyc_dst = np.arange(n2) + 1
    cyc_dst[np.cumsum(lens) - 1] = starts
    link_a = rng.integers(0, lens.size - 1, lens.size)
    link_b = link_a + 1 + rng.integers(0, 3, lens.size)
    link_b = np.minimum(link_b, lens.size - 1)
    p = rng.permutation(n2)
    s = p[np.r_[cyc_src, starts[link_a]]]
    d = p[np.r_[cyc_dst, starts[link_b]]]
    yield "small_cycles", n2, s.astype(np.uint32), d.astype(np.uint32)
    # random graph with about 2 out-edges per state: one giant SCC and a fringe
    yield "random", n, rng.integers(0, n, 2 * n).astype(np.uint32), rng.integers(0, n, 2 * n).astype(np.uint32)


def _dag(rng, n, m):
    a = rng.integers(0, n, m)
    b = rng.integers(0, n, m)
    return np.minimum(a, b).astype(np.uint32), np.maximum(a, b).astype(np.uint32)


GRAPHS = {name: (n, s, d) for name, n, s, d in _graphs()}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GRAPHS))
@pytest.mark.parametrize("masked", [False, True])
def test_scc_matches_scipy(name, masked):
    from tla_rust_b200 import engine
    n, s, d = GRAPHS[name]
    rng = np.random.default_rng(3)
    vm = (rng.random(n) < 0.9).astype(np.uint8) if masked else None
    em = (rng.random(s.size) < 0.9).astype(np.uint8) if masked else None
    got, k, ms = engine.scc(n, s, d, vm, em)
    want = canon(ref_scc(n, s, d, vm, em), -1)
    assert np.array_equal(canon(got, NO), want)
    assert k == len(set(want[want >= 0].tolist()))
    assert ms >= 0


@pytest.mark.gpu
def test_scc_ten_million_edges():
    from tla_rust_b200 import engine
    rng = np.random.default_rng(5)
    n, m = 4_000_000, 10_000_000
    s = rng.integers(0, n, m).astype(np.uint32)
    d = rng.integers(0, n, m).astype(np.uint32)
    vm = (rng.random(n) < 0.95).astype(np.uint8)
    got, k, _ = engine.scc(n, s, d, vm)
    want = canon(ref_scc(n, s, d, vm), -1)
    assert np.array_equal(canon(got, NO), want)
    assert k == np.count_nonzero(want == np.arange(n))


@pytest.mark.gpu
def test_fair_cycles_match_reference():
    from tla_rust_b200 import engine
    rng = np.random.default_rng(13)
    for i in range(60):
        n = int(rng.integers(1, 9)) if i < 30 else int(rng.integers(100, 3000))
        c = random_case(rng, n, int(rng.integers(0, 3 * n + 1)), n_bits=3 if i < 30 else 5)
        r = engine.fair_cycles(n, c["src"], c["dst"], c["elab"], c["slab"], c["vmask"], c["emask"], c["fairness"],
                               c["need_clear"], c["seeds"])
        acc, w = ref_fair(n, c["src"], c["dst"], c["elab"], c["slab"], c["vmask"], c["emask"], c["fairness"],
                          c["need_clear"], c["seeds"])
        assert np.array_equal(canon(r["scc"], NO), canon(acc, -1)), (i, c)
        assert r["witness"] == w and r["violated"] == (w is not None), (i, c)
        assert r["fair_sccs"] == len(set(acc[acc >= 0].tolist()))


@pytest.mark.gpu
def test_endpoint_out_of_range_is_einval():
    """the C entry points check endpoints themselves (the Python wrapper's own check is bypassed here)"""
    import ctypes as C
    from tla_rust_b200 import engine
    L = engine._graph_lib()
    for n, bad in ((4, 4), (4, 0xFFFFFFFF), (0, 0)):
        src = np.array([0, 1, bad] if n else [bad], np.uint32)
        dst = np.array([1, 2, 0] if n else [bad], np.uint32)
        g = engine.TlagGraph(n, src.size, src.ctypes.data, dst.ctypes.data, None, None, None, None, 0)
        out = np.empty(max(n, 1), np.uint32)
        k, ms = C.c_uint64(), C.c_float()
        assert L.tlag_scc(C.byref(g), out.ctypes.data_as(C.c_void_p), C.byref(k), C.byref(ms)) == -1
        assert b">= n_states" in L.tlag_graph_last_error()
        q, r = engine.TlagFairQuery(None, 0, 0, None), engine.TlagFairResult()
        assert L.tlag_fair_cycles(C.byref(g), C.byref(q), None, C.byref(r)) == -1
    # the library still works after a refused call
    ids, k, _ = engine.scc(3, np.array([0, 1, 2], np.uint32), np.array([1, 2, 0], np.uint32))
    assert k == 1 and len(set(ids.tolist())) == 1


@pytest.mark.gpu
def test_fair_cycles_sf_refinement():
    """an SCC that fails SF loses its ENABLED states and is split again (Emerson-Lei needs a second round)"""
    from tla_rust_b200 import engine
    # 0 <-> 1 <-> 2 <-> 0 with state 1 ENABLED and no action edge: {0, 2} stays, 1 goes
    src = np.array([0, 1, 1, 2, 2, 0], np.uint32)
    dst = np.array([1, 0, 2, 1, 0, 2], np.uint32)
    slab = np.array([0, 1, 0], np.uint32)
    r = engine.fair_cycles(3, src, dst, state_label=slab, fairness=[("SF", 0, 0)])
    assert r["rounds"] == 2 and r["fair_sccs"] == 1 and r["witness"] == 0
    assert r["scc"][1] == NO and r["scc"][0] == r["scc"][2] != NO
    # WF: state 0 disables the action, so the whole cycle is fair
    r = engine.fair_cycles(3, src, dst, state_label=slab, fairness=[("WF", 0, 0)])
    assert r["rounds"] == 1 and r["fair_sccs"] == 1 and NO not in r["scc"].tolist()
    # seeds that reach no fair SCC: nothing violates
    r = engine.fair_cycles(3, src, dst, state_label=np.array([1, 1, 1], np.uint32), fairness=[("WF", 0, 0)],
                           seeds=np.array([1, 0, 0], np.uint8))
    assert not r["violated"] and r["witness"] is None and r["fair_sccs"] == 0
