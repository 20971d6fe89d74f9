"""Liveness in `tlc` (DESIGN.md §7h): the front end's normal form, the label plan and image, and on the GPU the labels,
tlag_live_check and `tlc`'s reports on small specs written for it (tests/specs/Live*), every verdict against an
independent reference: ORACLE O1's state graph, labelled with the AST evaluator, and a numpy Emerson-Lei search."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import pytest
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import connected_components

from conftest import REF, ROOT

SPECS = os.path.join(ROOT, "tests", "specs")
LIVENESS = os.path.join(REF, "examples", "SpecifyingSystems", "Liveness")


def _model(name, cfg=None):
    from tla_rust_b200.front.spec import Model
    m = Model(os.path.join(SPECS, name + ".tla"), cfg_path=os.path.join(SPECS, cfg + ".cfg") if cfg else None)
    m.ev.out = io.StringIO()
    return m


# ---- the reference: O1's graph, labels from the AST evaluator, Emerson-Lei in numpy ---------------------------------
def o1_graph(m):
    from oracle.tlc_oracle import Oracle
    o = Oracle(m)
    states, index, edges = [], {}, set()
    for st in m.initial_states():
        if o.key(st) not in index:
            index[o.key(st)] = len(states)
            states.append(st)
    n_init = len(states)
    i = 0
    while i < len(states):
        for t, _act in o.successors(states[i]):
            if o.key(t) not in index:
                index[o.key(t)] = len(states)
                states.append(t)
            if index[o.key(t)] != i:
                edges.add((i, index[o.key(t)]))
        i += 1
    return states, sorted(edges), n_init


def ref_labels(m, plan, states, edges):
    from tla_rust_b200.front.eval import Fr
    ev = m.ev
    sl = np.zeros(len(states), dtype=np.uint32)
    el = np.zeros(len(edges), dtype=np.uint32)
    for i, st in enumerate(states):
        for j, p in enumerate(plan.state):
            if ev.eval(p.node, dict(p.env), Fr(p.ctx, st, None)) is True:
                sl[i] |= 1 << j
    for k, (s, t) in enumerate(edges):
        for j, p in enumerate(plan.edge):
            if ev.truth(p.node, dict(p.env), Fr(p.ctx, states[s], states[t])):
                el[k] |= 1 << j
    en, nen = plan.en_map()
    out = np.zeros(len(states), dtype=np.uint32)
    for k, (s, _t) in enumerate(edges):
        out[s] |= el[k]
    for a, b in en.items():
        sl |= ((out >> a) & 1).astype(np.uint32) << b
    for a, b in nen.items():
        sl |= (1 - ((out >> a) & 1)).astype(np.uint32) << b
    return sl, el


def ref_fair_sccs(n, edges, sl, el, fairness, keep_set, keep_clear, edge_drop, need_clear):
    """accepted SCC id per state (-1: none), Emerson-Lei as tlag_fair_cycles defines it"""
    alive = ((sl & keep_set) == keep_set) & ((sl & keep_clear) == 0)
    src = np.array([s for s, _ in edges], dtype=np.int64)
    dst = np.array([t for _, t in edges], dtype=np.int64)
    ekeep = (el & edge_drop) == 0 if len(edges) else np.zeros(0, bool)
    while True:
        keep = ekeep & alive[src] & alive[dst] if len(edges) else ekeep
        g = csr_matrix((np.ones(int(keep.sum())), (src[keep], dst[keep])), shape=(n, n))
        _, comp = connected_components(g, directed=True, connection="strong")
        comp = np.where(alive, comp, -1)
        resplit = False
        for c in set(comp[alive].tolist()):
            vs = comp == c
            s_or = np.bitwise_or.reduce(sl[vs]) if vs.any() else 0
            s_and = np.bitwise_and.reduce(sl[vs])
            inner = keep & (comp[src] == c) & (comp[dst] == c) if len(edges) else keep
            e_or = np.bitwise_or.reduce(el[inner]) if inner.any() else 0
            drop = bool(s_and & need_clear)
            sf_drop = np.zeros(n, bool)
            for kind, enb, act in fairness:
                en, a = 1 << enb, 1 << act
                if kind == "WF" and (s_and & en) and not (e_or & a):
                    drop = True
                if kind == "SF" and (s_or & en) and not (e_or & a):
                    sf_drop |= vs & ((sl & en) != 0)
            if drop:
                alive &= ~vs
            elif sf_drop.any():
                alive &= ~sf_drop
                resplit = True
        if not resplit:
            return np.where(alive, comp, -1), keep


def ref_check(n, edges, sl, el, args):
    """-> (witness or None, accepted SCCs) as tlag_live_check defines them"""
    if args["flags"] & 2:
        seeds = ((sl & args["seed_set"]) == args["seed_set"]) & ((sl & args["seed_clear"]) == 0)
        return (int(np.flatnonzero(seeds)[0]) if seeds.any() else None), 0
    comp, _ = ref_fair_sccs(n, edges, sl, el, args["fairness"], args["keep_set"], args["keep_clear"], args["edge_drop"],
                            args["need_clear"])
    hit = ref_reach(n, edges, sl, el, args, comp)
    return (int(np.flatnonzero(hit)[0]) if hit.any() else None), len(set(comp[comp >= 0].tolist()))


def ref_reach(n, edges, sl, el, args, comp):
    """states of accepted SCCs that count: all, or (seeds) those reachable from a seed in the restricted graph"""
    if not args["flags"] & 1:
        return comp >= 0
    # reachability over the whole restricted graph (states of SCCs dropped on the way included)
    vmask = ((sl & args["keep_set"]) == args["keep_set"]) & ((sl & args["keep_clear"]) == 0)
    ekeep = np.array([bool(vmask[s] and vmask[t] and not (el[k] & args["edge_drop"])) for k, (s, t) in enumerate(edges)],
                     dtype=bool)
    rows = np.arange(n) < (args["seed_rows"] or n)
    reach = rows & vmask & ((sl & args["seed_set"]) == args["seed_set"]) & ((sl & args["seed_clear"]) == 0)
    while True:
        nxt = reach.copy()
        for k, (s, t) in enumerate(edges):
            if reach[s] and ekeep[k]:
                nxt[t] = True
        if (nxt == reach).all():
            break
        reach = nxt
    return reach & (comp >= 0)


def test_emerson_lei_reference_against_brute_force():
    """On tiny graphs the numpy search accepts an SCC iff some cycle through all its states is fair (brute force over
    the conditions as TLA+ defines WF / SF on the cycle repeated for ever)."""
    rng = np.random.default_rng(3)
    for _ in range(200):
        n = int(rng.integers(1, 6))
        edges = sorted({(int(a), int(b)) for a, b in rng.integers(0, n, (int(rng.integers(0, 9)), 2)) if a != b})
        el = rng.integers(0, 2, len(edges)).astype(np.uint32)
        out = np.zeros(n, dtype=np.uint32)
        for k, (s, _t) in enumerate(edges):
            out[s] |= el[k]
        sl = out.copy()                  # bit 0: ENABLED <<A>> (some A-edge out of the state)
        for kind in ("WF", "SF"):
            comp, _ = ref_fair_sccs(n, edges, sl, el, [(kind, 0, 0)], 0, 0, 0, 0)
            # brute force: the SCCs of the whole graph; a fair cycle in C exists iff C (or a sub-SCC for SF) qualifies
            g = csr_matrix((np.ones(len(edges)), ([s for s, _ in edges], [t for _, t in edges])), shape=(n, n))
            _, c0 = connected_components(g, directed=True, connection="strong")
            want = set()
            for c in set(c0.tolist()):
                vs = np.flatnonzero(c0 == c)
                inner = [k for k, (s, t) in enumerate(edges) if c0[s] == c and c0[t] == c]
                took = any(el[k] for k in inner)
                if kind == "WF":
                    ok = took or not all(sl[v] & 1 for v in vs)
                    if ok:
                        want |= set(vs.tolist())
                else:
                    if took or not any(sl[v] & 1 for v in vs):
                        want |= set(vs.tolist())
                    else:                # fair cycles avoid the EN states: the non-EN sub-SCCs
                        sub = [v for v in vs if not sl[v] & 1]
                        want |= set(sub)
            got = set(np.flatnonzero(comp >= 0).tolist())
            if kind == "WF":
                assert got == want
            else:
                assert got <= want and (bool(got) == bool(want))


# ---- front end ---------------------------------------------------------------------------------------------------------
def test_normal_form_of_each_obligation():
    m = _model("LiveClock")
    assert [f.kind for f in m.fairness] == ["WF"]
    kinds = [(o.name, o.kind, [t[0] for t in o.terms]) for o in m.obligations]
    assert kinds == [("AlwaysTick", "inf", ["iea"])] + [("AllTimes", "inf", ["ie"])] * 3 + [("TypeOK", "always", [])]
    assert [o.terms[0][1].env for o in m.obligations[1:4]] == [{"n": 1}, {"n": 2}, {"n": 3}]
    assert [o.kind for o in _model("LiveLeads").obligations] == ["leadsto", "leadsto"]
    assert [o.kind for o in _model("LiveStrong").obligations] == ["eventually"]
    assert [f.kind for f in _model("LiveStrong", "LiveStrongSF").fairness] == ["WF", "SF"]
    assert not _model("LiveClock", "LiveClockNoFair").fairness


def test_unsupported_conjunct_keeps_its_warning(tmp_path):
    from tla_rust_b200.front.spec import Model
    (tmp_path / "T.tla").write_text("---- MODULE T ----\nVARIABLE x\nInit == x = 0\nNext == x' = x\n"
                                    "Spec == Init /\\ [][Next]_x\nP == [](x = 0 => ENABLED Next)\nQ == <>[]<>(x = 0)\n====\n")
    (tmp_path / "T.cfg").write_text("SPECIFICATION Spec\nPROPERTY P Q\n")
    m = Model(str(tmp_path / "T.tla"))
    assert not m.obligations
    assert len([w for w in m.warnings if "is not checked" in w]) == 2


def test_label_image_leaves_the_model_image_alone():
    from tla_rust_b200.checker import compile_model
    from tla_rust_b200.compile.lower import compile_labels
    from tla_rust_b200.liveness import LabelPlan
    m = _model("LiveStrong", "LiveStrongSF")
    cm = compile_model(m)
    code, cpool = np.array(cm.code).copy(), np.array(cm.cpool).copy()
    plan = LabelPlan(m)
    img = compile_labels(m, cm, plan.state, plan.edge)
    assert (np.array(cm.code) == code).all() and (np.array(cm.cpool) == cpool).all()
    assert img.n_states == len(plan.state) and img.n_edges == len(plan.edge) == 2
    assert set(img.entries) == {"states", "edges"}


# ---- the label image on the CPU reference (tests/label_ref.c) against the AST evaluator -------------------------------
_LIB = {}


def label_lib(tmp_dir):
    if "L" not in _LIB:
        so = os.path.join(tmp_dir, "label_ref.so")
        subprocess.check_call(["gcc", "-O1", "-std=gnu11", "-fPIC", "-shared", "-o", so,
                               os.path.join(ROOT, "tests", "label_ref.c")])
        _LIB["L"] = C.CDLL(so)
    return _LIB["L"]


def ref_run_labels(L, cm, img, entry, n_preds, s_words, t_words=None):
    code = np.ascontiguousarray(img.code, dtype=np.uint64)
    cpool = np.ascontiguousarray(img.cpool if len(img.cpool) else [0], dtype=np.int32)
    layout = np.ascontiguousarray(cm.layout, dtype=np.int32)
    s_words = np.ascontiguousarray(s_words, dtype=np.uint32)
    t_arr = None if t_words is None else np.ascontiguousarray(t_words, dtype=np.uint32)
    out = np.zeros(s_words.shape[0], dtype=np.uint32)
    rc = L.tlagcpu_labels(code.ctypes.data_as(C.c_void_p), cpool.ctypes.data_as(C.c_void_p), C.c_uint32(entry),
                          layout.ctypes.data_as(C.c_void_p), C.c_int(layout.shape[0]), C.c_uint32(img.frame_words + 8),
                          C.c_uint32(cm.state_words_unpacked), C.c_int(cm.W), s_words.ctypes.data_as(C.c_void_p),
                          None if t_arr is None else t_arr.ctypes.data_as(C.c_void_p), C.c_uint64(s_words.shape[0]),
                          C.c_uint32(n_preds), out.ctypes.data_as(C.c_void_p))
    assert rc == 0
    return out


def corpus(name):
    if not os.path.isdir(REF):
        pytest.skip("no tla-rust spec corpus (oracle/_ref/tla-rust)")
    from tla_rust_b200.front.spec import Model
    paths = {"LiveHourClock": os.path.join(LIVENESS, "LiveHourClock.tla"),
             "MCLiveInternalMemory": os.path.join(LIVENESS, "MCLiveInternalMemory.tla"),
             "HourClock": os.path.join(REF, "examples", "SpecifyingSystems", "HourClock", "HourClock.tla"),
             "MCAlternatingBit": os.path.join(REF, "examples", "SpecifyingSystems", "TLC", "MCAlternatingBit.tla")}
    m = Model(paths[name])
    m.ev.out = io.StringIO()
    return m


MODELS = {"LiveClock": lambda: _model("LiveClock"), "LiveLeads": lambda: _model("LiveLeads"),
          "LiveStrongSF": lambda: _model("LiveStrong", "LiveStrongSF"), "LiveGuard": lambda: _model("LiveGuard"),
          "LiveHourClock": lambda: corpus("LiveHourClock"), "MCLiveInternalMemory": lambda: corpus("MCLiveInternalMemory")}


@pytest.mark.parametrize("name", list(MODELS))
def test_label_image_on_the_cpu_reference_equals_the_ast_evaluator(tmp_path, name):
    from tla_rust_b200.checker import compile_model, encode_states
    from tla_rust_b200.compile.lower import compile_labels
    from tla_rust_b200.liveness import LabelPlan
    m = MODELS[name]()
    plan = LabelPlan(m)
    assert plan.queries, name
    cm = compile_model(m)
    img = compile_labels(m, cm, plan.state, plan.edge)
    states, edges, _ = o1_graph(m)
    words = encode_states(cm, states)
    plain = LabelPlan.__new__(LabelPlan)                 # the predicates only, without the derived ENABLED bits
    plain.state, plain.edge, plain.en, plain.nen = plan.state, plan.edge, [], []
    sl, el = ref_labels(m, plain, states, edges)
    L = label_lib(str(tmp_path))
    assert (ref_run_labels(L, cm, img, img.entries["states"], img.n_states, words) == sl).all()
    if edges:
        s_w = words[[s for s, _ in edges]]
        t_w = words[[t for _, t in edges]]
        assert (ref_run_labels(L, cm, img, img.entries["edges"], img.n_edges, s_w, t_w) == el).all()


def test_a_label_image_larger_than_the_models_frame_is_a_compile_error():
    """MCAlternatingBit's obligations need one word more than its kernels' frame: a clean CompileError, which `tlc`
    turns into a warning that the temporal properties are not checked"""
    from tla_rust_b200.checker import compile_model
    from tla_rust_b200.compile.lower import CompileError, compile_labels
    from tla_rust_b200.liveness import LabelPlan, check
    m = corpus("MCAlternatingBit")
    cm = compile_model(m)
    plan = LabelPlan(m)
    with pytest.raises(CompileError, match="liveness labels need a frame of"):
        compile_labels(m, cm, plan.state, plan.edge)
    warned = []
    assert check(None, m, cm, warned.append) is None
    assert warned and "not checked" in warned[-1]


def test_guarded_fairness_is_unfolded_and_unknown_fairness_recorded(tmp_path):
    from tla_rust_b200.front.spec import Model
    assert [f.kind for f in _model("LiveGuard").fairness] == ["WF"]
    assert not _model("LiveGuard", "LiveGuardOff").fairness
    (tmp_path / "U.tla").write_text("---- MODULE U ----\nVARIABLE x\nInit == x = 0\nNext == x' = 1 - x\n"
                                    "Spec == Init /\\ [][Next]_x /\\ \\A i \\in {1, 2} : <>[](x = i)\nP == <>(x = 1)\n====\n")
    (tmp_path / "U.cfg").write_text("SPECIFICATION Spec\nPROPERTY P\n")
    m = Model(str(tmp_path / "U.tla"))
    assert len(m.fairness_unknown) == 1 and len([w for w in m.warnings if "SPECIFICATION" in w]) == 1


# ---- every lasso against the AST evaluator ------------------------------------------------------------------------------
def check_lasso(m, cm, e, ob, r):
    """The lasso r of obligation ob: each step a transition of O1, the spec's fairness holds on it, ob is false on it"""
    from oracle.tlc_oracle import Oracle
    from tla_rust_b200.checker import decode_state
    from tla_rust_b200.front.eval import Fr
    o, ev = Oracle(m), m.ev
    st = lambda row: decode_state(cm, e.read_states(row, 1)[0])
    prefix, cycle = [st(x) for x in r["prefix"]], [st(x) for x in r["cycle"]]
    if ob.kind == "always":
        assert ev.eval(ob.p.node, dict(ob.p.env), Fr(ob.p.ctx, prefix[-1], None)) is not True
        return
    succ = lambda s: [t for t, _ in o.successors(s) if o.key(t) != o.key(s)]
    for a, b in zip(prefix + cycle[1:], prefix[1:] + cycle[1:]):
        assert any(o.key(b) == o.key(t) for t in succ(a))
    steps = list(zip(cycle, cycle[1:] + cycle[:1])) if len(cycle) > 1 else []
    for b in (steps[-1:] if steps else []):
        assert any(o.key(b[1]) == o.key(t) for t in succ(b[0]))
    holds = lambda p, s: ev.eval(p.node, dict(p.env), Fr(p.ctx, s, None)) is True
    act = lambda p, s, t: bool(ev.truth(p.node, dict(p.env), Fr(p.ctx, s, t)))
    enabled = lambda p, s: any(act(p, s, t) for t in succ(s))
    for f in m.fairness:
        a = f.act()
        took = any(act(a, s, t) for s, t in steps)
        if f.kind == "WF":
            assert took or not all(enabled(a, s) for s in cycle), "the lasso is not weakly fair"
        else:
            assert took or not any(enabled(a, s) for s in cycle), "the lasso is not strongly fair"
    if ob.kind == "eventually":
        assert not any(holds(ob.p, s) for s in prefix + cycle)
        assert r["prefix"][0] < e.result()["init_states"]
    elif ob.kind == "leadsto":
        assert holds(ob.p, prefix[0]) and not any(holds(ob.q, s) for s in prefix + cycle)
    elif ob.kind == "inf":
        for kind, p in ob.terms:
            if kind == "ie":
                assert not any(holds(p, s) for s in cycle)
            elif kind == "iea":
                assert not any(act(p, s, t) for s, t in steps)
            else:
                assert not all(holds(p, s) for s in cycle)
    else:
        a = ob.fair.act()
        assert not any(act(a, s, t) for s, t in steps)
        if ob.kind == "wf":
            assert all(enabled(a, s) for s in cycle)
        else:
            assert any(enabled(a, s) for s in cycle)


# ---- GPU ----------------------------------------------------------------------------------------------------------------
CASES = [("LiveClock", None), ("LiveClock", "AlwaysTick"), ("LiveLeads", "Reach2"), ("LiveStrong", "Done"),
         ("LiveStrongSF", None), ("LiveClockSmall", "Small"), ("LiveGuard", None), ("LiveGuardOff", "Done"),
         ("LiveHourClock", None), ("MCLiveInternalMemory", None)]
CFGS = {"LiveClock": ("LiveClock", None), "LiveLeads": ("LiveLeads", None), "LiveStrong": ("LiveStrong", None),
        "LiveStrongSF": ("LiveStrong", "LiveStrongSF"), "LiveClockSmall": ("LiveClock", "LiveClockSmall"),
        "LiveGuard": ("LiveGuard", None), "LiveGuardOff": ("LiveGuard", "LiveGuardOff")}


def _case(name, fails):
    if name == "LiveClock" and fails:
        return _model("LiveClock", "LiveClockNoFair")
    if name in CFGS:
        return _model(*CFGS[name])
    return corpus(name)


def run_case(m, native=False):
    """-> (engine, compiled model, plan, view, store row -> O1 index, O1 states, edges over store rows, labels)"""
    from tla_rust_b200.checker import compile_model, encode_states
    from tla_rust_b200.compile.lower import compile_labels
    from tla_rust_b200.engine import Engine
    from tla_rust_b200.liveness import LabelPlan
    cm = compile_model(m)
    e = Engine(cm, deadlock=False, native=native)
    e.seed(encode_states(cm, [st for st in m.initial_states() if m.in_model(st)]))
    e.run()
    gi = e.build_graph()
    plan = LabelPlan(m)
    e.label_graph(compile_labels(m, cm, plan.state, plan.edge), *plan.en_map())
    return e, cm, plan, gi


@pytest.mark.gpu
@pytest.mark.parametrize("hook", [None, "TLAG_NO_SORT", "TLAG_GRAPH_EDGES"])
@pytest.mark.parametrize("name,fails", CASES)
def test_live_check_matches_the_reference(name, fails, hook, monkeypatch):
    from tla_rust_b200.checker import encode_states
    from tla_rust_b200.engine import live_check
    if hook is not None and name not in ("LiveLeads", "LiveStrong", "MCLiveInternalMemory"):
        pytest.skip("the store-order hooks run on three models")
    if hook:
        monkeypatch.setenv(hook, "1" if hook == "TLAG_NO_SORT" else "4096")
    m = _case(name, fails)
    e, cm, plan, gi = run_case(m)
    view = e.graph_view()
    states, edges, _ = o1_graph(m)
    rows = e.read_states(0, gi["n_states"])
    key = {bytes(w): i for i, w in enumerate(encode_states(cm, states))}
    perm = [key[bytes(w)] for w in rows]            # store row -> O1 index
    inv = {o: r for r, o in enumerate(perm)}
    redges = sorted((inv[s], inv[t]) for s, t in edges)
    off, dst, _ = e.state_graph()
    assert sorted((s, int(dst[j])) for s in range(len(perm)) for j in range(int(off[s]), int(off[s + 1]))) == redges
    sl, el = ref_labels(m, plan, [states[p] for p in perm], redges)
    failed = None
    for ob, q in plan.queries:
        args = plan.args(q, view.n_init)
        r = live_check(view, **args)
        witness, n_fair = ref_check(len(perm), redges, sl, el, args)
        assert (r["violated"], r["witness"]) == (witness is not None, witness), ob.name
        if not args["flags"] & 2:
            assert r["fair_sccs"] == n_fair, ob.name
        if r["violated"]:
            assert r["prefix"][-1] == r["cycle"][0] if r["cycle"] else r["prefix"] == [witness]
            check_lasso(m, cm, e, ob, r)
            failed = failed or ob
    assert (failed and failed.name) == fails
    e.close()


@pytest.mark.gpu
def test_sliced_engine_labels_and_verdicts_equal_the_interpreter():
    from tla_rust_b200.engine import live_check
    got = {}
    for native in (False, "sliced"):
        for cfg in (None, "LiveStrongSF"):
            m = _model("LiveStrong", cfg)
            e, cm, plan, gi = run_case(m, native)
            view = e.graph_view()
            rows = [bytes(w) for w in e.read_states(0, gi["n_states"])]
            out = []
            for ob, q in plan.queries:
                r = live_check(view, **plan.args(q, view.n_init))
                out.append((r["violated"], r["fair_sccs"], [rows[x] for x in r["prefix"] + r["cycle"]]))
                if r["violated"]:
                    check_lasso(m, cm, e, ob, r)
            got[(native, cfg)] = out
            e.close()
    assert got[(False, None)] == got[("sliced", None)] and got[(False, None)][0][0]
    assert got[(False, "LiveStrongSF")] == got[("sliced", "LiveStrongSF")] and not got[(False, "LiveStrongSF")][0][0]


COUNTERS = """---- MODULE Counters ----
EXTENDS Naturals
VARIABLE c
Init == c = [i \\in 1..7 |-> 0]
Inc(i) == c' = [c EXCEPT ![i] = (c[i] + 1) % 10]
Next == \\E i \\in 1..7 : Inc(i)
Spec == Init /\\ [][Next]_c /\\ \\A i \\in 1..7 : WF_c(Inc(i))
Spec6 == Init /\\ [][Next]_c /\\ \\A i \\in 2..7 : WF_c(Inc(i))
Zero == \\A i \\in 1..7 : []<>(c[i] = 0)
====
"""


@pytest.mark.gpu
def test_scale_seven_counters(tmp_path):
    """7 counters mod 10 (10^7 states, 7 * 10^7 edges): []<>(c[i] = 0) holds under WF on every Inc(i) and fails, with a
    lasso the evaluator accepts, when WF on Inc(1) is dropped"""
    from tla_rust_b200.engine import live_check
    from tla_rust_b200.front.spec import Model
    (tmp_path / "Counters.tla").write_text(COUNTERS)
    for spec, want in (("Spec", False), ("Spec6", True)):
        (tmp_path / "Counters.cfg").write_text(f"SPECIFICATION {spec}\nPROPERTY Zero\n")
        m = Model(str(tmp_path / "Counters.tla"))
        m.ev.out = io.StringIO()
        e, cm, plan, gi = run_case(m)
        assert (gi["n_states"], gi["n_edges"]) == (10 ** 7, 7 * 10 ** 7)
        view = e.graph_view()
        results = [(ob, live_check(view, **plan.args(q, view.n_init))) for ob, q in plan.queries]
        assert any(r["violated"] for _, r in results) == want
        for ob, r in results:
            if r["violated"]:
                assert ob.terms[0][1].env == {"i": 1}
                check_lasso(m, cm, e, ob, r)
        e.close()


@pytest.mark.gpu
def test_tlc_reports_liveness(monkeypatch):
    from tla_rust_b200.cli import check_file
    monkeypatch.setenv("TLAG_NO_STATES_DIR", "1")

    def run(name, cfg=None):
        out = io.StringIO()
        rc = check_file(os.path.join(SPECS, name + ".tla"), cfg_path=os.path.join(SPECS, cfg + ".cfg") if cfg else None,
                        out=out, engine="interp", deadlock=False)
        return rc, out.getvalue()
    rc, text = run("LiveClock")
    assert rc == 0 and "No error has been found" in text and "Checking temporal properties" in text
    rc, text = run("LiveClock", "LiveClockNoFair")
    assert rc == 12 and "Error: Temporal properties were violated." in text
    assert "State 1: <Initial predicate>" in text and "State 2: Stuttering" in text
    rc, text = run("LiveLeads")
    assert rc == 12 and "Back to state " in text
    rc, text = run("LiveStrong")
    assert rc == 12 and "Temporal properties were violated" in text
    assert run("LiveStrong", "LiveStrongSF")[0] == 0
    assert run("LiveGuard")[0] == 0 and run("LiveGuard", "LiveGuardOff")[0] == 12
    rc, text = run("LiveClock", "LiveClockSmall")
    assert rc == 12 and "Error: Invariant Small is violated." in text
