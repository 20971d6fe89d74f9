"""`tlc`'s liveness check (DESIGN.md §7h): the fairness conditions and the temporal PROPERTY obligations of a model
(front/spec.py) become label bits, a label image (compile/lower.py compile_labels) labels the state graph on the device,
and each obligation is one query of tlag_live_check on that graph."""
from __future__ import annotations

from .compile.lower import compile_labels


class LabelPlan:
    """Label bits of a model: state predicates take state bits [0, len(state)), the ENABLED bits (and complements) of
    the actions the bits after them; actions <<A>>_v take edge bits.  queries: (obligation, tlag_live_check arguments)."""

    def __init__(self, m):
        self.state, self.edge = [], []              # Pred lists
        self._skey, self._ekey = {}, {}
        self.en, self.nen = [], []                  # edge bits whose ENABLED / ~ENABLED state bit is derived
        self.queries, self.skipped = [], []
        self.fairness = []                          # (kind, ("en", edge bit), edge bit)
        for f in m.fairness:
            a = self._edge(f.act())
            self._need(self.en, a)
            self.fairness.append((f.kind, ("en", a), a))
        if not self._fits():
            raise ValueError("the fairness conditions need more than 32 state or edge label bits")
        for ob in m.obligations:
            saved = (list(self.state), list(self.edge), dict(self._skey), dict(self._ekey), list(self.en), list(self.nen))
            q = self._query(ob)
            if self._fits():
                self.queries.append((ob, q))
            else:
                self.state, self.edge, self._skey, self._ekey, self.en, self.nen = saved
                self.skipped.append(ob)

    def _fits(self):
        return len(self.state) + len(self.en) + len(self.nen) <= 32 and len(self.edge) <= 32

    def _state(self, p):
        k = p.key()
        if k not in self._skey:
            self._skey[k] = len(self.state)
            self.state.append(p)
        return ("p", self._skey[k])

    def _edge(self, p):
        k = p.key()
        if k not in self._ekey:
            self._ekey[k] = len(self.edge)
            self.edge.append(p)
        return self._ekey[k]

    @staticmethod
    def _need(lst, a):
        if a not in lst:
            lst.append(a)

    def _query(self, ob):
        q = {"keep_set": [], "keep_clear": [], "edge_drop": [], "need_clear": [], "seed_set": [], "seed_clear": [],
             "flags": 0, "init_only": False}
        if ob.kind == "always":
            q["flags"] = 2
            q["seed_clear"].append(self._state(ob.p))
        elif ob.kind == "eventually":
            p = self._state(ob.p)
            q["flags"], q["init_only"] = 1, True
            q["seed_clear"].append(p)
            q["keep_clear"].append(p)
        elif ob.kind == "leadsto":
            p, r = self._state(ob.p), self._state(ob.q)
            q["flags"] = 1
            q["seed_set"].append(p)
            q["seed_clear"].append(r)
            q["keep_clear"].append(r)
        elif ob.kind == "inf":
            for kind, pred in ob.terms:
                if kind == "ie":
                    q["keep_clear"].append(self._state(pred))
                elif kind == "iea":
                    q["edge_drop"].append(self._edge(pred))
                else:
                    q["need_clear"].append(self._state(pred))
        else:                                       # WF / SF asserted as a property
            a = self._edge(ob.fair.act())
            q["edge_drop"].append(a)
            if ob.kind == "wf":
                self._need(self.en, a)
                q["keep_set"].append(("en", a))
            else:
                self._need(self.nen, a)
                q["need_clear"].append(("nen", a))
        return q

    def bit(self, ref):
        """the state bit of ("p", j), ("en", a) or ("nen", a)"""
        kind, j = ref
        if kind == "p":
            return j
        if kind == "en":
            return len(self.state) + self.en.index(j)
        return len(self.state) + len(self.en) + self.nen.index(j)

    def en_map(self):
        return {a: self.bit(("en", a)) for a in self.en}, {a: self.bit(("nen", a)) for a in self.nen}

    def args(self, q, n_init):
        """tlag_live_check's arguments for one query"""
        mask = lambda refs: sum(1 << self.bit(r) for r in set(refs))
        return dict(fairness=[(k, self.bit(en), a) for k, en, a in self.fairness], keep_set=mask(q["keep_set"]),
                    keep_clear=mask(q["keep_clear"]), edge_drop=sum(1 << a for a in set(q["edge_drop"])),
                    need_clear=mask(q["need_clear"]), seed_set=mask(q["seed_set"]), seed_clear=mask(q["seed_clear"]),
                    seed_rows=n_init if q["init_only"] else 0, flags=q["flags"])


def check(e, m, cm, warn):
    """Check every obligation of model m on engine e's state graph (the search at its fixpoint).
    -> None when all hold, else (obligation, live_check result)"""
    from .compile.lower import CompileError
    from .engine import EngineError, live_check
    try:
        plan = LabelPlan(m)
    except ValueError as ex:
        warn(f"the temporal properties are not checked: {ex}")
        return None
    for ob in plan.skipped:
        warn(f"PROPERTY {ob.name}: the conjunct at line {ob.loc[0]}, col {ob.loc[1]} needs more than 32 label bits; "
             f"it is not checked")
    if not plan.queries:
        return None
    try:
        img = compile_labels(m, cm, plan.state, plan.edge)
    except CompileError as ex:
        warn(f"the temporal properties are not checked: their predicates do not compile: {ex}")
        return None
    e.build_graph()
    en, nen = plan.en_map()
    try:
        e.label_graph(img, en, nen)
    except EngineError as ex:
        if "rc=-6" not in str(ex):              # TLAG_EEVAL: a predicate trapped; anything else is an error
            raise
        warn(f"the temporal properties are not checked: {ex}")
        return None
    view = e.graph_view()
    for ob, q in plan.queries:
        r = live_check(view, **plan.args(q, view.n_init))
        if r["violated"]:
            return ob, r
    return None


def edge_action(e, s, t):
    """the action id of an edge s -> t of e's state graph"""
    off, dst, act = e.state_graph(s, 1)
    for j in range(int(off[1])):
        if int(dst[j]) == t:
            return int(act[j])
    raise ValueError(f"no edge {s} -> {t} in the state graph")


def lasso(e, r):
    """-> (trace [(words, action id)], index in the trace the cycle goes back to, or None: the last state stutters) of a
    violation: the parent chain of the lasso's first row, the rest of its prefix, its cycle"""
    states, acts = e.trace(r["prefix"][0], cap=int(e.result()["depth"]) + 1)     # a parent chain has at most depth states
    trace = list(zip(states, acts.tolist()))
    rows = r["prefix"][1:] + r["cycle"][1:]
    prev = r["prefix"][0]
    for t in rows:
        trace.append((e.read_states(t, 1)[0], edge_action(e, prev, t)))
        prev = t
    if len(r["cycle"]) <= 1:
        return trace, None, None
    back = len(trace) - len(r["cycle"])       # 0-based index of the cycle's first state
    return trace, back, edge_action(e, prev, r["cycle"][0])
