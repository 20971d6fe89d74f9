"""Module loading (EXTENDS / INSTANCE), TLC .cfg parsing and model assembly.

cfg grammar: examples/SpecifyingSystems/TLC/ConfigFileGrammar.tla:8-33 plus the
module-scoped override `c <-[Mod] d` used by examples/Paxos/MCPaxos.cfg:9 and the
comment forms of MCInnerSerial.cfg:2-5.  `=` vs `<-` semantics:
CachingMemory/MCInternalMemory.cfg:24-33.
"""
from __future__ import annotations

import os
import re

from .parser import parse_module_text, read_text, Node, OpDef, Module
from .values import ModelValue, EvalError, fmt
from .eval import Evaluator, ModCtx, Fr

STD_MODULES = {"Naturals", "Integers", "Reals", "Sequences", "FiniteSets", "TLC", "Bags",
               "Peano", "ProtoReals", "RealTime_"}


class SpecError(Exception):
    pass


class Loader:
    def __init__(self, dirs):
        self.dirs = list(dirs)
        self.cache = {}
        self.texts = {}

    def add_text(self, name, text):
        self.texts[name] = text

    def load(self, name) -> Module:
        m = self.cache.get(name)
        if m is not None:
            return m
        if name in self.texts:
            m = parse_module_text(self.texts[name])
        else:
            for d in self.dirs:
                p = os.path.join(d, name + ".tla")
                if os.path.exists(p):
                    m = parse_module_text(read_text(p))
                    break
            else:
                raise SpecError(f"cannot find module {name}.tla in {self.dirs}")
        self.cache[name] = m
        return m


def build_ctx(loader: Loader, modname: str) -> ModCtx:
    ctx = ModCtx(modname)
    _merge_module(loader, loader.load(modname), ctx, root=ctx)
    return ctx


def _merge_module(loader, m: Module, ctx: ModCtx, root: ModCtx):
    if m.name in ctx.extended:
        return
    ctx.extended.add(m.name)
    for ext in m.extends:
        if ext in STD_MODULES:
            continue
        _merge_module(loader, loader.load(ext), ctx, root)
    for name, ar in m.constants:
        ctx.const_decls[name] = ar
    for v in m.variables:
        if v not in ctx.varset:
            ctx.vars.append(v)
            ctx.varset.add(v)
    for name, d in m.defs.items():
        ctx.defs[name] = (d, ctx)
    for nm, e in m.assumes:
        ctx.assumes.append((nm, e, ctx))
    for inst in m.instances:
        if inst.module in STD_MODULES:
            continue
        if inst.params:
            continue  # parametrised instances are not supported
        child = ModCtx(inst.module)
        cm = loader.load(inst.module)
        _merge_module(loader, cm, child, root)
        explicit = dict(inst.substs)
        for nm in list(child.const_decls) + list(child.vars):
            if nm in explicit:
                child.substs[nm] = (explicit[nm], ctx)
            else:
                child.substs[nm] = (Node("id", (nm,)), ctx)
        root.all_instances.append(child)
        if inst.name is not None:
            ctx.instances[inst.name] = child
        else:
            for nm, pair in child.defs.items():
                if not pair[0].local and nm not in ctx.defs:
                    ctx.defs[nm] = pair
            for nm, ic in child.instances.items():
                ctx.instances.setdefault(nm, ic)


# ---------------------------------------------------------------------------
class Cfg:
    def __init__(self):
        self.specification = None
        self.init = None
        self.next = None
        self.invariants = []
        self.properties = []
        self.constraints = []
        self.action_constraints = []
        self.symmetry = None
        self.view = None
        self.const_assign = []    # (name, value)
        self.const_subst = []     # (name, module|None, defname)
        self.check_deadlock = None


_CFG_KW = {"SPECIFICATION", "INIT", "NEXT", "INVARIANT", "INVARIANTS", "PROPERTY", "PROPERTIES",
           "CONSTRAINT", "CONSTRAINTS", "ACTION-CONSTRAINT", "ACTION-CONSTRAINTS", "ACTION_CONSTRAINT",
           "ACTION_CONSTRAINTS", "SYMMETRY", "VIEW", "CONSTANT", "CONSTANTS", "CHECK_DEADLOCK", "ALIAS",
           "POSTCONDITION"}


def _cfg_tokens(text):
    # strip comments
    out = []
    i, n = 0, len(text)
    depth = 0
    buf = []
    while i < n:
        if text.startswith("(*", i):
            depth += 1
            i += 2
            continue
        if depth > 0:
            if text.startswith("*)", i):
                depth -= 1
                i += 2
            else:
                i += 1
            continue
        if text.startswith("\\*", i):
            while i < n and text[i] != "\n":
                i += 1
            continue
        buf.append(text[i])
        i += 1
    text = "".join(buf)
    tok_re = re.compile(r'\s*(<-\[[A-Za-z0-9_]+\]|<-|"(?:[^"\\]|\\.)*"|ACTION-CONSTRAINTS?|[A-Za-z0-9_!]+|-?\d+|[{},=])')
    pos = 0
    toks = []
    while pos < len(text):
        m = tok_re.match(text, pos)
        if not m:
            if text[pos:].strip() == "":
                break
            raise SpecError(f"cfg: cannot tokenise near {text[pos:pos+30]!r}")
        toks.append(m.group(1))
        pos = m.end()
    return toks


def _cfg_value(toks, i):
    t = toks[i]
    if t == "{":
        i += 1
        items = []
        while toks[i] != "}":
            v, i = _cfg_value(toks, i)
            items.append(v)
            if toks[i] == ",":
                i += 1
        return frozenset(items), i + 1
    if t.startswith('"'):
        return bytes(t[1:-1], "utf-8").decode("unicode_escape"), i + 1
    if re.fullmatch(r"-?\d+", t):
        return int(t), i + 1
    if t == "TRUE":
        return True, i + 1
    if t == "FALSE":
        return False, i + 1
    return ModelValue(t), i + 1


def parse_cfg(text: str) -> Cfg:
    toks = _cfg_tokens(text)
    cfg = Cfg()
    i = 0
    n = len(toks)
    while i < n:
        kw = toks[i]
        if kw not in _CFG_KW:
            raise SpecError(f"cfg: unexpected token {kw!r}")
        i += 1
        if kw == "SPECIFICATION":
            cfg.specification = toks[i]
            i += 1
        elif kw == "INIT":
            cfg.init = toks[i]
            i += 1
        elif kw == "NEXT":
            cfg.next = toks[i]
            i += 1
        elif kw == "SYMMETRY":
            cfg.symmetry = toks[i]
            i += 1
        elif kw == "VIEW":
            cfg.view = toks[i]
            i += 1
        elif kw == "CHECK_DEADLOCK":
            cfg.check_deadlock = toks[i] == "TRUE"
            i += 1
        elif kw in ("ALIAS", "POSTCONDITION"):
            i += 1
        elif kw in ("CONSTANT", "CONSTANTS"):
            while i < n and toks[i] not in _CFG_KW:
                name = toks[i]
                op = toks[i + 1]
                if op == "=":
                    v, i = _cfg_value(toks, i + 2)
                    cfg.const_assign.append((name, v))
                elif op == "<-":
                    cfg.const_subst.append((name, None, toks[i + 2]))
                    i += 3
                elif op.startswith("<-["):
                    cfg.const_subst.append((name, op[3:-1], toks[i + 2]))
                    i += 3
                else:
                    raise SpecError(f"cfg: bad constant binding for {name}")
        else:
            lst = {"INVARIANT": cfg.invariants, "INVARIANTS": cfg.invariants, "PROPERTY": cfg.properties,
                   "PROPERTIES": cfg.properties, "CONSTRAINT": cfg.constraints, "CONSTRAINTS": cfg.constraints,
                   }.get(kw, cfg.action_constraints)
            while i < n and toks[i] not in _CFG_KW:
                lst.append(toks[i])
                i += 1
    return cfg


# ---------------------------------------------------------------------------
_TEMPORAL = {"box", "diamond", "wf", "sf", "tforall", "texists"}


def _has_temporal(n, ctx, seen=None, depth=0):
    if not isinstance(n, Node):
        if isinstance(n, (tuple, list)):
            return any(_has_temporal(x, ctx, seen, depth) for x in n)
        return False
    if n.k in _TEMPORAL:
        return True
    if n.k == "bin" and n.a[0] in ("~>", "-+->"):
        return True
    if n.k == "id" and depth < 8:
        d = ctx.defs.get(n.a[0])
        if d is not None and not d[0].params:
            seen = seen or set()
            if n.a[0] in seen:
                return False
            seen.add(n.a[0])
            return _has_temporal(d[0].body, d[1], seen, depth + 1)
        return False
    if n.k == "let":
        return _has_temporal(n.a[1], ctx, seen, depth)
    return any(_has_temporal(x, ctx, seen, depth) for x in n.a)


def _state_pred(n, ctx, seen=None, depth=0):
    """n is a state predicate: no temporal operator, prime, ENABLED, UNCHANGED or action form, definitions included"""
    if not isinstance(n, Node):
        if isinstance(n, (tuple, list)):
            return all(_state_pred(x, ctx, seen, depth) for x in n)
        return True
    if n.k in _TEMPORAL or n.k in ("prime", "enabled", "unchanged", "aangle", "abox"):
        return False
    if n.k == "bin" and n.a[0] in ("~>", "-+->", "\\cdot"):
        return False
    if n.k in ("id", "app") and depth < 8 and isinstance(n.a[0], str):
        d = ctx.defs.get(n.a[0])
        if n.k == "app" and not _state_pred(n.a[1], ctx, seen, depth):
            return False
        if d is not None:
            seen = seen or set()
            if n.a[0] in seen:
                return True
            seen.add(n.a[0])
            return _state_pred(d[0].body, d[1], seen, depth + 1)
        return True
    if n.k == "let":
        return _state_pred(n.a[1], ctx, seen, depth)
    return all(_state_pred(x, ctx, seen, depth) for x in n.a)


class Pred:
    """A state predicate, or an action (<<A>>_v), with the context and the bound variables it is evaluated in"""

    def __init__(self, node, ctx, env):
        self.node, self.ctx, self.env = node, ctx, dict(env)

    def key(self):
        return (repr(self.node), id(self.ctx), repr(sorted(self.env.items(), key=lambda kv: kv[0])))


class Fairness:
    """WF_v(A) or SF_v(A): kind "WF" / "SF"; act() is <<A>>_v as a Pred"""

    def __init__(self, kind, a, sub, ctx, env, loc):
        self.kind, self.a, self.sub, self.ctx, self.env, self.loc = kind, a, sub, ctx, dict(env), loc

    def act(self):
        return Pred(Node("aangle", (self.a, self.sub), *self.loc), self.ctx, self.env)


class Obligation:
    """One temporal PROPERTY conjunct in normal form (DESIGN.md §7h).  kind:
      "always" []p, "eventually" <>p, "leadsto" p ~> q, "inf" a disjunction of terms ("ie", X) []<>X, ("iea", A)
      []<><<A>>_v, ("eg", X) <>[]X, "wf" / "sf" a fairness condition asserted as a property (fair)."""

    def __init__(self, name, loc, kind, p=None, q=None, terms=(), fair=None):
        self.name, self.loc, self.kind, self.p, self.q, self.terms, self.fair = name, loc, kind, p, q, list(terms), fair


class Model:
    """A checkable model: root context + Init / Next / invariants, after cfg application."""

    def __init__(self, tla_path: str, cfg_path: str | None = None, cfg_text: str | None = None,
                 extra_dirs=(), loader: Loader | None = None, module_name: str | None = None):
        self.tla_path = tla_path
        d = os.path.dirname(os.path.abspath(tla_path)) if tla_path else "."
        self.loader = loader or Loader([d] + list(extra_dirs))
        self.module_name = module_name or os.path.splitext(os.path.basename(tla_path))[0]
        self.ev = Evaluator()
        self.ctx = build_ctx(self.loader, self.module_name)
        if cfg_text is None:
            if cfg_path is None:
                cfg_path = os.path.splitext(tla_path)[0] + ".cfg"
            if os.path.exists(cfg_path):
                cfg_text = read_text(cfg_path)
            else:
                cfg_text = ""
        self.cfg = parse_cfg(cfg_text)
        self.warnings = []
        if self.cfg.view:
            # TLC would fingerprint the VIEW expression instead of the whole state; here every state is distinguished by
            # all of its variables (a superset of the view's classes: sound, possibly more states)
            self.warnings.append(f"cfg: VIEW {self.cfg.view} is not applied -- states are identified by all variables")
        self._apply_cfg()
        self._assemble()

    # -- cfg -----------------------------------------------------------------
    def _apply_cfg(self):
        ctx, cfg = self.ctx, self.cfg
        for name, v in cfg.const_assign:
            ctx.consts[name] = v
        for name, mod, dname in cfg.const_subst:
            targets = [ctx] if mod is None else [c for c in ctx.all_instances if mod in c.extended]
            if mod is not None and not targets:
                self.warnings.append(f"cfg: no instance of module {mod} for override of {name}")
            src = ctx.defs.get(dname)
            if src is None:
                raise SpecError(f"cfg: {dname} (override for {name}) is not defined")
            for tc in targets:
                tc.defs[name] = src
                tc.consts.pop(name, None)
                tc.substs.pop(name, None)
        for c in [ctx] + ctx.all_instances:
            c.cache.clear()
        # every declared constant must be bound
        for name in ctx.const_decls:
            if name not in ctx.consts and name not in ctx.defs:
                raise SpecError(f"constant {name} is not assigned a value by the configuration file")

    def _def(self, name):
        d = self.ctx.defs.get(name)
        if d is None:
            raise SpecError(f"{name} (named in the cfg) is not defined in module {self.module_name}")
        return d

    def _assemble(self):
        cfg, ctx = self.cfg, self.ctx
        self.init_nodes = []
        self.next_node = None
        self.next_ctx = ctx
        self.vars = list(ctx.vars)
        self.fairness = []
        self.fairness_unknown = []      # source locations of SPECIFICATION temporal conjuncts outside the supported forms
        if cfg.specification:
            self._split_spec(Node("id", (cfg.specification,)), ctx)
        else:
            if cfg.init:
                d, c = self._def(cfg.init)
                self.init_nodes.append((d.body, c))
            if cfg.next:
                d, c = self._def(cfg.next)
                self.next_node, self.next_ctx = Node("id", (cfg.next,)), ctx
        self.invariants = []
        for nm in cfg.invariants:
            d, c = self._def(nm)
            self.invariants.append((nm, d.body, c))
        self.constraints = []
        for nm in cfg.constraints:
            d, c = self._def(nm)
            self.constraints.append((nm, d.body, c))
        self.action_constraints = []
        for nm in cfg.action_constraints:
            d, c = self._def(nm)
            self.action_constraints.append((nm, d.body, c))
        # PROPERTYs: the safety part  Init2 /\\ [][Next2]_v2  becomes a refinement obligation: Init => Init2 and
        # every transition satisfies [Next2]_v2 (MCPaxos.cfg:12, MCVoting.cfg:9, HourClock2.cfg:9); each temporal
        # conjunct in one of the forms of DESIGN.md §7h becomes a liveness obligation (checked on the state graph), any
        # other one is ignored with a warning that names it.
        self.properties = list(cfg.properties)
        self.refinements = []
        self.obligations = []
        for nm in cfg.properties:
            d, c = self._def(nm)
            acc = {"init": [], "next": None, "sub": None, "ctx": None, "name": nm}
            self._split_prop(d.body, c, acc)
            if acc["next"] is not None or acc["init"]:
                self.refinements.append((nm, acc["init"], acc["next"], acc["sub"], acc["ctx"]))
        self.symmetry = cfg.symmetry
        self.check_deadlock = True if cfg.check_deadlock is None else cfg.check_deadlock

    def _conjuncts(self, n, ctx, env=None):
        """The conjuncts of n, as (node, ctx, env): through conjunction lists, parameterless definitions and instance
        selectors whose bodies are temporal, and  \\A x \\in S : body  with a temporal body and S a finite constant
        set (one conjunct per element, x bound in env)."""
        env = env or {}
        if n.k == "and":
            for x in n.a[0]:
                yield from self._conjuncts(x, ctx, env)
            return
        if n.k == "id" and n.a[0] not in env:
            d = ctx.defs.get(n.a[0])
            if d is not None and not d[0].params and _has_temporal(d[0].body, d[1]):
                yield from self._conjuncts(d[0].body, d[1])
                return
        if n.k == "sel":
            r = self.ev.resolve_sel(n.a[0], {}, Fr(ctx))
            if r[0] == "def" and not r[1].params and _has_temporal(r[1].body, r[2]):
                yield from self._conjuncts(r[1].body, r[2])
                return
        if n.k == "bin" and n.a[0] == "=>" and _has_temporal(n.a[2], ctx) and not _has_temporal(n.a[1], ctx):
            try:                 # a constant-level guard (InnerSerial.tla:116): the conjunct applies when it holds
                g = self.ev.eval(n.a[1], env, Fr(ctx))
            except EvalError:
                g = None
            if g is True:
                yield from self._conjuncts(n.a[2], ctx, env)
                return
            if g is False:
                return
        if n.k == "forall" and _has_temporal(n.a[1], ctx):
            try:
                envs = list(self.ev.iter_bounds(n.a[0], env, Fr(ctx)))
            except EvalError:
                envs = None
            if envs is not None:
                for env2 in envs:
                    yield from self._conjuncts(n.a[1], ctx, env2)
                return
        yield n, ctx, env

    def _split_spec(self, n, ctx):
        """Decompose  Init /\\ [][Next]_vars /\\ fairness  (SURVEY.md §3.2)."""
        for x, c, env in self._conjuncts(n, ctx):
            if x.k == "box" and x.a[0].k == "abox":
                if self.next_node is not None:
                    raise SpecError("specification has more than one [][Next]_v conjunct")
                self.next_node = x.a[0].a[0]
                self.next_ctx = c
                self.subscript = x.a[0].a[1]
            elif x.k in ("wf", "sf"):
                self.fairness.append(Fairness(x.k.upper(), x.a[1], x.a[0], c, env, x.loc()))
            elif _has_temporal(x, c):
                # the fairness the spec states is not known: a liveness verdict could be wrong either way
                if x.loc() not in self.fairness_unknown:
                    self.fairness_unknown.append(x.loc())
                    self.warnings.append(f"SPECIFICATION {self.cfg.specification}: the temporal conjunct at line "
                                         f"{x.line}, col {x.col} is not a WF or SF condition in a supported form")
            else:
                self.init_nodes.append((x, c))

    def symmetry_group(self):
        """Non-identity elements of the group generated by the SYMMETRY set (Paxos/MCPaxos.cfg:13:
        Permutations(MCAcceptor) \\cup Permutations(MCValue)).  TLC applies the listed permutations as given; a
        set that is not closed under composition does not define an equivalence, so the generated group is used
        (identical to TLC's result whenever the listed set is itself a group)."""
        if not self.symmetry:
            return []
        from .values import permutation_group, to_finite, Fcn, ModelValue
        d, c = self._def(self.symmetry)
        val = to_finite(self.ev.eval(d.body, {}, Fr(c)))
        perms = []
        for f in val:
            if isinstance(f, tuple):
                raise SpecError("SYMMETRY permutations must be over model values")
            if not isinstance(f, Fcn) or not all(isinstance(k, ModelValue) and isinstance(x, ModelValue)
                                                 for k, x in f.d.items()):
                raise SpecError("SYMMETRY must be a set of permutations of model values")
            perms.append(dict(f.d))
        return permutation_group(perms)

    def _split_prop(self, n, ctx, acc):
        for x, c, env in self._conjuncts(n, ctx):
            if x.k == "box" and x.a[0].k == "abox":
                acc["next"], acc["sub"], acc["ctx"] = x.a[0].a[0], x.a[0].a[1], c
            elif _has_temporal(x, c):
                ob = self._obligation(x, c, env, acc["name"])
                if ob is None and x.loc() not in acc.setdefault("warned", set()):
                    acc["warned"].add(x.loc())
                    self.warnings.append(f"PROPERTY {acc['name']}: the temporal (liveness) conjunct at line {x.line}, "
                                         f"col {x.col} is not checked (not one of the forms of DESIGN.md §7h)")
                elif ob is not None:
                    self.obligations.append(ob)
            else:
                acc["init"].append((x, c))

    def _unfold(self, n, ctx):
        """n with parameterless definitions and instance selectors replaced by their bodies (one level at a time)"""
        for _ in range(16):
            if n.k == "id" and ctx.defs.get(n.a[0]) is not None and not ctx.defs[n.a[0]][0].params:
                n, ctx = ctx.defs[n.a[0]][0].body, ctx.defs[n.a[0]][1]
            elif n.k == "sel":
                r = self.ev.resolve_sel(n.a[0], {}, Fr(ctx))
                if r[0] != "def" or r[1].params:
                    break
                n, ctx = r[1].body, r[2]
            else:
                break
        return n, ctx

    def _obligation(self, n, ctx, env, name):
        """The liveness obligation of a temporal PROPERTY conjunct (DESIGN.md §7h), or None outside its forms"""
        sp = lambda x, c: _state_pred(x, c) and Pred(x, c, env)

        def term(x, c):          # []<>X, []<><<A>>_v, <>[]X -> ("ie" | "iea" | "eg", Pred)
            x, c = self._unfold(x, c)
            if x.k == "box":
                y, c2 = self._unfold(x.a[0], c)
                if y.k == "diamond":
                    z = y.a[0]
                    if z.k == "aangle" and not _has_temporal(z, c2):
                        return "iea", Pred(z, c2, env)
                    p = sp(z, c2)
                    return p and ("ie", p)
            if x.k == "diamond":
                y, c2 = self._unfold(x.a[0], c)
                if y.k == "box":
                    p = sp(y.a[0], c2)
                    return p and ("eg", p)
            return None

        loc = n.loc()
        if n.k in ("wf", "sf"):
            return Obligation(name, loc, n.k, fair=Fairness(n.k.upper(), n.a[1], n.a[0], ctx, env, loc))
        if n.k == "bin" and n.a[0] == "~>":
            p, q = sp(n.a[1], ctx), sp(n.a[2], ctx)
            return Obligation(name, loc, "leadsto", p=p, q=q) if p and q else None
        t = term(n, ctx)
        if t:
            return Obligation(name, loc, "inf", terms=[t])
        if n.k == "or":
            terms = [term(x, ctx) for x in n.a[0]]
            return Obligation(name, loc, "inf", terms=terms) if all(terms) else None
        if n.k == "box":
            p = sp(n.a[0], ctx)
            return Obligation(name, loc, "always", p=p) if p else None
        if n.k == "diamond":
            p = sp(n.a[0], ctx)
            return Obligation(name, loc, "eventually", p=p) if p else None
        return None

    def in_model(self, st) -> bool:
        """CONSTRAINTs on a state (host side: used for the initial states; on successors the device evaluates them)"""
        from .eval import Fr
        for _nm, node, c in self.constraints:
            if self.ev.eval(node, {}, Fr(c, st, None)) is not True:
                return False
        return True

    def check_refinement_init(self, st):
        """Init => Init2 for every refinement PROPERTY; returns the name of a violated property or None."""
        for nm, inits, _, _, _ in self.refinements:
            for node, c in inits:
                if self.ev.eval(node, {}, Fr(c, st, None)) is not True:
                    return nm
        return None

    # -- evaluation helpers ------------------------------------------------------
    def check_assumes(self):
        """Evaluate every ASSUME (SimpleMath.tla, PrintValues.tla:48-54, Paxos.tla:13)."""
        res = []
        for nm, e, c in self.ctx.assumes:
            v = self.ev.eval(e, {}, Fr(c))
            res.append((nm, v))
            if v is not True:
                raise SpecError(f"Assumption {nm or ''} line {e.line} is false")
        return res

    def initial_states(self):
        """Enumerate initial states (dict var -> value) in TLC order (lexicographic, SURVEY §3.4)."""
        if not self.init_nodes:
            raise SpecError("no initial predicate")
        nodes = [n for n, _ in self.init_nodes]
        ctx = self.init_nodes[0][1]
        conj = Node("and", (tuple(nodes),)) if len(nodes) > 1 else nodes[0]
        out = []
        for asg, _ in self.ev.solve(conj, {}, ctx, None, {}, "cur"):
            missing = [v for v in self.vars if v not in asg]
            if missing:
                raise SpecError(f"initial predicate does not assign {missing}")
            out.append(asg)
        return out

    def eval_const(self, name):
        return self.ev.lookup(name, {}, Fr(self.ctx))
