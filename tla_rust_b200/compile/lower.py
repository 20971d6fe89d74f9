"""Lowering of a Model (Next action, invariants, constraints) to fixed-width bytecode.

Pipeline (SURVEY.md §7 step 3, north_star "lowers each next-state action and invariant
to a fixed-width state-vector bytecode"):
  1. variable types from a TypeOK-style definition (or widened shapes of the initial
     states) -> state layout (compile/types.py)
  2. Next -> one straight-line program with guards, loops over runtime sets and an
     EMIT per completed successor (continuation-passing over TLC's conjunct/disjunct
     evaluation order; constant quantifiers are unrolled, constant subexpressions are
     folded by the host evaluator)
  3. invariants / constraints -> predicate programs over the unpacked state.
"""
from __future__ import annotations

import re

from ..front.parser import Node, OpDef
from ..front.eval import Evaluator, Fr, Thunk, Closure, OpVal, AssertFailure, BuiltinOp
from ..front.values import (EvalError, ModelValue, Fcn, LazySet, LazyFcn, SetNat, SetInt, mk_fcn, sorted_vals,
                            set_contains, set_iter, to_finite, is_set, is_enumerable, fmt, vkey, fcn_items)
from .types import (T, TInt, TBool, TAtom, TRec, TTuple, TFun, TSet, TSeq, TPFun, TSparse, TBottom, TypeErr, Atoms,
                    Codec, join, type_of_value, type_of_set, widen_init, is_atom, subset_type, has_dynamic)
from . import types as _types
from .types import ATOM_ALT
from .bytecode import (Asm, Label, TRAP_EVAL, TRAP_OVERFLOW, TRAP_CASE, TRAP_CHOOSE, IMM28_MAX, IMM28_MIN, MAXREG)

UNROLL_MAX = 24
UNIV_TABLE_MAX = 1 << 16


class CompileError(Exception):
    pass


class CompileBudget(CompileError):
    """Inline expansion exceeded its budget: the caller retries with operator subroutines."""


class Const:
    __slots__ = ("v",)

    def __init__(self, v):
        self.v = v

    def __repr__(self):
        return f"Const({fmt(self.v)})"


class Val:
    __slots__ = ("t", "loc")

    def __init__(self, t, loc):
        self.t = t
        self.loc = loc

    def __repr__(self):
        return f"Val({self.t}@{self.loc})"


class MVal(Val):
    """A set value known to be a subset of a compile-time mask (`alive` = admissible ordinals)."""
    __slots__ = ("alive",)

    def __init__(self, t, loc, alive):
        self.t, self.loc, self.alive = t, loc, alive


class OVal(Val):
    """Element of an enumerable composite type known only by its ordinal (loop variable over a
    bitset universe).  Fields are decoded on demand with one table lookup each; touching `.loc`
    materialises the whole value (fresh temporaries every time, so it is valid on any path)."""
    __slots__ = ("lw", "oreg", "alive")

    def __init__(self, lw, t, oreg, alive=None):
        self.lw = lw
        self.t = t
        self.oreg = oreg
        self.alive = alive

    @property
    def loc(self):
        return self.lw.unord(self.t, self.oreg).loc

    def __repr__(self):
        return f"OVal({self.t}#{self.oreg})"


class PVal(Val):
    """A call-by-name binding (operator argument / LET definition) that was evaluated ONCE at its binding
    site because it is referenced several times and yields a large value (raft.tla:117-147: the message bag
    flows through WithMessage / WithoutMessage by name).  Lazy semantics are kept: a trap raised while
    computing it only sets `poison`, and is re-raised where the value is used."""
    __slots__ = ("poison", "lazy")

    def __init__(self, t, loc, poison, lazy):
        self.t, self.loc, self.poison, self.lazy = t, loc, poison, lazy


class Lazy:
    __slots__ = ("node", "env", "ctx", "base")

    def __init__(self, node, env, ctx, base):
        self.node, self.env, self.ctx, self.base = node, env, ctx, base


class OpC:
    """Operator value at compile time (definition with parameters, LET operator, LAMBDA)."""
    __slots__ = ("params", "body", "env", "ctx", "name")

    def __init__(self, params, body, env, ctx, name):
        self.params, self.body, self.env, self.ctx, self.name = params, body, env, ctx, name


_RUNTIME_NODE = Node("runtime", ())


class CompiledModel:
    """Everything the engine needs + what the host needs to decode states."""

    def __init__(self):
        self.code = None
        self.cpool = None
        self.entries = {}
        self.W = 0
        self.frame_words = 0
        self.layout = None       # np.int32 [nslots,3]: frame_off, width, bias
        self.n_off = 0
        self.p_off = 0
        self.state_words_unpacked = 0
        self.var_types = {}
        self.var_off = {}
        self.vars = []
        self.actions = []        # id -> (name, loc, module)
        self.invariants = []     # names
        self.asserts = []        # id -> message
        self.atoms = None
        self.codec = None
        self.group = []          # SYMMETRY group (non-identity permutations of model values)
        self.warnings = []


class Lowering:
    def __init__(self, model, seq_cap=None, type_hint=None):
        self.m = model
        self.ev = model.ev
        self.ev.disp["runtime"] = self._runtime_node
        self.ctx = model.ctx
        self.asm = Asm()
        self.atoms = Atoms()
        self.codec = Codec(self.atoms)
        self.seq_cap = seq_cap
        self.type_hint = type_hint
        self.top = 0
        self.high = 0
        self.bound = frozenset()
        self.actions = []
        self.asserts = []
        self.warnings = []
        self._evenv_cache = {}
        self.hoisted = {}
        self.def_uses = {}
        self.def_info = {}
        self.program = "inv"
        self.hoist_keys = []
        self.dry = False
        self._seg_top, self._seg_buf, self._seg_clean, self._seg_last = False, None, -1, -1
        self.seg_cuts = {"inv": [], "next": []}
        self.blocks = set()
        self.group = model.symmetry_group() if hasattr(model, "symmetry_group") else []
        self._rec_depth = {}
        self.use_subs = False          # compile module-level operators as CALL/RET subroutines instead of inlining
        self.subs = {}
        self.sub_bufs = []
        self.sub_base0 = MAXREG // 2   # discovery pass: every subroutine frame starts here (only sizes matter)
        self.sub_plan = None           # final pass: key -> base of the subroutine's static frame
        self.sub_calls = {}            # caller key (None = main programs) -> set of callee keys
        self._sub_stack = []
        self._sub_active = set()
        self._cx_count = 0
        self.cx_budget = self.CX_BUDGET
        self.copy_once = False
        self.rec_depth = 6
        self._intern_all_atoms()
        # unrolling depth of RECURSIVE operators: recursions in the bundled specs walk a set of model values (a path of
        # transactions, visited nodes), so |largest constant set| + 2 levels suffice; deeper activations trap
        big = max([len(v) for c in [self.ctx] + self.ctx.all_instances for v in c.consts.values()
                   if isinstance(v, frozenset)] + [1])
        self.rec_depth = min(6, max(3, big + 2))

    @staticmethod
    def _runtime_node(n, env, fr):
        raise EvalError("runtime value")

    # ------------------------------------------------------------------ atoms
    def _intern_all_atoms(self):
        strs = set()
        mvs = set()

        def walk(n):
            if isinstance(n, Node):
                if n.k == "str":
                    strs.add(n.a[0])
                for x in n.a:
                    walk(x)
            elif isinstance(n, (tuple, list)):
                for x in n:
                    walk(x)
            elif isinstance(n, OpDef):
                walk(n.body)

        def walkv(v):
            if isinstance(v, ModelValue):
                mvs.add(v)
            elif isinstance(v, str):
                strs.add(v)
            elif isinstance(v, (frozenset, tuple)):
                for x in v:
                    walkv(x)
            elif isinstance(v, Fcn):
                for k, x in v.d.items():
                    walkv(k)
                    walkv(x)

        for name in self.m.loader.cache:
            mod = self.m.loader.cache[name]
            for d in mod.defs.values():
                walk(d.body)
            for _, e in mod.assumes:
                walk(e)
        for c in [self.ctx] + self.ctx.all_instances:
            for v in c.consts.values():
                walkv(v)
        for s in sorted(strs):
            self.atoms.id(s)
        for mv in sorted(mvs, key=lambda x: x.name):
            self.atoms.id(mv)
        self.all_strings = sorted(strs)
        self.all_mvs = sorted(mvs, key=lambda x: x.name)

    # ------------------------------------------------------------- allocation
    def alloc(self, n):
        loc = self.top
        self.top += max(n, 0)
        if n > 1:
            self.blocks.add((loc, n))       # extents for the scalar form of the sliced build (compile/sliced.py)
        if self.top > self.high:
            self.high = self.top
        if self.high > MAXREG and not self.dry:
            raise CompileError("frame exceeds 16K words")
        return loc

    def mark(self):
        return self.top

    def release(self, m):
        self.top = m

    # ------------------------------------------------------------- var types
    def _auto_seq_cap(self, init_states):
        """No -seqcap given: capacity of Seq(S)-typed variables = longest sequence in a bounded sample of reachable
        states + 2, at least 4.  Longer sequences trap at run time (capacity overflow), they are never truncated."""
        def longest(v):
            if isinstance(v, tuple):
                return max([len(v)] + [longest(x) for x in v])
            if isinstance(v, frozenset):
                return max([0] + [longest(x) for x in v])
            if isinstance(v, Fcn):
                return max([0] + [longest(x) for x in v.d.values()])
            return 0
        n = 0
        for st in self._sample_reachable(init_states):
            for v in self.m.vars:
                n = max(n, longest(st[v]))
        self.seq_cap = max(4, n + 2)
        self.warnings.append(f"sequence capacity set to {self.seq_cap} (from a sample of reachable states; "
                             f"override with -seqcap)")

    def infer_var_types(self, init_states):
        m = self.m
        if self.seq_cap is None:
            def mentions_seq(x):
                if isinstance(x, Node):
                    return (x.k == "app" and x.a[0] == "Seq") or any(mentions_seq(y) for y in x.a)
                if isinstance(x, (tuple, list)):
                    return any(mentions_seq(y) for y in x)
                return isinstance(x, OpDef) and mentions_seq(x.body)
            if any(mentions_seq(d[0].body) for d in self.ctx.defs.values()):
                self._auto_seq_cap(init_states)
        types = {}
        hint = self.type_hint
        # candidate type invariants: an explicit hint, the cfg's INVARIANTs, then every definition whose
        # name looks like one (TypeOK, TypeInv, ABTypeInv, TypeInvariant, ITypeOK ...)
        cand = [hint] if hint else []
        if not hint:
            cand += [nm for nm, _, _ in m.invariants]
            named = [n for n in self.ctx.defs if re.search(r"Type(OK|Inv|Invariant|Correct)", n)]
            named.sort(key=lambda n: (n.startswith("I"), len(n), n))
            cand += [n for n in named if n not in cand]

        quiet = False

        def harvest(node, ctx, got, depth=0):
            """collect  v \\in S / v \\subseteq S  conjuncts, following nested conjunctions and definitions"""
            nonlocal quiet
            if depth > 6:
                return
            if node.k == "and":
                for x in node.a[0]:
                    harvest(x, ctx, got, depth)
                return
            isvar = lambda x: x.k == "id" and x.a[0] in ctx.varset and x.a[0] not in ctx.substs
            if node.k == "bin" and node.a[0] in ("\\in", "\\subseteq") and isvar(node.a[1]):
                v = node.a[1].a[0]
                try:
                    sv = self.ev.eval(node.a[2], {}, Fr(ctx))
                    et = type_of_set(sv, self.seq_cap)
                    got.setdefault(v, subset_type(et) if node.a[0] == "\\subseteq" else et)
                except (EvalError, TypeErr) as ex:
                    if quiet is False:
                        self.warnings.append(f"type hint: cannot use conjunct for {v}: {ex}")
                return
            # function with a dynamic domain (raft.tla:35 `messages`):  DOMAIN v \subseteq K  /\
            # \A x \in DOMAIN v : v[x] \in R   [/\ Cardinality(DOMAIN v) <= n]
            if node.k == "bin" and node.a[0] == "\\subseteq" and node.a[1].k == "domain" and isvar(node.a[1].a[0]):
                v = node.a[1].a[0].a[0]
                try:
                    dyn.setdefault(v, {})["k"] = type_of_set(self.ev.eval(node.a[2], {}, Fr(ctx)), self.seq_cap)
                except (EvalError, TypeErr) as ex:
                    self.warnings.append(f"type hint: cannot use conjunct for DOMAIN {v}: {ex}")
                return
            if node.k == "forall" and len(node.a[0]) == 1 and isinstance(node.a[0][0][0], str) \
                    and node.a[0][0][1] is not None and node.a[0][0][1].k == "domain" and isvar(node.a[0][0][1].a[0]):
                v = node.a[0][0][1].a[0].a[0]
                b = node.a[1]
                if b.k == "bin" and b.a[0] == "\\in" and b.a[1].k == "fapp" and b.a[1].a[0].k == "id" \
                        and b.a[1].a[0].a[0] == v:
                    try:
                        dyn.setdefault(v, {})["v"] = type_of_set(self.ev.eval(b.a[2], {}, Fr(ctx)), self.seq_cap)
                    except (EvalError, TypeErr) as ex:
                        self.warnings.append(f"type hint: cannot use conjunct for {v}[..]: {ex}")
                return
            if node.k == "bin" and node.a[0] in ("<=", "=<", "\\leq", "<") and node.a[1].k == "app" \
                    and node.a[1].a[0] == "Cardinality":
                arg = node.a[1].a[1][0]
                if arg.k == "domain":
                    arg = arg.a[0]
                if isvar(arg):
                    try:
                        n_ = self.ev.eval(node.a[2], {}, Fr(ctx))
                        caps.setdefault(arg.a[0], n_ - 1 if node.a[0] == "<" else n_)
                    except EvalError:
                        pass
                return
            if node.k == "id":
                d2 = ctx.defs.get(node.a[0])
                if d2 is not None and not d2[0].params and node.a[0] not in ctx.varset:
                    harvest(d2[0].body, d2[1], got, depth + 1)
                return
            if node.k == "sel":
                try:
                    r = self.ev.resolve_sel(node.a[0], {}, Fr(ctx))
                except EvalError:
                    return
                if r[0] == "def" and not r[1].params:
                    # variables of an instance are substituted: only root-module variables are typed here
                    harvest(r[1].body, r[2], got, depth + 1)

        dyn, caps = {}, {}
        for name in cand:
            d = self.ctx.defs.get(name)
            if d is None or d[0].params:
                continue
            # ordinary invariants are scanned too, but only a definition that looks like a type invariant is
            # worth a warning when one of its conjuncts cannot be used
            quiet = not (name == hint or re.search(r"Type(OK|Inv|Invariant|Correct)", name))
            got = {}
            harvest(d[0].body, d[1], got)
            for v, di in dyn.items():
                if "k" in di and "v" in di:
                    got.setdefault(v, TSparse(di["k"], di["v"], _types.SPARSE_CAP))
            for v, t in got.items():
                if isinstance(t, TSparse) and v in caps:
                    t = TSparse(t.kt, t.vt, int(caps[v]))
                if v in m.vars:
                    types.setdefault(v, t)
            if all(v in types for v in m.vars):
                break
        all_atoms = [self.atoms.val(i) for i in range(1, len(self.atoms.vals))]
        str_atoms = [a for a in all_atoms if isinstance(a, str)]
        mv_atoms = [a for a in all_atoms if isinstance(a, ModelValue)]
        untyped = [v for v in m.vars if v not in types]
        sample = self._sample_reachable(init_states) if untyped else init_states
        for v in untyped:
            t = None
            for st in sample:
                try:
                    t = join(t, type_of_value(st[v], self.seq_cap))
                except TypeErr as ex:
                    raise CompileError(f"cannot infer a fixed-width type for variable {v}: {ex}; add a TypeOK-style "
                                       f"definition")
            if t is None:
                raise CompileError(f"cannot infer a type for variable {v}: no initial states")
            types[v] = self._widen(t, str_atoms, mv_atoms, all_atoms)
        # initial states must inhabit the types
        for v in m.vars:
            for st in init_states[:64]:
                try:
                    self.codec.rep(types[v], st[v])
                except TypeErr as ex:
                    raise CompileError(f"initial value of {v} does not fit its type {types[v]}: {ex}")
        return types

    SAMPLE_STATES = 400
    SAMPLE_SECONDS = 8.0

    def _sample_reachable(self, init_states):
        """Shapes for variables that no type invariant mentions (MemoryInterface.tla:2 `memInt`): the host front end
        enumerates a bounded prefix of the reachable states (initial states and a few hundred successors) and the
        types are the widened join of what it sees.  This is compile-time typing only -- the search itself runs on
        the device, and a value outside the inferred type traps there (capacity overflow), it is never wrong."""
        m = self.m
        seen, out, queue = set(), [], []
        key = lambda st: tuple(repr(st[v]) for v in m.vars)
        for st in init_states:
            k = key(st)
            if k not in seen:
                seen.add(k)
                out.append(st)
                queue.append(st)
        # bounded in time as well: one successor of some specs costs the host evaluator minutes
        # (AdvancedExamples/InnerSerial.tla enumerates sets of orderings)
        import signal
        import threading

        class _Budget(Exception):
            pass

        def _expired(*_a):
            raise _Budget()
        use_alarm = threading.current_thread() is threading.main_thread() and hasattr(signal, "setitimer")
        old = None
        if use_alarm:
            old = signal.signal(signal.SIGALRM, _expired)
            signal.setitimer(signal.ITIMER_REAL, self.SAMPLE_SECONDS)
        qi = 0
        try:
            while qi < len(queue) and len(out) < self.SAMPLE_STATES:
                st = queue[qi]
                qi += 1
                try:
                    for asg, _act in self.ev.solve(m.next_node, {}, m.next_ctx, st, {}, "next"):
                        if len(asg) != len(m.vars):
                            continue
                        k = key(asg)
                        if k not in seen:
                            seen.add(k)
                            out.append(asg)
                            queue.append(asg)
                            if len(out) >= self.SAMPLE_STATES:
                                break
                except (EvalError, AssertFailure, RecursionError):
                    continue
        except _Budget:
            self.warnings.append(f"type sampling stopped after {self.SAMPLE_SECONDS}s ({len(out)} states)")
        finally:
            if use_alarm:
                signal.setitimer(signal.ITIMER_REAL, 0)
                signal.signal(signal.SIGALRM, old)
        return out

    def _widen(self, t, strs, mvs, alla):
        if isinstance(t, TAtom):
            has_s = any(isinstance(a, str) for a in t.atoms)
            has_m = any(isinstance(a, ModelValue) for a in t.atoms)
            pool = alla if (has_s and has_m) else (strs if has_s else mvs)
            return TAtom(sorted(pool, key=vkey))
        if isinstance(t, TInt):
            return TInt()
        if isinstance(t, TTuple):
            return TTuple([self._widen(e, strs, mvs, alla) for e in t.elems])
        if isinstance(t, TFun):
            return TFun(t.keys, self._widen(t.elem, strs, mvs, alla))
        if isinstance(t, TRec):
            return TRec([{f: self._widen(x, strs, mvs, alla) for f, x in d.items()} for d in t.alt_dicts()])
        if isinstance(t, TSet):
            if isinstance(t.elem, TBottom):
                raise CompileError("cannot infer the element type of an initially-empty set variable; "
                                   "add a TypeOK-style definition (v \\in S / v \\subseteq S conjuncts)")
            e = t.elem
            if isinstance(e, TInt):
                return t
            return TSet(self._widen(e, strs, mvs, alla))
        return t

    # ------------------------------------------------------------ const eval
    def eval_env(self, env):
        key = id(env)
        hit = self._evenv_cache.get(key)
        if hit is not None and hit[0] is env:
            return hit[1]
        out = {}
        self._evenv_cache[key] = (env, out)   # registered first: LET environments are self-referential
        for k, v in env.items():
            if type(v) is Const:
                out[k] = v.v
            elif isinstance(v, Val):
                out[k] = Thunk(_RUNTIME_NODE, {}, None)
            elif type(v) is Lazy:
                if v.base != "N":
                    out[k] = Thunk(_RUNTIME_NODE, {}, None)
                else:
                    out[k] = Thunk(v.node, self.eval_env(v.env), v.ctx)
            elif type(v) is OpC:
                out[k] = Closure([p for p, _ in v.params], v.body, self.eval_env(v.env), v.ctx, v.name)
        self._evenv_cache[key] = (env, out)
        return out

    def try_const(self, node, env, ctx, base):
        if base != "N" and node.k not in ("num", "str", "bool"):
            # primed context: only literals are constant for sure; still try (constants don't read state)
            pass
        try:
            v = self.ev.eval(node, self.eval_env(env), Fr(ctx, None, None))
            if isinstance(v, LazyFcn):
                v = v.force()
        except (EvalError, AssertFailure, RecursionError, TypeErr, TypeError, KeyError, AttributeError,
                ValueError, IndexError):
            return None
        if isinstance(v, (OpVal, Closure, BuiltinOp)):
            return None
        return Const(v)

    # ------------------------------------------------------- materialisation
    def materialize(self, c: Const, t: T) -> Val:
        try:
            words = self.codec.rep(t, c.v)
        except TypeErr as ex:
            raise CompileError(f"constant {fmt(c.v)} does not fit type {t}: {ex}")
        loc = self.alloc(t.size)
        self.load_words(loc, words)
        return Val(t, loc)

    def load_words(self, loc, words):
        if len(words) <= 2:
            for i, w in enumerate(words):
                self.li(loc + i, w)
        elif all(w == 0 for w in words):
            self.asm.emit("ZERO", loc, len(words))
        else:
            base = self.asm.const_table(words)
            i = 0
            while i < len(words):
                n = min(len(words) - i, MAXREG)
                self.asm.emit("LDC", loc + i, base + i, n)
                i += n

    def li(self, loc, w):
        w = int(w)
        if IMM28_MIN <= w <= IMM28_MAX:
            self.asm.emit("LI", loc, w)
        else:
            self.asm.emit("LIW", loc, self.asm.const_table([w]))

    def natural_type(self, v) -> T:
        t = type_of_value(v, self.seq_cap)
        return t

    def as_val(self, x, want=None) -> Val:
        if isinstance(x, Val):
            return x
        t = want if want is not None else self.natural_type(x.v)
        if want is None and isinstance(t, TSet) and isinstance(t.elem, TBottom):
            raise CompileError("cannot type the empty set here (no expected type)")
        return self.materialize(x, t)

    # ------------------------------------------------------------- coercion
    def coerce(self, x, t: T) -> Val:
        if type(x) is Const:
            return self.materialize(x, t)
        s = x.t
        if s == t:
            return x
        if isinstance(s, TBottom):          # value of an activation past the recursion bound (already trapped)
            dst = self.alloc(t.size)
            self.asm.emit("ZERO", dst, t.size)
            return Val(t, dst)
        if isinstance(t, TInt) and isinstance(s, TInt):
            return Val(t, x.loc)
        if isinstance(t, TAtom) and isinstance(s, TAtom):
            return Val(t, x.loc)
        if isinstance(t, TBool) and isinstance(s, TBool):
            return x
        if isinstance(t, TRec) and isinstance(s, TAtom) and ATOM_ALT in t.fields:
            dst = self.alloc(t.size)
            self.asm.emit("ZERO", dst, t.size)
            if t.tagged:
                self.li(dst, t.alt_index((ATOM_ALT,)))
            self.asm.emit("MOV", dst + t.off[ATOM_ALT], x.loc)
            return Val(t, dst)
        if isinstance(t, TRec) and isinstance(s, TRec):
            dst = self.alloc(t.size)
            self.asm.emit("ZERO", dst, t.size)
            if s.tagged:
                # map tags through a table; an alternative the target type does not have is a run-time narrowing
                # failure (trap), e.g. buf[p] : MReq | Val | NoVal appended to a queue of requests
                # (WriteThroughCache.tla:112) after the guard r.op = "Wr" has established that it is a request
                tbl = []
                for alt in s.alts:
                    ai = t.alt_index(alt)
                    tbl.append(ai if ai >= 0 else -(1 << 31))
                if all(i < 0 for i in tbl):
                    raise CompileError(f"no record alternative of {s} fits {t}")
                tagr = self.alloc(1)
                self.asm.emit("TBLT" if any(i < 0 for i in tbl) else "TBL", tagr, self.asm.const_table(tbl), x.loc)
                if t.tagged:
                    self.asm.emit("MOV", dst, tagr)
            else:
                ai = t.alt_index(s.alts[0])
                if ai < 0:
                    raise CompileError(f"record with fields {s.alts[0]} does not fit {t}")
                if t.tagged:
                    self.li(dst, ai)
            for f in s.fnames:
                if f not in t.fields:
                    if s.tagged:
                        continue            # only in alternatives the target lacks (those trapped above)
                    raise CompileError(f"field {f} missing in target record type")
                sub = self.coerce(Val(s.fields[f], x.loc + s.off[f]), t.fields[f])
                self.movn(dst + t.off[f], sub.loc, t.fields[f].size)
            return Val(t, dst)
        if isinstance(t, TTuple) and isinstance(s, TTuple) and len(t.elems) == len(s.elems):
            dst = self.alloc(t.size)
            for te, se, to, so in zip(t.elems, s.elems, t.offs, s.offs):
                sub = self.coerce(Val(se, x.loc + so), te)
                self.movn(dst + to, sub.loc, te.size)
            return Val(t, dst)
        if isinstance(t, TFun) and isinstance(s, TFun) and t.keys == s.keys:
            dst = self.alloc(t.size)
            for j in range(len(t.keys)):
                sub = self.coerce(Val(s.elem, x.loc + j * s.elem.size), t.elem)
                self.movn(dst + j * t.elem.size, sub.loc, t.elem.size)
            return Val(t, dst)
        if isinstance(t, TFun) and isinstance(s, TTuple) and t.keys == tuple(range(1, len(s.elems) + 1)):
            dst = self.alloc(t.size)
            for j in range(len(t.keys)):
                sub = self.coerce(Val(s.elems[j], x.loc + s.offs[j]), t.elem)
                self.movn(dst + j * t.elem.size, sub.loc, t.elem.size)
            return Val(t, dst)
        if isinstance(t, TSet) and isinstance(s, TSet):
            if isinstance(s.elem, TBottom):
                dst = self.alloc(t.size)
                self.asm.emit("ZERO", dst, t.size)
                return Val(t, dst)
            if self._same_universe_prefix(s.elem, t.elem):
                dst = self.alloc(t.size)
                self.asm.emit("ZERO", dst, t.size)
                self.movn(dst, x.loc, s.size)
                return Val(t, dst)
            # re-index element by element
            dst = self.alloc(t.size)
            self.asm.emit("ZERO", dst, t.size)

            def body(ev):
                o = self.ord_in(t.elem, ev)
                bad = Label("ovf")
                ok = Label("ok")
                self.asm.emit("JNEG", o, bad)
                self.asm.emit("BSET", dst, o)
                self.asm.emit("JMP", ok)
                self.asm.label(bad)
                self.asm.emit("TRAP", TRAP_OVERFLOW, 0)
                self.asm.label(ok)
            self.loop_set(x, body)
            return Val(t, dst)
        if isinstance(t, TSeq) and isinstance(s, TTuple):
            if len(s.elems) > t.cap:
                raise CompileError("tuple longer than sequence capacity")
            dst = self.alloc(t.size)
            self.asm.emit("ZERO", dst, t.size)
            self.li(dst, len(s.elems))
            for j, (se, so) in enumerate(zip(s.elems, s.offs)):
                sub = self.coerce(Val(se, x.loc + so), t.elem)
                self.movn(dst + 1 + j * t.elem.size, sub.loc, t.elem.size)
            return Val(t, dst)
        if isinstance(t, TSeq) and isinstance(s, TSeq) and t.elem == s.elem and s.cap <= t.cap:
            dst = self.alloc(t.size)
            self.asm.emit("ZERO", dst, t.size)
            self.movn(dst, x.loc, s.size)
            return Val(t, dst)
        if isinstance(t, TSeq) and isinstance(s, TSeq):
            # different capacity / element type: element-wise, trapping when the length does not fit
            dst = self.alloc(t.size)
            self.asm.emit("ZERO", dst, t.size)
            self.asm.emit("MOV", dst, x.loc)
            done = Label("sqd")
            if s.cap > t.cap:
                ok = Label("sqk")
                t1 = self.alloc(1)
                self.asm.emit("LEI", t1, x.loc, t.cap)
                self.asm.emit("JNZ", t1, ok)
                self.asm.emit("TRAP", TRAP_OVERFLOW, 0)
                self.asm.label(ok)
            for j in range(min(s.cap, t.cap)):
                t2 = self.alloc(1)
                self.asm.emit("LEI", t2, x.loc, j)
                self.asm.emit("JNZ", t2, done)
                sub = self.coerce(Val(s.elem, x.loc + 1 + j * s.elem.size), t.elem)
                self.movn(dst + 1 + j * t.elem.size, sub.loc, t.elem.size)
            self.asm.label(done)
            return Val(t, dst)
        if isinstance(t, TPFun) and isinstance(s, TPFun) and t.keys == s.keys:
            dst = self.alloc(t.size)
            self.asm.emit("ZERO", dst, t.size)
            for j in range(len(t.keys)):
                skip = Label("pfc")
                self.asm.emit("JZ", x.loc + j * s.stride, skip)
                self.li(dst + j * t.stride, 1)
                sub = self.coerce(Val(s.elem, x.loc + j * s.stride + 1), t.elem)
                self.movn(dst + j * t.stride + 1, sub.loc, t.elem.size)
                self.asm.label(skip)
            return Val(t, dst)
        if isinstance(t, TSparse) and isinstance(s, TSparse) and (t.vt is None) == (s.vt is None):
            if t.kt == s.kt and t.vt == s.vt and s.cap <= t.cap:
                dst = self.alloc(t.size)
                self.asm.emit("ZERO", dst, t.size)
                self.movn(dst, x.loc, s.size)
                return Val(t, dst)
            out = self.sp_new(t)
            self.sp_loop(x, lambda k, v: self.sp_insert(out, self.sp_entry(t, k, v)))
            return out
        if isinstance(t, TSparse) and t.vt is None and isinstance(s, TSet):
            out = self.sp_new(t)
            if not isinstance(s.elem, TBottom):
                self.loop_set(x, lambda ev: self.sp_insert(out, self.sp_entry(t, ev)))
            return out
        raise CompileError(f"cannot coerce {s} to {t}")

    @staticmethod
    def _same_universe_prefix(a: T, b: T):
        """True if enumeration of a is a prefix-compatible renumbering-free subset of b (same ordinals)."""
        if a == b:
            return True
        if isinstance(a, TInt) and isinstance(b, TInt) and a.lo is not None and b.lo is not None:
            return a.lo == b.lo and a.hi <= b.hi
        if isinstance(a, TAtom) and isinstance(b, TAtom):
            return b.atoms[:len(a.atoms)] == a.atoms
        return False

    def movn(self, dst, src, n):
        if dst == src or n == 0:
            return
        if n == 1:
            self.asm.emit("MOV", dst, src)
        else:
            self.asm.emit("MOVN", dst, src, n)

    # --------------------------------------------------------------- ordinals
    def ord_can_fail(self, E: T, v) -> bool:
        """Static check: can the ordinal of v in E come out as -1 (value outside the universe)?"""
        if type(v) is Const:
            return self.codec.ord_of(E, v.v) < 0
        if type(v) is OVal and v.t == E:
            return False
        s = v.t
        if isinstance(E, TInt):
            return not (isinstance(s, TInt) and s.lo is not None and E.lo is not None and E.lo <= s.lo and s.hi <= E.hi)
        if isinstance(E, TBool):
            return not isinstance(s, TBool)
        if isinstance(E, TAtom):
            return not (isinstance(s, TAtom) and set(s.atoms) <= set(E.atoms))
        if isinstance(E, TRec):
            if not isinstance(s, TRec):
                return True
            for alt in s.alts:
                ai = E.alt_index(alt)
                if ai < 0:
                    return True
                for f in alt:
                    if self.ord_can_fail(E.alt_types[ai][f], Val(s.fields[f], 0)):
                        return True
            return False
        if isinstance(E, TTuple):
            if not (isinstance(s, TTuple) and len(s.elems) == len(E.elems)):
                return True
            return any(self.ord_can_fail(ee, Val(se, 0)) for ee, se in zip(E.elems, s.elems))
        if isinstance(E, TSet):
            return not isinstance(s, TSet)
        if isinstance(E, TFun):
            if not (isinstance(s, TFun) and s.keys == E.keys):
                return True
            return self.ord_can_fail(E.elem, Val(s.elem, 0))
        return True

    def horner(self, r, card, o):
        """r = r * card + o  (one fused instruction when the radix fits the 14-bit immediate)."""
        if 0 < card < (1 << 13):
            self.asm.emit("MADI", r, card, o)
        else:
            self.asm.emit("MULI", r, r, card)
            self.asm.emit("ADD", r, r, o)

    def ord_in(self, E: T, v) -> int:
        """Emit code computing the ordinal of v within E (or -1 when outside); returns the reg."""
        if type(v) is Const:
            o = self.codec.ord_of(E, v.v)
            r = self.alloc(1)
            if isinstance(E, TSet):
                self.li(r, o if o < (1 << 31) else o - (1 << 32))
            else:
                self.li(r, o)
            return r
        if type(v) is OVal and v.t == E:
            return v.oreg
        s = v.t
        r = self.alloc(1)
        if isinstance(E, TInt):
            if not isinstance(s, TInt):
                self.li(r, -1)
                return r
            if E.lo is None:
                raise CompileError("ordinal of an unbounded integer type")
            fail = self.ord_can_fail(E, v)
            if E.lo == 0 and not fail:
                return v.loc              # the value is its own ordinal
            if E.lo != 0:
                self.asm.emit("ADDI", r, v.loc, -E.lo)
            else:
                self.asm.emit("MOV", r, v.loc)
            if fail:
                self.asm.emit("UCLAMP", r, E.card())
            return r
        if isinstance(E, TBool):
            if not isinstance(s, TBool):
                self.li(r, -1)
                return r
            return v.loc
        if isinstance(E, TAtom):
            if not isinstance(s, TAtom):
                self.li(r, -1)
                return r
            tbl = [-1] * len(self.atoms.vals)
            for i, a in enumerate(E.atoms):
                tbl[self.atoms.id(a)] = i
            self.asm.emit("TBL", r, self.asm.const_table(tbl), v.loc)
            return r
        if isinstance(E, TRec):
            if not isinstance(s, TRec):
                self.li(r, -1)
                return r
            bad = Label("obad")
            end = Label("oend")
            if not s.tagged:
                self._ord_rec_alt(E, s, s.alts[0], v, r, bad)
                self.asm.emit("JMP", end)
            else:
                for j, alt in enumerate(s.alts):
                    nxt = Label("oalt")
                    t1 = self.alloc(1)
                    self.asm.emit("EQI", t1, v.loc, j)
                    self.asm.emit("JZ", t1, nxt)
                    self._ord_rec_alt(E, s, alt, v, r, bad)
                    self.asm.emit("JMP", end)
                    self.asm.label(nxt)
            self.asm.label(bad)
            self.li(r, -1)
            self.asm.label(end)
            return r
        if isinstance(E, TTuple):
            if not (isinstance(s, TTuple) and len(s.elems) == len(E.elems)):
                self.li(r, -1)
                return r
            bad = Label("obad")
            end = Label("oend")
            self.li(r, 0)
            for ee, se, so in zip(E.elems, s.elems, s.offs):
                sub = Val(se, v.loc + so)
                o = self.ord_in(ee, sub)
                if self.ord_can_fail(ee, sub):
                    self.asm.emit("JNEG", o, bad)
                self.horner(r, ee.card(), o)
            self.asm.emit("JMP", end)
            self.asm.label(bad)
            self.li(r, -1)
            self.asm.label(end)
            return r
        if isinstance(E, TSet):
            if not isinstance(s, TSet):
                self.li(r, -1)
                return r
            if E.nbits > 31:
                raise CompileError("set-of-sets universe too large")
            cv = self.coerce(v, E)
            self.asm.emit("MOV", r, cv.loc)
            return r
        if isinstance(E, TFun):
            if not (isinstance(s, TFun) and s.keys == E.keys):
                self.li(r, -1)
                return r
            bad = Label("obad")
            end = Label("oend")
            self.li(r, 0)
            for j in range(len(E.keys)):
                sub = Val(s.elem, v.loc + j * s.elem.size)
                o = self.ord_in(E.elem, sub)
                if self.ord_can_fail(E.elem, sub):
                    self.asm.emit("JNEG", o, bad)
                self.horner(r, E.elem.card(), o)
            self.asm.emit("JMP", end)
            self.asm.label(bad)
            self.li(r, -1)
            self.asm.label(end)
            return r
        raise CompileError(f"ord_in: unsupported universe type {E}")

    def _ord_rec_alt(self, E: TRec, s: TRec, alt, v: Val, r, bad):
        ai = E.alt_index(alt)
        if ai < 0:
            self.asm.emit("JMP", bad)
            return
        self.li(r, 0)
        for f in E.alts[ai]:
            ft = E.alt_types[ai][f]
            sub = Val(s.fields[f], v.loc + s.off[f])
            o = self.ord_in(ft, sub)
            if self.ord_can_fail(ft, sub):
                self.asm.emit("JNEG", o, bad)
            self.horner(r, ft.card(), o)
        base = E.alt_base(ai)
        if base:
            self.asm.emit("ADDI", r, r, base)

    def unord(self, E: T, oreg, dst=None) -> Val:
        """Decode ordinal in oreg to a frame value of type E."""
        if dst is None:
            dst = self.alloc(E.size)
        if isinstance(E, TInt):
            self.asm.emit("ADDI", dst, oreg, E.lo)
            return Val(E, dst)
        if isinstance(E, TBool):
            self.asm.emit("MOV", dst, oreg)
            return Val(E, dst)
        if isinstance(E, TAtom):
            self.asm.emit("TBL", dst, self.asm.const_table([self.atoms.id(a) for a in E.atoms]), oreg)
            return Val(E, dst)
        if isinstance(E, TSet) and E.nbits <= 31:
            self.asm.emit("MOV", dst, oreg)
            return Val(E, dst)
        n = E.card()
        if n > UNIV_TABLE_MAX:
            raise CompileError(f"universe of {n} elements too large for table decoding")
        key = ("univ", E)
        tabs = self._univ_tables(E)
        for w in range(E.size):
            self.asm.emit("TBL", dst + w, tabs[w], oreg)
        return Val(E, dst)

    def _field_tables(self, E: TRec, f):
        """Per-word column tables of field f over the enumeration of E; ordinals whose alternative
        lacks f hold INT32_MIN in word 0 (TBLT traps on it, like TLC's missing-field error)."""
        cache = self.__dict__.setdefault("_field_cache", {})
        key = (E, f)
        if key in cache:
            return cache[key]
        vals = self.codec.enum(E)
        ft = E.fields[f]
        cols = [[] for _ in range(ft.size)]
        for v in vals:
            d = v.d if isinstance(v, Fcn) else {ATOM_ALT: v}       # bare atom of an atom | record union
            if f in d:
                r = self.codec.rep(ft, d[f])
            else:
                r = [-(1 << 31)] + [0] * (ft.size - 1)
            for w in range(ft.size):
                cols[w].append(r[w])
        tabs = [self.asm.const_table(c) for c in cols]
        cache[key] = tabs
        return tabs

    def _univ_tables(self, E):
        cache = self.__dict__.setdefault("_univ_cache", {})
        if E in cache:
            return cache[E]
        vals = self.codec.enum(E)
        reps = [self.codec.rep(E, v) for v in vals]
        tabs = []
        for w in range(E.size):
            tabs.append(self.asm.const_table([r[w] for r in reps]))
        cache[E] = tabs
        return tabs

    # ------------------------------------------------------------------ loops
    def loop_set(self, sv: Val, body, elem_dst=None):
        """for x in (runtime bitset sv): body(Val elem).  body may emit jumps to its own labels."""
        E = sv.t.elem
        if isinstance(E, TBottom):
            return
        idx = self.alloc(1)
        lazy = elem_dst is None and isinstance(E, (TRec, TTuple)) and E.card() <= UNIV_TABLE_MAX
        xloc = None if lazy else (self.alloc(E.size) if elem_dst is None else elem_dst)
        self.li(idx, -1)
        top = Label("loop")
        done = Label("done")
        self.asm.label(top)
        self.asm.emit("BNEXT", idx, sv.loc, idx, sv.t.nbits)
        self.asm.emit("JNEG", idx, done)
        if lazy:
            body(OVal(self, E, idx, getattr(sv, "alive", None)))
        else:
            self.unord(E, idx, xloc)
            body(Val(E, xloc))
        self.asm.emit("JMP", top)
        self.asm.label(done)

    def set_elements(self, node, env, ctx, base):
        """Classify a quantifier / comprehension domain: ('const', [values]) | ('val', Val) |
        ('range', lo, hi) with runtime bounds."""
        c = self.try_const(node, env, ctx, base)
        if c is not None:
            if not is_set(c.v):
                raise CompileError(f"quantifier domain is not a set: {fmt(c.v)}")
            return ("const", list(set_iter(c.v)))
        if node.k == "bin" and node.a[0] == "..":
            lo = self.cx(node.a[1], env, ctx, base)
            hi = self.cx(node.a[2], env, ctx, base)
            return ("range", lo, hi)
        node, filters = self._peel_filters(node, env, ctx, base)
        if filters:
            inner = self.set_elements(node[0], node[1], node[2], node[3])
            if inner[0] in ("sparse", "subsets"):
                return (inner[0], inner[1], inner[2] + filters)
            node, env, ctx, base = node[4]
        else:
            node, env, ctx, base = node
        if node.k == "subset":
            # SUBSET S for a run-time S (InnerSerial.tla:47,67): the sub-masks of S's bitset are enumerated in place
            sv = self.cx(node.a[0], env, ctx, base)
            if type(sv) is Const:
                t0 = self.natural_type(sv.v)
                sv = self.materialize(sv, t0)
            if isinstance(sv.t, TSet) and not isinstance(sv.t.elem, TBottom) and sv.t.size <= 8:
                return ("subsets", sv, [])
            raise CompileError(f"SUBSET of a run-time set over a universe of more than 256 values (line {node.line})")
        if node.k == "domain":
            f = self.cx(node.a[0], env, ctx, base)
            if isinstance(f, Val) and isinstance(f.t, TSparse):
                return ("sparse", f, [])
            if isinstance(f, Val) and isinstance(f.t, TPFun):
                return ("val", self.pf_domain(f))
            if isinstance(f, Val) and isinstance(f.t, TSeq):
                return ("range", Const(1), Val(TInt(0, f.t.cap), f.loc))
            if isinstance(f, Val) and isinstance(f.t, TFun):
                return ("const", list(f.t.keys))
            if isinstance(f, Val) and isinstance(f.t, TTuple):
                return ("const", list(range(1, len(f.t.elems) + 1)))
        v = self.cx(node, env, ctx, base)
        if type(v) is Const:
            return ("const", list(set_iter(v.v)))
        if isinstance(v.t, TSparse) and v.t.vt is None:
            return ("sparse", v, [])
        if not isinstance(v.t, TSet):
            raise CompileError(f"quantifier domain has non-set type {v.t}")
        return ("val", v)

    def _peel_filters(self, node, env, ctx, base):
        """Follow operator applications / set filters down to the underlying domain:
        ValidMessage(messages) == {m \\in DOMAIN messages : msgs[m] > 0}  (raft.tla:127-131) is iterated as
        DOMAIN messages with the predicate applied inside the loop instead of building the filtered set.
        -> ((node, env, ctx, base, original), [(pat, pred, env, ctx, base), ...])"""
        orig = (node, env, ctx, base)
        filters = []
        cur = orig
        for _ in range(8):
            nd, e_, c_, b_ = cur
            if self.try_const(nd, e_, c_, b_) is not None:
                break
            if nd.k in ("id", "app", "sel"):
                try:
                    tgt = self._expand(nd, e_, c_, b_)
                except (CompileError, EvalError):
                    tgt = None
                if tgt is None or tgt[0].k not in ("setfilter", "domain", "id", "app", "sel"):
                    break
                cur = tgt
                continue
            if nd.k == "setfilter" and isinstance(nd.a[0][0], str):
                (pat, s2), pred = nd.a
                filters.append((pat, pred, e_, c_, b_))
                cur = (s2, e_, c_, b_)
                continue
            break
        if not filters:
            return orig, []
        return cur + (orig,), filters

    def bind(self, env, pat, x):
        env2 = dict(env)
        if isinstance(pat, str):
            env2[pat] = x
            return env2
        names = pat[1]
        if type(x) is Const:
            if not isinstance(x.v, tuple) or len(x.v) != len(names):
                raise CompileError("tuple pattern mismatch")
            for nm, xv in zip(names, x.v):
                env2[nm] = Const(xv)
        else:
            if not isinstance(x.t, TTuple) or len(x.t.elems) != len(names):
                raise CompileError("tuple pattern mismatch")
            base = x.loc
            for nm, te, to in zip(names, x.t.elems, x.t.offs):
                env2[nm] = Val(te, base + to)
        return env2

    def for_each(self, bounds, env, ctx, base, body, i=0):
        """Emit nested iteration over quantifier bounds; body(env2) emits the per-combination code."""
        if i == len(bounds):
            body(env)
            return
        pat, sn = bounds[i]
        if sn is None:
            raise CompileError("unbounded quantifier")
        kind = self.set_elements(sn, env, ctx, base)
        if kind[0] == "const":
            vals = kind[1]
            if len(vals) <= UNROLL_MAX or not vals:
                for v in vals:
                    self.for_each(bounds, self.bind(env, pat, Const(v)), ctx, base, body, i + 1)
                return
            # long constant domain: iterate a table of representations
            t = None
            for v in vals:
                t = join(t, type_of_value(v, self.seq_cap))
            reps = []
            for v in vals:
                reps += self.codec.rep(t, v)
            tbase = self.asm.const_table(reps)
            cnt = self.alloc(1)
            off = self.alloc(1)
            xloc = self.alloc(t.size)
            self.li(cnt, 0)
            top, done = Label("cl"), Label("cd")
            self.asm.label(top)
            tmp = self.alloc(1)
            self.asm.emit("LTI", tmp, cnt, len(vals))
            self.asm.emit("JZ", tmp, done)
            self.asm.emit("MULI", off, cnt, t.size)
            for w in range(t.size):
                self.asm.emit("TBL", xloc + w, tbase + w, off)
            self.asm.emit("ADDI", cnt, cnt, 1)
            self.for_each(bounds, self.bind(env, pat, Val(t, xloc)), ctx, base, body, i + 1)
            self.asm.emit("JMP", top)
            self.asm.label(done)
            return
        if kind[0] == "range":
            lo = self.as_val(kind[1], TInt())
            hi = self.as_val(kind[2], TInt())
            tl = lo.t if isinstance(lo.t, TInt) else TInt()
            th = hi.t if isinstance(hi.t, TInt) else TInt()
            xt = TInt(tl.lo, th.hi) if (tl.lo is not None and th.hi is not None) else TInt()
            x = self.alloc(1)
            hi_s = self.alloc(1)
            self.asm.emit("MOV", hi_s, hi.loc)
            self.asm.emit("ADDI", x, lo.loc, -1)
            top, done = Label("rl"), Label("rd")
            self.asm.label(top)
            self.asm.emit("ADDI", x, x, 1)
            tmp = self.alloc(1)
            self.asm.emit("LE", tmp, x, hi_s)
            self.asm.emit("JZ", tmp, done)
            self.for_each(bounds, self.bind(env, pat, Val(xt, x)), ctx, base, body, i + 1)
            self.asm.emit("JMP", top)
            self.asm.label(done)
            return
        if kind[0] == "subsets":
            sv, filters = kind[1], kind[2]
            nw = sv.t.size
            full, sub, t1 = self.alloc(nw), self.alloc(nw), self.alloc(1)
            self.movn(full, sv.loc, nw)
            self.movn(sub, full, nw)
            top, skip, done = Label("sbl"), Label("sbs"), Label("sbd")
            self.asm.label(top)
            rv = Val(sv.t, sub)
            for fpat, fpred, fenv, fctx, fbase in filters:
                nxt = Label("sbp")
                self.cc(fpred, self.bind(fenv, fpat, rv), fctx, fbase, nxt, skip)
                self.asm.label(nxt)
            self.for_each(bounds, self.bind(env, pat, rv), ctx, base, body, i + 1)
            self.asm.label(skip)
            # next sub-mask: (sub - 1) & full on the multi-word integer; the empty set was the last one
            self.asm.emit("BISZ", t1, sub, nw)
            self.asm.emit("JNZ", t1, done)
            andl = Label("sba")
            for w in range(nw):
                dec = Label("sbw")
                self.asm.emit("JNZ", sub + w, dec)
                self.li(sub + w, -1)                    # borrow from the next word
                continue_l = Label("sbc")
                self.asm.emit("JMP", continue_l)
                self.asm.label(dec)
                self.asm.emit("ADDI", sub + w, sub + w, -1)
                self.asm.emit("JMP", andl)
                self.asm.label(continue_l)
            self.asm.label(andl)
            self.asm.emit("BAND", sub, sub, full, nw)
            self.asm.emit("JMP", top)
            self.asm.label(done)
            return
        if kind[0] == "sparse":
            cont, filters = kind[1], kind[2]

            def each_entry(k, v):
                skip = Label("sfk")
                for fpat, fpred, fenv, fctx, fbase in filters:
                    nxt = Label("sfp")
                    self.cc(fpred, self.bind(fenv, fpat, k), fctx, fbase, nxt, skip)
                    self.asm.label(nxt)
                self.for_each(bounds, self.bind(env, pat, k), ctx, base, body, i + 1)
                self.asm.label(skip)
            self.sp_loop(cont, each_entry)
            return
        sv = kind[1]
        self.loop_set(sv, lambda xv: self.for_each(bounds, self.bind(env, pat, xv), ctx, base, body, i + 1))

    # --------------------------------------------------------- name resolution
    def resolve(self, name, env, ctx):
        """-> ('env', x) | ('var', name) | ('def', OpDef, dctx) | ('subst', node, octx) | ('const', v) |
        ('builtin', b)"""
        if name in env:
            return ("env", env[name])
        sb = ctx.substs.get(name)
        if sb is not None:
            return ("subst", sb[0], sb[1])
        if name in ctx.varset:
            return ("var", name)
        if name in ctx.consts:
            return ("const", ctx.consts[name])
        d = ctx.defs.get(name)
        if d is not None:
            return ("def", d[0], d[1])
        b = self.ev.builtins.get(name)
        if b is not None:
            return ("builtin", b)
        raise CompileError(f"unknown identifier {name}")

    def var_val(self, name, base) -> Val:
        if base == "P":
            if name not in self.bound:
                raise CompileError(f"primed variable {name}' is read before it is assigned")
            return Val(self.var_types[name], self.p_off[name])
        return Val(self.var_types[name], self.n_off[name])

    def bind_args(self, params, args, env, ctx, base, body=None):
        env2 = {}
        for (pn, ar), a in zip(params, args):
            if ar > 0:
                env2[pn] = self.op_value(a, env, ctx)
            else:
                c = self.try_const(a, env, ctx, base) if a.k in ("num", "str", "bool", "id") else None
                if c is not None:
                    env2[pn] = c
                else:
                    env2[pn] = self._bind_by_name(Lazy(a, env, ctx, base), pn, (body,))
        return env2

    @staticmethod
    def _count_uses(name, x):
        if isinstance(x, Node):
            if x.k == "id" and x.a[0] == name:
                return 1
            return sum(Lowering._count_uses(name, y) for y in x.a)
        if isinstance(x, (tuple, list)):
            return sum(Lowering._count_uses(name, y) for y in x)
        if isinstance(x, OpDef):
            return Lowering._count_uses(name, x.body)
        return 0

    @staticmethod
    def _has_prime(x):
        if isinstance(x, Node):
            return x.k in ("prime", "unchanged") or any(Lowering._has_prime(y) for y in x.a)
        if isinstance(x, (tuple, list)):
            return any(Lowering._has_prime(y) for y in x)
        if isinstance(x, OpDef):
            return Lowering._has_prime(x.body)
        return False

    CX_BUDGET = 1_000_000      # expression nodes lowered before inline expansion is abandoned for subroutines
    EAGER_MIN_WORDS = 8
    EAGER_MIN_CODE = 40

    def _bind_by_name(self, lz: Lazy, name, scope):
        """Decide between call-by-name re-lowering at every use (Lazy) and one evaluation at the binding site
        (PVal): the latter when the name is used at least twice and the value is large or dynamically shaped."""
        if lz.base != "N" or self.dry or scope is None or any(x is None for x in scope):
            return lz
        if sum(self._count_uses(name, x) for x in scope) < 2:
            return lz
        # an alias of an outer by-name binding (a history prefix handed down through several operators,
        # serializableSnapshotIsolation.tla:269-399): decide on the underlying expression, here, where it is
        # used repeatedly -- each level of the chain on its own sees a single use
        orig = lz
        for _ in range(16):
            nd = lz.node
            if nd.k == "id" and type(lz.env.get(nd.a[0])) is Lazy and lz.env[nd.a[0]].base == "N":
                lz = lz.env[nd.a[0]]
            else:
                break
        node = lz.node
        if node.k in ("id", "num", "str", "bool", "lambda") or self._has_prime(node):
            return orig
        save_top, save_bound = self.top, self.bound
        try:
            with self.asm.capture() as cap:
                poison = self.alloc(1)
                x = self.cx(node, lz.env, lz.ctx, "N")
        except (CompileError, TypeErr):
            self.top, self.bound = save_top, save_bound
            return orig
        self.bound = save_bound
        if type(x) is Const:
            self.top = save_top
            return x
        ninstr = sum(1 for i in cap.buf if i[0] != "label")
        if type(x) is not Val or not (x.t.size >= self.EAGER_MIN_WORDS or has_dynamic(x.t)
                                      or ninstr >= self.EAGER_MIN_CODE) \
                or any(i[0] in ("ASSERTF", "EMIT", "GEN", "INVF", "EMITD") for i in cap.buf):
            self.top = save_top
            return orig
        end = Label("pve")
        ntrap = 0
        out = []
        for ins in cap.buf:
            if ins[0] == "TRAP":
                ntrap += 1
                out.append(("LI", poison, int(ins[1]) | (int(ins[2]) << 4)))
                out.append(("JMP", end))
            else:
                out.append(ins)
        if ntrap:
            self.li(poison, 0)
        self.asm.splice(out)
        self.asm.label(end)
        return PVal(x.t, x.loc, poison if ntrap else None, lz)

    def op_value(self, a, env, ctx) -> OpC:
        if a.k == "lambda":
            return OpC([(p, 0) for p in a.a[0]], a.a[1], env, ctx, "LAMBDA")
        if a.k == "id":
            r = self.resolve(a.a[0], env, ctx)
            if r[0] == "env" and type(r[1]) is OpC:
                return r[1]
            if r[0] == "def":
                return OpC(r[1].params, r[1].body, {}, r[2], r[1].name)
        raise CompileError(f"operator argument expected at line {a.line}")

    def let_env(self, defs, env, ctx, base, body=None):
        env2 = dict(env)
        for i, d in enumerate(defs):
            if d.params:
                env2[d.name] = OpC(d.params, d.body, env2, ctx, d.name)
            else:
                env2[d.name] = self._bind_by_name(Lazy(d.body, env2, ctx, base), d.name,
                                                  None if body is None else (body,) + tuple(defs[i + 1:]))
        return env2

    # ------------------------------------------------------------ expressions
    def cx(self, n: Node, env, ctx, base="N", want=None):
        """Compile expression n in value context -> Const | Val."""
        c = self.try_const(n, env, ctx, base)
        if c is not None:
            return c
        self._cx_count += 1
        if self._cx_count > self.cx_budget and not self.use_subs:
            raise CompileBudget(f"inline expansion of the specification exceeds {self.cx_budget} expression nodes")
        k = n.k
        if n.line:
            self.asm.cur_line = n.line
        m = getattr(self, "x_" + k, None)
        if m is None:
            raise CompileError(f"unsupported construct `{k}` at line {n.line} col {n.col}")
        return m(n, env, ctx, base, want)

    def x_id(self, n, env, ctx, base, want):
        r = self.resolve(n.a[0], env, ctx)
        if r[0] == "env":
            x = r[1]
            if type(x) is Lazy:
                save = self.bound
                return self.cx(x.node, x.env, x.ctx, x.base if x.base == "P" else base, want)
            if type(x) is OpC:
                raise CompileError(f"operator {n.a[0]} used as a value")
            if type(x) is PVal:
                if base == "P":
                    return self.cx(x.lazy.node, x.lazy.env, x.lazy.ctx, "P", want)
                if x.poison is not None:
                    ok = Label("pvk")
                    self.asm.emit("JZ", x.poison, ok)
                    self.asm.emit("TRAP", TRAP_EVAL, n.line)
                    self.asm.label(ok)
                return Val(x.t, x.loc)
            return x
        if r[0] == "var":
            return self.var_val(r[1], base)
        if r[0] == "subst":
            return self.cx(r[1], {}, r[2], base, want)
        if r[0] == "const":
            return Const(r[1])
        if r[0] == "def":
            if r[1].params:
                raise CompileError(f"operator {n.a[0]} used without arguments")
            key = (n.a[0], id(r[2]), base, self.program)
            hv = self.hoisted.get(key)
            if hv is not None:
                return hv
            self.def_uses[key] = self.def_uses.get(key, 0) + 1
            self.def_info[key] = (r[1], r[2])
            if self.use_subs:
                v = self._sub_call(r[1], r[2], (), env, ctx, base, want, n)
                if v is not None:
                    return v
            return self.cx(r[1].body, {}, r[2], base, want)
        raise CompileError(f"cannot compile identifier {n.a[0]}")

    def x_prime(self, n, env, ctx, base, want):
        return self.cx(n.a[0], env, ctx, "P", want)

    def x_at(self, n, env, ctx, base, want):
        if "@" not in env:
            raise CompileError("@ outside EXCEPT")
        return env["@"]

    def x_app(self, n, env, ctx, base, want):
        name, args = n.a
        r = self.resolve(name, env, ctx)
        if r[0] == "env" and type(r[1]) is OpC:
            op = r[1]
            env2 = dict(op.env)
            env2.update(self.bind_args(op.params, args, env, ctx, base, op.body))
            return self._inline(op.body, env2, op.ctx, base, want, n)
        if r[0] == "def":
            d = r[1]
            if len(d.params) != len(args):
                raise CompileError(f"arity mismatch calling {name}")
            if self.use_subs:
                v = self._sub_call(d, r[2], args, env, ctx, base, want, n)
                if v is not None:
                    return v
            return self._inline(d.body, self.bind_args(d.params, args, env, ctx, base, d.body), r[2], base, want, n)
        if r[0] == "builtin":
            return self.builtin(name, args, n, env, ctx, base, want)
        raise CompileError(f"cannot apply {name} at line {n.line}")

    COMPACT_MIN = 24

    def _compact(self, m0, x):
        """x was computed with temporaries allocated since mark m0, all of which are dead except x itself: slide x down
        to m0 and give the rest back (keeps the VM frame -- per-thread local memory on the GPU -- small)."""
        if type(x) is not Val or self.dry:
            return x
        size = x.t.size
        if x.loc + size <= m0:                       # lives in older storage
            self.release(m0)
            return x
        if x.loc < m0 or self.top - (m0 + size) < self.COMPACT_MIN:
            return x
        self.movn(m0, x.loc, size)
        self.top = m0 + size
        return Val(x.t, m0)

    def _inline(self, body, env2, ctx2, base, want, n):
        """Inline an operator body.  RECURSIVE operators (serializableSnapshotIsolation.tla:465,823,1042,1094)
        are unrolled: every nested activation of the same body is a fresh copy, up to `rec_depth` levels; an
        activation beyond that traps at run time (evaluation error), it is never silently cut off."""
        key = id(body)
        d = self._rec_depth.get(key, 0)
        if d >= self.rec_depth:
            self.asm.emit("TRAP", TRAP_EVAL, n.line)
            return Val(want if want is not None else TBottom(), 0)
        self._rec_depth[key] = d + 1
        m0 = self.mark()
        try:
            return self._compact(m0, self.cx(body, env2, ctx2, base, want))
        finally:
            self._rec_depth[key] = d

    # ------------------------------------------------------------ subroutines
    SUB_MIN_NODES = 12

    @staticmethod
    def _node_count(x, lim=64):
        """Size of an operator body (AST nodes), capped."""
        n = 0
        stack = [x]
        while stack and n < lim:
            y = stack.pop()
            if isinstance(y, Node):
                n += 1
                stack.extend(y.a)
            elif isinstance(y, (tuple, list)):
                stack.extend(y)
            elif isinstance(y, OpDef):
                stack.append(y.body)
        return n

    def _sub_call(self, d, dctx, args, env, ctx, base, want, n):
        """Call module-level operator d as a subroutine (one compiled copy per (operator, constant arguments, types
        of run-time arguments, expected type)); None => the caller inlines it as before.
        Arguments are evaluated once at the call site; a trap while evaluating one is deferred (poison word) to the
        first use of the parameter inside the body, which keeps call-by-name semantics."""
        if base != "N":
            return None
        if any(ar > 0 for _p, ar in d.params) or self._has_prime(d.body) or d.body.k == "fcndef":
            return None
        if self._node_count(d.body) < self.SUB_MIN_NODES:
            return None
        if id(d.body) in self._sub_active or id(d.body) in self._rec_depth and self._rec_depth[id(d.body)] > 0:
            return None                          # (mutually) recursive: unrolled by _inline
        m0 = self.mark()
        avals, key = [], [id(d.body), id(dctx), want]
        try:
            for (pn, _ar), a in zip(d.params, args):
                c = self.try_const(a, env, ctx, base)
                if c is not None:
                    avals.append(c)
                    key.append(("c", vkey(c.v)))
                    continue
                with self.asm.capture() as cap:
                    poison = self.alloc(1)
                    x = self.cx(a, env, ctx, "N")
                if type(x) is Const:
                    avals.append(x)
                    key.append(("c", vkey(x.v)))
                    continue
                if any(i[0] in ("ASSERTF", "EMIT", "GEN", "INVF", "EMITD") for i in cap.buf):
                    self.release(m0)
                    return None
                if type(x) is OVal:
                    x = Val(x.t, x.loc)
                end = Label("sae")
                ntrap = 0
                out = []
                for ins in cap.buf:
                    if ins[0] == "TRAP":
                        ntrap += 1
                        out.append(("LI", poison, 1))
                        out.append(("JMP", end))
                    else:
                        out.append(ins)
                self.li(poison, 0)
                self.asm.splice(out)
                self.asm.label(end)
                avals.append((x, poison))
                key.append(("t", x.t))
        except (CompileError, TypeErr):
            self.release(m0)
            return None
        key = tuple(key)
        sub = self.subs.get(key)
        if sub is None:
            sub = self._sub_compile(key, d, dctx, avals, want, n)
            if sub is None:
                self.release(m0)
                return None
        self.sub_calls.setdefault(self._sub_stack[-1] if self._sub_stack else None, set()).add(key)
        for (pslot, ppoison), av in zip(sub["params"], [a for a in avals if type(a) is not Const]):
            x, poison = av
            self.movn(pslot, x.loc, x.t.size)
            self.asm.emit("MOV", ppoison, poison)
        self.asm.emit("CALL", sub["ret"], sub["entry"])
        rt = sub["type"]
        self.release(m0)
        dst = self.alloc(rt.size)
        self.movn(dst, sub["res"], rt.size)
        return Val(rt, dst)

    def _sub_compile(self, key, d, dctx, avals, want, n):
        """Lower the body of d once into its own buffer (spliced after the main programs).  The subroutine owns a
        static frame region [base, base+size): return address, parameters (+ poison words), temporaries, result.
        Discovery pass: base is a dummy (frames overlap; the code is discarded, sizes and the call graph are kept).
        Final pass: base comes from the plan -- subroutines of one call-graph level share a region (they never call
        each other), callers sit on higher levels, the main programs below all of them."""
        base = self.sub_base0 if self.sub_plan is None else self.sub_plan.get(key)
        if base is None:
            return None                     # not in the plan (did not occur in the discovery pass): inline
        self._sub_active.add(id(d.body))
        self._sub_stack.append(key)
        save = (self.top, self.high, self.bound)
        self.top = self.high = base
        entry = Label("sub_" + d.name)
        ok = False
        try:
            with self.asm.capture() as cap:
                self.asm.label(entry)
                ret = self.alloc(1)
                params, env2 = [], {}
                for (pn, _ar), av in zip(d.params, avals):
                    if type(av) is Const:
                        env2[pn] = av
                    else:
                        x, _p = av
                        pslot = self.alloc(x.t.size)
                        ppoison = self.alloc(1)
                        params.append((pslot, ppoison))
                        env2[pn] = PVal(x.t, pslot, ppoison, Lazy(Node("runtime", ()), {}, dctx, "N"))
                r = self.cx(d.body, env2, dctx, "N", want)
                if type(r) is Const:
                    rt = want if want is not None else self.natural_type(r.v)
                    rv = self.materialize(r, rt)
                else:
                    rv = self.coerce(r, want) if want is not None and r.t != want else r
                    if type(rv) is OVal:
                        rv = Val(rv.t, rv.loc)
                    rt = rv.t
                res = self.alloc(rt.size)
                self.movn(res, rv.loc, rt.size)
                self.asm.emit("RET", ret)
            ok = True
        except CompileBudget:
            raise
        except (CompileError, TypeErr):
            ok = False
        finally:
            self._sub_active.discard(id(d.body))
            self._sub_stack.pop()
            size = self.high - base
            self.top, self.high, self.bound = save
        if not ok:
            return None
        self.sub_bufs.append(cap.buf)
        sub = {"entry": entry, "ret": ret, "params": params, "res": res, "type": rt, "size": size}
        self.subs[key] = sub
        return sub

    def _plan_sub_frames(self, main_high):
        """Static frame bases from the discovery pass.  Two instances are live together only along a call chain, so
        a subroutine sits just above the highest-ending of its callers (the main programs' temporaries for those
        called from there): the frame is as deep as the deepest call chain, like a stack's high-water mark, not the
        sum of the largest frame of every call-graph level.  (SSI 2 x 2: 4341 -> 3390 words -- the 1.6 K-word leaf
        `WellFormedTransactionsInHistory` is only ever called from an invariant.)"""
        level = {}

        def lv(k, seen=()):
            if k in level:
                return level[k]
            if k in seen:
                raise CompileError("internal: cycle in the subroutine call graph")
            cs = [c for c in self.sub_calls.get(k, ()) if c in self.subs]
            level[k] = 0 if not cs else 1 + max(lv(c, seen + (k,)) for c in cs)
            return level[k]
        for k in self.subs:
            lv(k)
        callers = {k: [] for k in self.subs}
        for p, cs in self.sub_calls.items():
            if p is None or p not in self.subs:
                continue
            for c in cs:
                if c in callers:
                    callers[c].append(p)
        base, b = {}, main_high + 8
        for k in sorted(self.subs, key=lambda k: -level[k]):     # callers (higher levels) before their callees
            base[k] = max([main_high + 8] + [base[p] + self.subs[p]["size"] + 2 for p in callers[k]])
            b = max(b, base[k] + self.subs[k]["size"] + 2)
        if b > MAXREG:
            raise CompileError(f"frame of {b} words exceeds the 16K-word limit (subroutine frames)")
        return base, b

    def x_recset(self, n, env, ctx, base, want):
        """[f1 : S1, ..., fk : Sk] with run-time component sets (InnerSerial.tla:5 `opId`): bitset over the record
        universe, filled by nested loops over the components."""
        pairs = list(n.a[0])
        ops = [self.cx(x, env, ctx, base) for _f, x in pairs]
        fts = {}
        for (f, _x), o in zip(pairs, ops):
            ot = o.t if isinstance(o, Val) else self.natural_type(o.v)
            if not isinstance(ot, TSet):
                raise CompileError(f"component {f} of the record set is not a bitset-typed set (line {n.line})")
            fts[f] = ot.elem
        rt = TRec([sorted(fts)], fts)
        t = want if isinstance(want, TSet) and isinstance(want.elem, TRec) else TSet(rt)
        dst = self.alloc(t.size)
        self.asm.emit("ZERO", dst, t.size)
        env2 = dict(env)
        bounds = []
        for i, o in enumerate(ops):
            env2[f"__ro{i}"] = o
            bounds.append((f"__rt{i}", Node("id", (f"__ro{i}",), n.line, n.col)))

        def body(env3):
            m0 = self.mark()
            loc = self.alloc(rt.size)
            for i, (f, _x) in enumerate(pairs):
                xv = self.coerce(env3[f"__rt{i}"], rt.fields[f])
                self.movn(loc + rt.off[f], xv.loc, rt.fields[f].size)
            self._set_add(dst, t, Val(rt, loc), n)
            self.release(m0)
        self.for_each(bounds, env2, ctx, base, body)
        return Val(t, dst)

    def x_times(self, n, env, ctx, base, want):
        """A \\X B \\X ... with run-time operands: bitset over the tuple universe."""
        ops = [self.cx(x, env, ctx, base) for x in n.a[0]]
        ets = []
        for o in ops:
            ot = o.t if isinstance(o, Val) else self.natural_type(o.v)
            if not isinstance(ot, TSet):
                raise CompileError(f"\\X operand is not a bitset-typed set (line {n.line})")
            ets.append(ot.elem)
        t = want if isinstance(want, TSet) and isinstance(want.elem, TTuple) else TSet(TTuple(ets))
        dst = self.alloc(t.size)
        self.asm.emit("ZERO", dst, t.size)
        env2 = dict(env)
        bounds = []
        for i, o in enumerate(ops):
            env2[f"__xo{i}"] = o
            bounds.append((f"__xt{i}", Node("id", (f"__xo{i}",), n.line, n.col)))

        def body(env3):
            m0 = self.mark()
            tt = t.elem
            loc = self.alloc(tt.size)
            for i in range(len(ops)):
                xv = self.coerce(env3[f"__xt{i}"], tt.elems[i])
                self.movn(loc + tt.offs[i], xv.loc, tt.elems[i].size)
            self._set_add(dst, t, Val(tt, loc), n)
            self.release(m0)
        self.for_each(bounds, env2, ctx, base, body)
        return Val(t, dst)

    def x_bigunion(self, n, env, ctx, base, want):
        arg = n.a[0]
        for _ in range(6):          # UNION Range(f): look through operator applications
            if arg.k not in ("id", "app", "sel"):
                break
            tgt = self._expand(arg, env, ctx, base)
            if tgt is None:
                break
            arg, env, ctx, base = tgt
        if arg.k == "setenum":
            parts = [lambda w, x=x: self.cx(x, env, ctx, base, w) for x in arg.a[0]]
            loop = None
        elif arg.k == "setmap":
            parts, loop = None, arg
        else:
            raise CompileError(f"UNION of a computed set of sets is not supported (line {n.line})")
        t = want if isinstance(want, (TSet, TSparse)) else None
        if t is None:
            # element type from a dry run of the member expression(s)
            holder = []
            with self.asm.capture():
                save_top = self.top
                if loop is not None:
                    def probe(env2):
                        x = self.cx(loop.a[0], env2, ctx, base)
                        holder.append(x.t if isinstance(x, Val) else self.natural_type(x.v))
                    self.for_each(loop.a[1], env, ctx, base, probe)
                else:
                    for p_ in parts:
                        x = p_(None)
                        holder.append(x.t if isinstance(x, Val) else self.natural_type(x.v))
                self.top = save_top
            t = TBottom()
            for h in holder:
                t = join(t, h)
            if isinstance(t, TBottom):
                t = TSet(TBottom())
        if isinstance(t, TSparse):
            dst = self.sp_new(t)
            add = lambda x: self.sp_loop(self.coerce(x, t), lambda k, v: self.sp_insert(dst, k.loc, n.line))
        else:
            dst = Val(t, self.alloc(t.size))
            self.asm.emit("ZERO", dst.loc, t.size)

            def add(x):
                xv = self.coerce(x, t)
                self.asm.emit("BOR", dst.loc, dst.loc, xv.loc, t.size)
        if loop is not None:
            def body(env2):
                m0 = self.mark()
                add(self.cx(loop.a[0], env2, ctx, base, t))
                self.release(m0)
            self.for_each(loop.a[1], env, ctx, base, body)
        else:
            for p_ in parts:
                add(p_(t))
        return dst

    def x_sel(self, n, env, ctx, base, want):
        r = self.ev.resolve_sel(n.a[0], self.eval_env(env), Fr(ctx))
        if r[0] == "def":
            _, od, dctx, args = r
            return self.cx(od.body, self.bind_args(od.params, args, env, ctx, base), dctx, base, want)
        if r[0] == "name":
            _, name, c2, args = r
            return self.cx(Node("id", (name,)), {}, c2, base, want)
        _, node, dctx, (od, args) = r
        return self.cx(node, self.bind_args(od.params, args, env, ctx, base), dctx, base, want)

    def x_let(self, n, env, ctx, base, want):
        m0 = self.mark()
        return self._compact(m0, self.cx(n.a[1], self.let_env(n.a[0], env, ctx, base, n.a[1]), ctx, base, want))

    # booleans in value context
    def _bool_value(self, n, env, ctx, base, want):
        dst = self.alloc(1)
        lt, lf, end = Label("bt"), Label("bf"), Label("be")
        self.cc(n, env, ctx, base, lt, lf)
        self.asm.label(lt)
        self.li(dst, 1)
        self.asm.emit("JMP", end)
        self.asm.label(lf)
        self.li(dst, 0)
        self.asm.label(end)
        return Val(TBool(), dst)

    x_and = x_or = x_not = x_forall = x_exists = _bool_value

    def x_bin(self, n, env, ctx, base, want):
        op, ln, rn = n.a
        if op in ("=", "#", "<", ">", "<=", ">=", "\\in", "\\notin", "\\subseteq", "=>", "<=>", "\\subset",
                  "\\supseteq"):
            return self._bool_value(n, env, ctx, base, want)
        if op in ("+", "-", "*", "\\div", "%"):
            a = self.cx(ln, env, ctx, base)
            b = self.cx(rn, env, ctx, base)
            ta = self._int_t(a)
            tb = self._int_t(b)
            rt = self._arith_type(op, ta, tb)
            dst = self.alloc(1)
            if type(b) is Const and op in ("+", "-") and IMM28_MIN < b.v < IMM28_MAX:
                av = self.as_val(a, TInt())
                self.asm.emit("ADDI", dst, av.loc, b.v if op == "+" else -b.v)
            elif type(b) is Const and op == "*" and IMM28_MIN < b.v < IMM28_MAX:
                av = self.as_val(a, TInt())
                self.asm.emit("MULI", dst, av.loc, b.v)
            else:
                av = self.as_val(a, TInt())
                bv = self.as_val(b, TInt())
                self.asm.emit({"+": "ADD", "-": "SUB", "*": "MUL", "\\div": "DIV", "%": "MOD"}[op],
                              dst, av.loc, bv.loc)
            return Val(rt, dst)
        if op == "@@":
            return self.fcn_merge(ln, rn, env, ctx, base, want, n)
        if op == ":>" and isinstance(want, TSparse) and want.vt is not None:
            dst = self.sp_new(want)
            k = self.cx(ln, env, ctx, base, want.kt)
            v = self.cx(rn, env, ctx, base, want.vt)
            self.sp_insert(dst, self.sp_entry(want, k, v), n.line)
            return dst
        if op in ("\\cup", "\\cap", "\\"):
            a = self.cx(ln, env, ctx, base, want)
            tw = want if want is not None else (a.t if isinstance(a, Val) else None)
            if isinstance(tw, TSparse):
                b = self.cx(rn, env, ctx, base, tw)
                return self.sp_setop(op, a, b, tw, n.line)
            b = self.cx(rn, env, ctx, base, tw)
            if isinstance(b, Val) and isinstance(b.t, TSparse):
                return self.sp_setop(op, a, b, b.t, n.line)
            if type(a) is Const and isinstance(b, Val) and want is None:
                a2 = a
                t = b.t
            t = want
            if t is None:
                ta = a.t if isinstance(a, Val) else self.natural_type(a.v)
                tb = b.t if isinstance(b, Val) else self.natural_type(b.v)
                t = join(ta, tb)
            if not isinstance(t, TSet):
                raise CompileError(f"set operator {op} on non-set type {t}")
            av = self.coerce(a, t)
            bv = self.coerce(b, t)
            dst = self.alloc(t.size)
            self.asm.emit({"\\cup": "BOR", "\\cap": "BAND", "\\": "BANDN"}[op], dst, av.loc, bv.loc, t.size)
            return Val(t, dst)
        if op == "..":
            a = self.cx(ln, env, ctx, base)
            b = self.cx(rn, env, ctx, base)
            ta, tb = self._int_t(a), self._int_t(b)
            if ta.lo is None or tb.hi is None:
                raise CompileError("a..b with unbounded runtime bounds used as a value")
            t = want if isinstance(want, TSet) else TSet(TInt(ta.lo, tb.hi))
            E = t.elem
            dst = self.alloc(t.size)
            self.asm.emit("ZERO", dst, t.size)
            av, bv = self.as_val(a, TInt()), self.as_val(b, TInt())
            x = self.alloc(1)
            tmp = self.alloc(1)
            top, done = Label("rg"), Label("rgd")
            self.asm.emit("MOV", x, av.loc)
            self.asm.label(top)
            self.asm.emit("LE", tmp, x, bv.loc)
            self.asm.emit("JZ", tmp, done)
            o = self.ord_in(E, Val(TInt(E.lo, E.hi), x))
            ok = Label("rok")
            self.asm.emit("JNEG", o, ok)
            self.asm.emit("BSET", dst, o)
            self.asm.label(ok)
            self.asm.emit("ADDI", x, x, 1)
            self.asm.emit("JMP", top)
            self.asm.label(done)
            return Val(t, dst)
        if op == "\\o":
            return self.seq_concat(ln, rn, env, ctx, base, want)
        if op in ctx.defs or op in env:
            r = self.resolve(op, env, ctx)
            if r[0] == "def":
                return self.cx(r[1].body, self.bind_args(r[1].params, (ln, rn), env, ctx, base), r[2], base, want)
        raise CompileError(f"unsupported operator {op} at line {n.line}")

    def _int_t(self, x) -> TInt:
        if type(x) is Const:
            if type(x.v) is not int:
                raise CompileError(f"integer expected, got {fmt(x.v)}")
            return TInt(x.v, x.v)
        if not isinstance(x.t, TInt):
            raise CompileError(f"integer expected, got type {x.t}")
        return x.t

    @staticmethod
    def _arith_type(op, a: TInt, b: TInt) -> TInt:
        if a.lo is None or b.lo is None:
            return TInt()
        if op == "+":
            lo, hi = a.lo + b.lo, a.hi + b.hi
        elif op == "-":
            lo, hi = a.lo - b.hi, a.hi - b.lo
        elif op == "*":
            c = [a.lo * b.lo, a.lo * b.hi, a.hi * b.lo, a.hi * b.hi]
            lo, hi = min(c), max(c)
        elif op == "%":
            lo, hi = 0, max(b.hi - 1, 0)
        else:
            m = max(abs(a.lo), abs(a.hi))
            lo, hi = -m, m
        if lo < -(1 << 30) or hi > (1 << 30):
            return TInt()
        return TInt(lo, hi)

    def x_neg(self, n, env, ctx, base, want):
        a = self.as_val(self.cx(n.a[0], env, ctx, base), TInt())
        dst = self.alloc(1)
        self.asm.emit("NEG", dst, a.loc)
        t = a.t
        return Val(TInt(-t.hi, -t.lo) if t.lo is not None else TInt(), dst)

    def x_if(self, n, env, ctx, base, want):
        c, a, b = n.a
        cc_ = self.try_const(c, env, ctx, base)
        if cc_ is not None:
            return self.cx(a if cc_.v else b, env, ctx, base, want)
        lt, lf, end = Label("it"), Label("if"), Label("ie")
        if want is not None:
            dst = self.alloc(want.size)
            m0 = self.mark()
            self.cc(c, env, ctx, base, lt, lf)
            self.release(m0)                # temporaries of the condition and of each branch are dead once the
            self.asm.label(lt)              # selected value sits in dst: the branches share one scratch area
            va = self.coerce(self.cx(a, env, ctx, base, want), want)
            self.movn(dst, va.loc, want.size)
            self.release(m0)
            self.asm.emit("JMP", end)
            self.asm.label(lf)
            vb = self.coerce(self.cx(b, env, ctx, base, want), want)
            self.movn(dst, vb.loc, want.size)
            self.release(m0)
            self.asm.label(end)
            return Val(want, dst)
        m0 = self.mark()
        with self.asm.capture() as ca:
            va = self.cx(a, env, ctx, base)
            if type(va) is OVal:
                va = Val(va.t, va.loc)
        top_a = self.top
        if not self.dry:
            self.release(m0)                  # only one branch runs: they share one scratch area
        with self.asm.capture() as cb:
            vb = self.cx(b, env, ctx, base)
            if type(vb) is OVal:
                vb = Val(vb.t, vb.loc)
        self.top = max(self.top, top_a)
        ta = va.t if isinstance(va, Val) else self.natural_type(va.v)
        tb = vb.t if isinstance(vb, Val) else self.natural_type(vb.v)
        t = join(ta, tb)
        dst = self.alloc(t.size)
        self.cc(c, env, ctx, base, lt, lf)
        self.asm.label(lt)
        self.asm.splice(ca.buf)
        va2 = self.coerce(va, t)
        self.movn(dst, va2.loc, t.size)
        self.asm.emit("JMP", end)
        self.asm.label(lf)
        self.asm.splice(cb.buf)
        vb2 = self.coerce(vb, t)
        self.movn(dst, vb2.loc, t.size)
        self.asm.label(end)
        return self._compact(m0, Val(t, dst))

    def x_case(self, n, env, ctx, base, want):
        arms, other = n.a
        node = other
        if node is None:
            node = Node("app", ("__trap_case", ()), n.line, n.col)
        for c, e in reversed(arms):
            node = Node("if", (c, e, node), n.line, n.col)
        return self.cx(node, env, ctx, base, want)

    def x_tuple(self, n, env, ctx, base, want):
        items = [self.cx(x, env, ctx, base) for x in n.a[0]]
        wants = None
        if isinstance(want, TTuple) and len(want.elems) == len(items):
            wants = want.elems
        elif isinstance(want, TSeq):
            wants = [want.elem] * len(items)
        elif isinstance(want, TFun) and want.keys == tuple(range(1, len(items) + 1)):
            wants = [want.elem] * len(items)
        vals = [self.as_val(x, wants[i] if wants else None) for i, x in enumerate(items)]
        if wants:
            vals = [self.coerce(v, w) for v, w in zip(vals, wants)]
        t = TTuple([v.t for v in vals])
        dst = self.alloc(t.size)
        for v, o in zip(vals, t.offs):
            self.movn(dst + o, v.loc, v.t.size)
        r = Val(t, dst)
        if isinstance(want, (TSeq, TFun)):
            return self.coerce(r, want)
        return r

    def x_record(self, n, env, ctx, base, want):
        pairs = n.a[0]
        names = [f for f, _ in pairs]
        wf = want.fields if isinstance(want, TRec) else {}
        vals = {}
        for f, e in pairs:
            x = self.cx(e, env, ctx, base, wf.get(f))
            vals[f] = self.as_val(x, wf.get(f))
        t = TRec([names], {f: vals[f].t for f in names})
        dst = self.alloc(t.size)
        for f in names:
            self.movn(dst + t.off[f], vals[f].loc, vals[f].t.size)
        r = Val(t, dst)
        if isinstance(want, TRec) and want != t:
            return self.coerce(r, want)
        return r

    def x_dot(self, n, env, ctx, base, want):
        r = self.cx(n.a[0], env, ctx, base)
        f = n.a[1]
        if type(r) is Const:
            return Const(r.v.d[f])
        if isinstance(r.t, TBottom):
            return r
        if not isinstance(r.t, TRec) or f not in r.t.fields:
            raise CompileError(f"no field {f} in type {r.t} (line {n.line})")
        t = r.t
        if type(r) is OVal:
            ft = t.fields[f]
            tabs = self._field_tables(t, f)
            dst = self.alloc(ft.size)
            partial = any(f not in alt for alt in t.alts)
            if partial and r.alive is not None:
                vals = self._enum_cached(t)
                partial = any(f not in vals[o].d for o in r.alive)
            for w in range(ft.size):
                self.asm.emit("TBLT" if (partial and w == 0) else "TBL", dst + w, tabs[w], r.oreg)
            return Val(ft, dst)
        if t.tagged:
            mask = 0
            for j, alt in enumerate(t.alts):
                if f in alt:
                    mask |= 1 << j
            if mask != (1 << len(t.alts)) - 1:
                mreg = self.alloc(1)
                tst = self.alloc(1)
                ok = Label("fok")
                self.li(mreg, mask)
                self.asm.emit("BTEST", tst, mreg, r.loc)
                self.asm.emit("JNZ", tst, ok)
                self.asm.emit("TRAP", TRAP_EVAL, n.line)
                self.asm.label(ok)
        return Val(t.fields[f], r.loc + t.off[f])

    def x_setenum(self, n, env, ctx, base, want):
        wel = want.elem if isinstance(want, TSet) else (want.kt if isinstance(want, TSparse) else None)
        items = [self.cx(x, env, ctx, base, wel) for x in n.a[0]]
        if isinstance(want, (TSet, TSparse)):
            t = want
        else:
            et = TBottom()
            for x in items:
                et = join(et, x.t if isinstance(x, Val) else self.natural_type(x.v))
            t = subset_type(self._enumerable(et))
        if isinstance(t, TSparse):
            dst = self.sp_new(t)
            for x in items:
                self.sp_insert(dst, self.sp_entry(t, x), n.line)
            return dst
        dst = self.alloc(t.size)
        self.asm.emit("ZERO", dst, t.size)
        for x in items:
            self._set_add(dst, t, x, n)
        return Val(t, dst)

    def _enumerable(self, t):
        if isinstance(t, TInt) and t.lo is None:
            raise CompileError("set of unbounded integers needs a bounded element type (TypeOK)")
        return t

    def _set_add(self, dst, t: TSet, x, n=None):
        o = self.ord_in(t.elem, x)
        if not self.ord_can_fail(t.elem, x):
            self.asm.emit("BSET", dst, o)
            return
        bad, ok = Label("sb"), Label("so")
        self.asm.emit("JNEG", o, bad)
        self.asm.emit("BSET", dst, o)
        self.asm.emit("JMP", ok)
        self.asm.label(bad)
        self.asm.emit("TRAP", TRAP_OVERFLOW, n.line if n is not None else 0)
        self.asm.label(ok)

    def x_setfilter(self, n, env, ctx, base, want):
        (pat, sn), pred = n.a
        kind = self.set_elements(sn, env, ctx, base)
        if kind[0] == "sparse":
            cont = kind[1]
            t = TSparse(cont.t.kt, None, cont.t.cap)
            if isinstance(want, TSparse) and want.vt is None:
                t = want
            dst = self.sp_new(t)

            def each_s(env2):
                yes, no = Label("sfy"), Label("sfn")
                self.cc(pred, env2, ctx, base, yes, no)
                self.asm.label(yes)
                self.sp_insert(dst, self.sp_entry(t, env2[pat]), n.line)
                self.asm.label(no)
            if not isinstance(pat, str):
                raise CompileError("tuple pattern over a sparse set")
            self.for_each([(pat, sn)], env, ctx, base, each_s)
            return dst
        if kind[0] == "val":
            sv = kind[1]
            t = sv.t
            if isinstance(t.elem, TBottom):
                return sv
            sv2, rest = self.narrow(sv, pat, self.flat_and(pred), env, ctx, base)
            if not rest:
                r = sv2
            else:
                pred2 = rest[0] if len(rest) == 1 else Node("and", (tuple(rest),), pred.line, pred.col)
                dst = self.alloc(t.size)
                self.asm.emit("ZERO", dst, t.size)

                def each(xv):
                    yes, no = Label("fy"), Label("fn")
                    self.cc(pred2, self.bind(env, pat, xv), ctx, base, yes, no)
                    self.asm.label(yes)
                    o = self.ord_in(t.elem, xv)
                    self.asm.emit("BSET", dst, o)
                    self.asm.label(no)
                self.loop_set(sv2, each)
                r = Val(t, dst)
            return self.coerce(r, want) if isinstance(want, TSet) and want != t else r
        if kind[0] == "const":
            vals = kind[1]
            if isinstance(want, TSet):
                t = want
            else:
                et = TBottom()
                for v in vals:
                    et = join(et, type_of_value(v, self.seq_cap))
                t = TSet(self._enumerable(et))
            dst = self.alloc(t.size)
            self.asm.emit("ZERO", dst, t.size)
            for v in vals:
                o = self.codec.ord_of(t.elem, v)
                if o < 0:
                    continue
                yes, no = Label("cy"), Label("cn")
                self.cc(pred, self.bind(env, pat, Const(v)), ctx, base, yes, no)
                self.asm.label(yes)
                self.asm.emit("BSETI", dst, o)
                self.asm.label(no)
            return Val(t, dst)
        if kind[0] == "range" and isinstance(pat, str):
            lo, hi = kind[1], kind[2]
            tl, th = self._int_t(lo), self._int_t(hi)
            if tl.lo is None or th.hi is None:
                raise CompileError("set filter over an unbounded integer range")
            t = want if isinstance(want, TSet) else TSet(TInt(tl.lo, max(th.hi, tl.lo)))
            dst = self.alloc(t.size)
            self.asm.emit("ZERO", dst, t.size)

            def each_r(env2):
                yes, no = Label("ry"), Label("rn")
                self.cc(pred, env2, ctx, base, yes, no)
                self.asm.label(yes)
                self._set_add(dst, t, env2[pat], n)
                self.asm.label(no)
            self.for_each([(pat, sn)], env, ctx, base, each_r)
            return Val(t, dst)
        raise CompileError("set filter over a runtime integer range is not supported")

    def x_setmap(self, n, env, ctx, base, want):
        e, bounds = n.a
        t = want if isinstance(want, (TSet, TSparse)) else None
        if t is None:
            # infer element type by a dry run
            with self.asm.capture():
                save_top = self.top
                holder = []

                def probe(env2):
                    x = self.cx(e, env2, ctx, base)
                    holder.append(x.t if isinstance(x, Val) else self.natural_type(x.v))
                self.for_each(bounds, env, ctx, base, probe)
                self.top = save_top
            et = TBottom()
            for x in holder:
                et = join(et, x)
            t = subset_type(self._enumerable(et))
        if isinstance(t, TSparse):
            sdst = self.sp_new(t)

            def sbody(env2):
                m0 = self.mark()
                x = self.cx(e, env2, ctx, base, t.kt)
                self.sp_insert(sdst, self.sp_entry(t, x), n.line)
                self.release(m0)
            self.for_each(bounds, env, ctx, base, sbody)
            return sdst
        dst = self.alloc(t.size)
        self.asm.emit("ZERO", dst, t.size)

        def body(env2):
            x = self.cx(e, env2, ctx, base, t.elem)
            self._set_add(dst, t, x, n)
        self.for_each(bounds, env, ctx, base, body)
        return Val(t, dst)

    def x_fcn(self, n, env, ctx, base, want):
        bounds, body = n.a
        if len(bounds) != 1:
            raise CompileError("multi-argument function constructors are not supported")
        pat, sn = bounds[0]
        kind = self.set_elements(sn, env, ctx, base)
        if kind[0] == "range" and type(kind[1]) is Const and kind[1].v == 1 and isinstance(pat, str):
            # [j \in 1..n |-> e] with a run-time n: a sequence of run-time length (AlternatingBit.tla Lose)
            hi = self.as_val(kind[2], TInt())
            cap = want.cap if isinstance(want, TSeq) else (hi.t.hi if hi.t.lo is not None else self.seq_cap)
            if cap is None:
                raise CompileError("sequence comprehension needs a capacity (seq_cap)")
            et = want.elem if isinstance(want, TSeq) else None
            if et is None:
                with self.asm.capture():
                    save_top = self.top
                    x0 = self.cx(body, self.bind(env, pat, Const(1)), ctx, base)
                    et = x0.t if isinstance(x0, Val) else self.natural_type(x0.v)
                    self.top = save_top
            t = want if isinstance(want, TSeq) else TSeq(et, cap)
            dst = self.alloc(t.size)
            self.asm.emit("ZERO", dst, t.size)
            done, ovf, okl = Label("scd"), Label("sco"), Label("sck")
            t1 = self.alloc(1)
            self.asm.emit("LEI", t1, hi.loc, 0)
            self.asm.emit("JNZ", t1, done)
            self.asm.emit("GTI", t1, hi.loc, t.cap)
            self.asm.emit("JNZ", t1, ovf)
            self.asm.emit("MOV", dst, hi.loc)
            for j in range(1, t.cap + 1):
                t2 = self.alloc(1)
                self.asm.emit("LTI", t2, hi.loc, j)
                self.asm.emit("JNZ", t2, done)
                xv = self.coerce(self.cx(body, self.bind(env, pat, Const(j)), ctx, base, t.elem), t.elem)
                self.movn(dst + 1 + (j - 1) * t.elem.size, xv.loc, t.elem.size)
            self.asm.emit("JMP", done)
            self.asm.label(ovf)
            self.asm.emit("TRAP", TRAP_OVERFLOW, n.line)
            self.asm.label(done)
            return Val(t, dst)
        if kind[0] != "const":
            raise CompileError("function constructor over a runtime domain is not supported")
        keys = sorted(kind[1], key=vkey)
        we = None
        if isinstance(want, TFun) and want.keys == tuple(keys):
            we = want.elem
        elif isinstance(want, TTuple) and tuple(keys) == tuple(range(1, len(want.elems) + 1)):
            we = None
        items = []
        for i, kv in enumerate(keys):
            w = we if we is not None else (want.elems[i] if isinstance(want, TTuple) and i < len(want.elems) else None)
            x = self.cx(body, self.bind(env, pat, Const(kv)), ctx, base, w)
            items.append(self.as_val(x, w))
        if isinstance(want, TTuple) and tuple(keys) == tuple(range(1, len(want.elems) + 1)):
            vals = [self.coerce(v, w) for v, w in zip(items, want.elems)]
            dst = self.alloc(want.size)
            for v, o in zip(vals, want.offs):
                self.movn(dst + o, v.loc, v.t.size)
            return Val(want, dst)
        et = we
        if et is None:
            et = TBottom()
            for v in items:
                et = join(et, v.t)
        n1 = len(keys)
        if n1 > 0 and all(type(kk) is int for kk in keys) and keys[0] == 1 and keys[-1] == n1 and we is None:
            t = TTuple([et] * n1)
        else:
            t = TFun(keys, et)
        dst = self.alloc(t.size)
        for j, v in enumerate(items):
            cv = self.coerce(v, et)
            self.movn(dst + j * et.size, cv.loc, et.size)
        return Val(t, dst)

    def key_index(self, ft: T, kx, n):
        """Index of key kx in function-like type ft: returns ('static', j) or ('dyn', reg)."""
        if isinstance(ft, TFun):
            if type(kx) is Const:
                j = ft.kindex.get(kx.v)
                if j is None:
                    return ("none", None)
                return ("static", j)
            keys = ft.keys
            if all(type(kk) is int for kk in keys) and list(keys) == list(range(keys[0], keys[0] + len(keys))):
                o = self.ord_in(TInt(keys[0], keys[-1]), kx)
            elif all(is_atom(kk) for kk in keys):
                o = self.ord_in(TAtom(keys), kx)
            else:
                raise CompileError("function with non-scalar keys indexed by a runtime value")
            return ("dyn", o)
        if isinstance(ft, TTuple):
            if type(kx) is Const:
                if type(kx.v) is int and 1 <= kx.v <= len(ft.elems):
                    return ("static", kx.v - 1)
                return ("none", None)
            if len(set(ft.elems)) > 1:
                raise CompileError("heterogeneous tuple indexed by a runtime value")
            o = self.ord_in(TInt(1, len(ft.elems)), kx)
            return ("dyn", o)
        raise CompileError(f"value of type {ft} is not a function")

    def _fcndef_target(self, fn, env, ctx, base):
        """fn names a function defined by  f[x \\in S] == e  (LET or module level): -> (fcndef node, env, ctx)."""
        if fn.k != "id":
            return None
        try:
            r = self.resolve(fn.a[0], env, ctx)
        except CompileError:
            return None
        if r[0] == "env" and type(r[1]) is Lazy and r[1].node.k == "fcndef":
            return r[1].node, r[1].env, r[1].ctx
        if r[0] == "env" and type(r[1]) is PVal and r[1].lazy.node.k == "fcndef":
            return r[1].lazy.node, r[1].lazy.env, r[1].lazy.ctx
        if r[0] == "def" and not r[1].params and r[1].body.k == "fcndef":
            return r[1].body, {}, r[2]
        return None

    def _share_recursive_apps(self, fname, body):
        """f[x \\in S] == ... f[e] ... f[e] ...: when the body applies f to the SAME argument expression more than once
        (WriteThroughCache.tla:117-123: THEN f[i-1] ELSE [f[i-1] EXCEPT ...]) wrap it as LET r == f[e] IN body[r/f[e]],
        so that unrolling the recursion is linear in the depth instead of 2^depth (the LET is evaluated once, with
        deferred traps, by the by-name binding logic)."""
        cache = self.__dict__.setdefault("_shared_rec_cache", {})
        hit = cache.get(id(body))
        if hit is not None:
            return hit[1]
        found = {}

        def key(x):
            if isinstance(x, Node):
                return (x.k,) + tuple(key(y) for y in x.a)
            if isinstance(x, (tuple, list)):
                return tuple(key(y) for y in x)
            if isinstance(x, OpDef):
                return ("opdef", x.name, key(x.body))
            return x

        def scan(x):
            if isinstance(x, Node):
                if x.k == "fapp" and x.a[0].k == "id" and x.a[0].a[0] == fname and len(x.a[1]) == 1:
                    found.setdefault(key(x.a[1][0]), []).append(x)
                for y in x.a:
                    scan(y)
            elif isinstance(x, (tuple, list)):
                for y in x:
                    scan(y)
        scan(body)
        shared = {k: v for k, v in found.items() if len(v) >= 2}
        out = body
        if shared:
            names = {}
            defs = []
            for i, (k, apps) in enumerate(shared.items()):
                nm = f"__rec{i}_{fname}"
                names[k] = nm
                defs.append(OpDef(nm, [], apps[0]))

            def subst(x):
                if isinstance(x, Node):
                    if x.k == "fapp" and x.a[0].k == "id" and x.a[0].a[0] == fname and len(x.a[1]) == 1:
                        nm = names.get(key(x.a[1][0]))
                        if nm is not None:
                            return Node("id", (nm,), x.line, x.col)
                    return Node(x.k, tuple(subst(y) for y in x.a), x.line, x.col)
                if isinstance(x, tuple):
                    return tuple(subst(y) for y in x)
                if isinstance(x, list):
                    return [subst(y) for y in x]
                return x
            out = Node("let", (tuple(defs), subst(body)), body.line, body.col)
        cache[id(body)] = (body, out)
        return out

    def x_fapp(self, n, env, ctx, base, want):
        fn, args = n.a
        tgt = self._fcndef_target(fn, env, ctx, base)
        if tgt is not None and self.try_const(fn, env, ctx, base) is None:
            # application of a (possibly recursive) function definition whose body depends on the state
            # (WriteThroughCache.tla:116-123 `vmem`: a fold over the memory queue): the body is inlined with the
            # bound variable := the argument, recursive applications unroll like RECURSIVE operators
            node, fenv, fctx = tgt
            _nm, bounds, body = node.a
            if len(bounds) == 1 and isinstance(bounds[0][0], str) and len(args) == 1:
                a = args[0]
                c = self.try_const(a, env, ctx, base)
                if c is not None:
                    arg = c
                else:
                    # evaluate the argument once and clamp its integer type to the function's domain lo..hi (an
                    # application outside the domain is an error in TLC): this is what ends the unrolling of
                    # f[i-1] after Len(q)+1 levels
                    arg = self.cx(a, env, ctx, base)
                    dn = bounds[0][1]
                    if isinstance(arg, Val) and isinstance(arg.t, TInt) and arg.t.lo is not None \
                            and dn is not None and dn.k == "bin" and dn.a[0] == "..":
                        try:
                            dlo = self.cx(dn.a[1], fenv, fctx, base)
                            dhi = self.cx(dn.a[2], fenv, fctx, base)
                            tl, th = self._int_t(dlo), self._int_t(dhi)
                            lo2 = max(arg.t.lo, tl.lo) if tl.lo is not None else arg.t.lo
                            hi2 = min(arg.t.hi, th.hi) if th.hi is not None else arg.t.hi
                            if lo2 > hi2:
                                self.asm.emit("TRAP", TRAP_EVAL, n.line)
                                return Val(want if want is not None else TBottom(), 0)
                            arg = Val(TInt(lo2, hi2), arg.loc)
                        except CompileError:
                            pass
                env2 = dict(fenv)
                env2[bounds[0][0]] = arg
                body = self._share_recursive_apps(fn.a[0], body)
                return self._inline(body, env2, fctx, base, want, n)
        f = self.cx(fn, env, ctx, base)
        if len(args) == 1:
            kx = self.cx(args[0], env, ctx, base)
        else:
            kx = self.cx(Node("tuple", (tuple(args),), n.line, n.col), env, ctx, base)
        if type(f) is Const:
            if type(kx) is Const:
                from ..front.values import fcn_apply
                return Const(fcn_apply(f.v, kx.v))
            f = self.as_val(f)
        ft = f.t
        if isinstance(ft, TBottom):
            return f
        if isinstance(ft, TSeq):
            return self.seq_index(f, kx, n)
        if isinstance(ft, TPFun):
            return self.pf_apply(f, kx, n)
        if isinstance(ft, TSparse) and ft.vt is not None:
            r = self.sp_find(f, kx)
            ok = Label("sak")
            self.asm.emit("JGEZ", r, ok)
            self.asm.emit("TRAP", TRAP_EVAL, n.line)
            self.asm.label(ok)
            ent = self.alloc(ft.stride)
            self.asm.emit("LDX", ent, f.loc + 1, r, ft.stride)
            return Val(ft.vt, ent + ft.keyw)
        if isinstance(ft, TSet) or not isinstance(ft, (TFun, TTuple)):
            raise CompileError(f"applying a non-function of type {ft} at line {n.line}")
        ki = self.key_index(ft, kx, n)
        if ki[0] == "none":
            self.asm.emit("TRAP", TRAP_EVAL, n.line)
            et = ft.elem if isinstance(ft, TFun) else ft.elems[0]
            return Val(et, f.loc)
        if ki[0] == "static":
            j = ki[1]
            if type(f) is OVal and isinstance(ft, TTuple):
                tabs = self._univ_tables(ft)
                et_ = ft.elems[j]
                dst = self.alloc(et_.size)
                for w in range(et_.size):
                    self.asm.emit("TBL", dst + w, tabs[ft.offs[j] + w], f.oreg)
                return Val(et_, dst)
            if isinstance(ft, TFun):
                return Val(ft.elem, f.loc + j * ft.elem.size)
            return Val(ft.elems[j], f.loc + ft.offs[j])
        o = ki[1]
        et = ft.elem if isinstance(ft, TFun) else ft.elems[0]
        if type(f) is OVal:
            f = Val(ft, f.loc)
        ok = Label("ak")
        bad = Label("ab")
        self.asm.emit("JNEG", o, bad)
        dst = self.alloc(et.size)
        self.asm.emit("LDX", dst, f.loc, o, et.size)
        self.asm.emit("JMP", ok)
        self.asm.label(bad)
        self.asm.emit("TRAP", TRAP_EVAL, n.line)
        self.asm.label(ok)
        return Val(et, dst)

    def x_except(self, n, env, ctx, base, want):
        fn, ups = n.a
        f = self.cx(fn, env, ctx, base, want)
        if isinstance(f, Val) and isinstance(f.t, TBottom):
            return f                    # value of an activation past the recursion bound (already trapped)
        f = self.as_val(f, want)
        if want is not None and f.t != want:
            f = self.coerce(f, want)
        dst = self.alloc(f.t.size)
        self.movn(dst, f.loc, f.t.size)
        cur = Val(f.t, dst)
        for path, valnode in ups:
            self._except_path(cur, path, 0, valnode, env, ctx, base, n)
        return cur

    def _except_path(self, cur: Val, path, i, valnode, env, ctx, base, n):
        """Update cur (a writable Val) in place at path[i:]."""
        if i == len(path):
            env2 = dict(env)
            env2["@"] = cur
            x = self.cx(valnode, env2, ctx, base, cur.t)
            xv = self.coerce(x, cur.t)
            self.movn(cur.loc, xv.loc, cur.t.size)
            return
        kind, p = path[i]
        t = cur.t
        if kind == "fld":
            if not isinstance(t, TRec) or p not in t.fields:
                raise CompileError(f"EXCEPT !.{p} on type {t}")
            self._except_path(Val(t.fields[p], cur.loc + t.off[p]), path, i + 1, valnode, env, ctx, base, n)
            return
        if len(p) == 1:
            kx = self.cx(p[0], env, ctx, base)
        else:
            kx = self.cx(Node("tuple", (tuple(p),)), env, ctx, base)
        if isinstance(t, TSparse) and t.vt is not None:
            r = self.sp_find(cur, kx)
            skip = Label("xs")
            self.asm.emit("JNEG", r, skip)
            ent = self.alloc(t.stride)
            self.asm.emit("LDX", ent, cur.loc + 1, r, t.stride)
            self._except_path(Val(t.vt, ent + t.keyw), path, i + 1, valnode, env, ctx, base, n)
            self.asm.emit("STX", cur.loc + 1, r, ent, t.stride)
            self.asm.label(skip)
            return
        if isinstance(t, TPFun):
            ki = self.pf_slot(cur, kx, n)
            if ki[0] == "none":
                return
            skip = Label("xs")
            if ki[0] == "static":
                b_ = cur.loc + ki[1] * t.stride
                self.asm.emit("JZ", b_, skip)
                self._except_path(Val(t.elem, b_ + 1), path, i + 1, valnode, env, ctx, base, n)
            else:
                o = ki[1]
                self.asm.emit("JNEG", o, skip)
                slot = self.alloc(t.stride)
                self.asm.emit("LDX", slot, cur.loc, o, t.stride)
                self.asm.emit("JZ", slot, skip)
                self._except_path(Val(t.elem, slot + 1), path, i + 1, valnode, env, ctx, base, n)
                self.asm.emit("STX", cur.loc, o, slot, t.stride)
            self.asm.label(skip)
            return
        if isinstance(t, TSeq):
            et = t.elem
            o = self.seq_index_reg(cur, kx, n, trap=False)
            skip = Label("xs")
            self.asm.emit("JNEG", o, skip)
            tmp = self.alloc(et.size)
            self.asm.emit("LDX", tmp, cur.loc + 1, o, et.size)
            self._except_path(Val(et, tmp), path, i + 1, valnode, env, ctx, base, n)
            self.asm.emit("STX", cur.loc + 1, o, tmp, et.size)
            self.asm.label(skip)
            return
        if not isinstance(t, (TFun, TTuple)):
            raise CompileError(f"EXCEPT on non-function type {t}")
        ki = self.key_index(t, kx, n)
        if ki[0] == "none":
            return
        if ki[0] == "static":
            j = ki[1]
            if isinstance(t, TFun):
                sub = Val(t.elem, cur.loc + j * t.elem.size)
            else:
                sub = Val(t.elems[j], cur.loc + t.offs[j])
            self._except_path(sub, path, i + 1, valnode, env, ctx, base, n)
            return
        o = ki[1]
        et = t.elem if isinstance(t, TFun) else t.elems[0]
        skip = Label("xs")
        self.asm.emit("JNEG", o, skip)
        tmp = self.alloc(et.size)
        self.asm.emit("LDX", tmp, cur.loc, o, et.size)
        self._except_path(Val(et, tmp), path, i + 1, valnode, env, ctx, base, n)
        self.asm.emit("STX", cur.loc, o, tmp, et.size)
        self.asm.label(skip)

    def _copy(self, v: Val):
        loc = self.alloc(v.t.size)
        self.movn(loc, v.loc, v.t.size)
        return loc

    def x_choose(self, n, env, ctx, base, want):
        pat, sn, body = n.a
        if sn is None:
            raise CompileError("unbounded CHOOSE")
        kind = self.set_elements(sn, env, ctx, base)
        if kind[0] == "const":
            t = want
            if t is None:
                t = TBottom()
                for v in kind[1]:
                    t = join(t, type_of_value(v, self.seq_cap))
        elif kind[0] == "val":
            t = kind[1].t.elem
        elif kind[0] == "sparse":
            t = kind[1].t.kt
        else:
            t = TInt()
        dst = self.alloc(t.size)
        end = Label("che")

        pat0 = pat
        if not isinstance(pat, str):
            pat = "__choose_elem"

        def each(env2):
            x = env2[pat]
            if pat0 is not pat:
                env2 = self.bind(env2, pat0, x)
            yes, no = Label("chy"), Label("chn")
            self.cc(body, env2, ctx, base, yes, no)
            self.asm.label(yes)
            xv = self.coerce(x, t) if isinstance(x, Val) else self.materialize(x, t)
            self.movn(dst, xv.loc, t.size)
            self.asm.emit("JMP", end)
            self.asm.label(no)
        self.for_each([(pat, sn)], env, ctx, base, each)
        self.asm.emit("TRAP", TRAP_CHOOSE, n.line)
        self.asm.label(end)
        return Val(t, dst)

    def x_domain(self, n, env, ctx, base, want):
        f = self.cx(n.a[0], env, ctx, base)
        if isinstance(f, Val) and isinstance(f.t, TSparse):
            return self.sp_keys(f)
        if isinstance(f, Val) and isinstance(f.t, TPFun):
            return self.pf_domain(f)
        if isinstance(f, Val) and isinstance(f.t, TFun):
            return Const(frozenset(f.t.keys))
        if isinstance(f, Val) and isinstance(f.t, TTuple):
            return Const(frozenset(range(1, len(f.t.elems) + 1)))
        if isinstance(f, Val) and isinstance(f.t, TSeq):
            t = TSet(TInt(1, f.t.cap))
            dst = self.alloc(t.size)
            self.asm.emit("ZERO", dst, t.size)
            # bits 0..len-1
            i = self.alloc(1)
            tmp = self.alloc(1)
            top, done = Label("dl"), Label("dd")
            self.li(i, 0)
            self.asm.label(top)
            self.asm.emit("LT", tmp, i, f.loc)
            self.asm.emit("JZ", tmp, done)
            self.asm.emit("BSET", dst, i)
            self.asm.emit("ADDI", i, i, 1)
            self.asm.emit("JMP", top)
            self.asm.label(done)
            return Val(t, dst)
        raise CompileError("DOMAIN of unsupported value")

    # ---------------------------------------------------------------- builtins
    def builtin(self, name, args, n, env, ctx, base, want):
        if name == "Cardinality":
            if args[0].k == "domain":
                f = self.cx(args[0].a[0], env, ctx, base)
                if isinstance(f, Val) and isinstance(f.t, TSparse):
                    return Val(TInt(0, f.t.cap), f.loc)
            s = self.cx(args[0], env, ctx, base)
            if isinstance(s, Val) and isinstance(s.t, TSparse):
                return Val(TInt(0, s.t.cap), s.loc)
            sv = self.as_val(s)
            dst = self.alloc(1)
            self.asm.emit("BCNT", dst, sv.loc, sv.t.size)
            return Val(TInt(0, sv.t.nbits), dst)
        if name == "Len":
            s = self.cx(args[0], env, ctx, base)
            if isinstance(s, Val) and isinstance(s.t, TSeq):
                return Val(TInt(0, s.t.cap), s.loc)
            if isinstance(s, Val) and isinstance(s.t, TTuple):
                return Const(len(s.t.elems))
            raise CompileError("Len of unsupported value")
        if name in ("Append", "Head", "Tail", "SubSeq", "SelectSeq"):
            return self.seq_builtin(name, args, n, env, ctx, base, want)
        if name in ("Assert", "Print", "PrintT"):
            return self._bool_value(n, env, ctx, base, want)
        if name == "IsFiniteSet":
            return Const(True)
        raise CompileError(f"builtin {name} is not supported on the device")

    # ------------------------------------------------ sparse containers / partial functions
    # TSparse values are built only through SINS (sorted insert), so they are canonical by construction.
    @staticmethod
    def sp_desc(t: TSparse):
        return (t.stride << 7) | t.keyw

    def sp_new(self, t: TSparse) -> Val:
        dst = self.alloc(t.size)
        self.asm.emit("ZERO", dst, t.size)
        return Val(t, dst)

    def sp_entry(self, t: TSparse, key, val=None):
        """Assemble one entry (key [, value]) of container type t in fresh temporaries."""
        e = self.alloc(t.stride)
        kv = self.coerce(key, t.kt)
        self.movn(e, kv.loc, t.keyw)
        if t.vt is not None:
            vv = self.coerce(val, t.vt)
            self.movn(e + t.keyw, vv.loc, t.vt.size)
        return e

    def sp_insert(self, cont: Val, eloc, line=0):
        t = cont.t
        st = self.alloc(1)
        self.li(st, t.cap)
        self.asm.emit("SINS", cont.loc, eloc, st, self.sp_desc(t))
        ok = Label("sio")
        self.asm.emit("JNZ", st, ok)
        self.asm.emit("TRAP", TRAP_OVERFLOW, line)
        self.asm.label(ok)

    def sp_find(self, cont: Val, key):
        """-> register holding the entry index of key in cont, or -1."""
        t = cont.t
        try:
            kv = self.coerce(key, t.kt)
        except CompileError:
            r = self.alloc(1)
            self.li(r, -1)
            return r
        r = self.alloc(1)
        self.asm.emit("SFIND", r, cont.loc, kv.loc, self.sp_desc(t))
        return r

    def sp_loop(self, cont: Val, body):
        """for each entry of cont: body(key Val, value Val | None) on a private copy of the entry."""
        t = cont.t
        i = self.alloc(1)
        n = self.alloc(1)
        e = self.alloc(t.stride)
        self.li(i, -1)
        self.asm.emit("MOV", n, cont.loc)
        top, done = Label("spl"), Label("spd")
        self.asm.label(top)
        self.asm.emit("ADDI", i, i, 1)
        tmp = self.alloc(1)
        self.asm.emit("LT", tmp, i, n)
        self.asm.emit("JZ", tmp, done)
        self.asm.emit("LDX", e, cont.loc + 1, i, t.stride)
        body(Val(t.kt, e), Val(t.vt, e + t.keyw) if t.vt is not None else None)
        self.asm.emit("JMP", top)
        self.asm.label(done)

    def sp_copy(self, x, t: TSparse) -> Val:
        xv = self.coerce(x, t)
        dst = self.alloc(t.size)
        self.movn(dst, xv.loc, t.size)
        return Val(t, dst)

    def sp_keys(self, f: Val) -> Val:
        """DOMAIN of a sparse function as a sparse set (same order, so a strided copy)."""
        t = f.t
        if t.vt is None:
            return f
        kt = TSparse(t.kt, None, t.cap)
        dst = self.alloc(kt.size)
        self.asm.emit("MOV", dst, f.loc)
        for j in range(t.cap):
            self.movn(dst + 1 + j * t.keyw, f.loc + 1 + j * t.stride, t.keyw)
        return Val(kt, dst)

    def sp_setop(self, op, a, b, t: TSparse, line=0) -> Val:
        if op == "\\cup":
            dst = self.sp_copy(a, t)
            bv = self.coerce(b, t)
            self.sp_loop(bv, lambda k, v: self.sp_insert(dst, k.loc, line))
            return dst
        av = self.coerce(a, t)
        bv = self.coerce(b, t)
        dst = self.sp_new(t)

        def each(k, v):
            r = self.sp_find(bv, k)
            skip = Label("sps")
            self.asm.emit("JGEZ" if op == "\\" else "JNEG", r, skip)
            self.sp_insert(dst, k.loc, line)
            self.asm.label(skip)
        self.sp_loop(av, each)
        return dst

    def pf_slot(self, f: Val, kx, n):
        """Index register / static index of key kx in partial function f (TPFun)."""
        t = f.t
        return self.key_index(TFun(t.keys, TBool()), kx, n)

    def pf_apply(self, f: Val, kx, n) -> Val:
        t = f.t
        ki = self.pf_slot(f, kx, n)
        if ki[0] == "none":
            self.asm.emit("TRAP", TRAP_EVAL, n.line)
            return Val(t.elem, f.loc + 1)
        ok = Label("pfo")
        if ki[0] == "static":
            base_ = f.loc + ki[1] * t.stride
            self.asm.emit("JNZ", base_, ok)
            self.asm.emit("TRAP", TRAP_EVAL, n.line)
            self.asm.label(ok)
            return Val(t.elem, base_ + 1)
        o = ki[1]
        bad = Label("pfb")
        self.asm.emit("JNEG", o, bad)
        slot = self.alloc(t.stride)
        self.asm.emit("LDX", slot, f.loc, o, t.stride)
        self.asm.emit("JNZ", slot, ok)
        self.asm.label(bad)
        self.asm.emit("TRAP", TRAP_EVAL, n.line)
        self.asm.label(ok)
        return Val(t.elem, slot + 1)

    def pf_domain(self, f: Val) -> Val:
        t = f.t
        st = TSet(self._key_type(t.keys))
        dst = self.alloc(st.size)
        self.asm.emit("ZERO", dst, st.size)
        for j, k in enumerate(t.keys):
            o = self.codec.ord_of(st.elem, k)
            skip = Label("pds")
            self.asm.emit("JZ", f.loc + j * t.stride, skip)
            self.asm.emit("BSETI", dst, o)
            self.asm.label(skip)
        return Val(st, dst)

    @staticmethod
    def _key_type(keys):
        if all(type(k) is int for k in keys):
            return TInt(min(keys), max(keys))
        if all(is_atom(k) for k in keys):
            return TAtom(sorted(keys, key=vkey))
        raise CompileError("partial function with non-scalar keys")

    def fcn_merge(self, ln, rn, env, ctx, base, want, n):
        """a @@ b  (a's entries win) for sparse / partial functions; b is usually `k :> v`."""
        a = self.cx(ln, env, ctx, base, want)
        t = want if isinstance(want, (TSparse, TPFun)) else (a.t if isinstance(a, Val) else None)
        if not isinstance(t, (TSparse, TPFun)):
            raise CompileError(f"@@ is supported for functions with a dynamic domain only (line {n.line})")
        pairs = None
        if rn.k == "bin" and rn.a[0] == ":>":
            pairs = [(rn.a[1], rn.a[2])]
        if isinstance(t, TSparse):
            dst = self.sp_copy(a, t)
            if pairs is not None:
                for kn, vn in pairs:
                    k = self.cx(kn, env, ctx, base, t.kt)
                    r = self.sp_find(dst, k)
                    skip = Label("mgs")
                    self.asm.emit("JGEZ", r, skip)
                    v = self.cx(vn, env, ctx, base, t.vt)
                    self.sp_insert(dst, self.sp_entry(t, k, v), n.line)
                    self.asm.label(skip)
                return dst
            bv = self.coerce(self.cx(rn, env, ctx, base, t), t)

            def each(k, v):
                r = self.sp_find(dst, k)
                skip = Label("mgs")
                self.asm.emit("JGEZ", r, skip)
                self.sp_insert(dst, k.loc, n.line)
                self.asm.label(skip)
            self.sp_loop(bv, each)
            return dst
        av = self.coerce(a, t)
        dst = Val(t, self._copy(av))
        if pairs is None:
            bv = self.coerce(self.cx(rn, env, ctx, base, t), t)
            for j in range(len(t.keys)):
                skip = Label("mgp")
                self.asm.emit("JNZ", dst.loc + j * t.stride, skip)
                self.movn(dst.loc + j * t.stride, bv.loc + j * t.stride, t.stride)
                self.asm.label(skip)
            return dst
        for kn, vn in pairs:
            k = self.cx(kn, env, ctx, base)
            ki = self.pf_slot(dst, k, n)
            if ki[0] == "none":
                self.asm.emit("TRAP", TRAP_OVERFLOW, n.line)
                continue
            v = self.cx(vn, env, ctx, base, t.elem)
            slot = self.alloc(t.stride)
            self.li(slot, 1)
            vv = self.coerce(v, t.elem)
            self.movn(slot + 1, vv.loc, t.elem.size)
            skip = Label("mgp")
            if ki[0] == "static":
                b_ = dst.loc + ki[1] * t.stride
                self.asm.emit("JNZ", b_, skip)
                self.movn(b_, slot, t.stride)
            else:
                o = ki[1]
                bad, go = Label("mgb"), Label("mgg")
                self.asm.emit("JGEZ", o, go)
                self.asm.label(bad)
                self.asm.emit("TRAP", TRAP_OVERFLOW, n.line)
                self.asm.label(go)
                cur = self.alloc(t.stride)
                self.asm.emit("LDX", cur, dst.loc, o, t.stride)
                self.asm.emit("JNZ", cur, skip)
                self.asm.emit("STX", dst.loc, o, slot, t.stride)
            self.asm.label(skip)
        return dst

    # --------------------------------------------------------------- sequences
    def _as_seq(self, x, want=None) -> Val:
        if type(x) is Const:
            if want is None:
                if not isinstance(x.v, tuple):
                    raise CompileError("constant sequence without an expected type")
                et = TBottom()
                for e in x.v:
                    et = join(et, self.natural_type(e))
                if isinstance(et, TBottom):
                    raise CompileError("empty constant sequence without an expected type")
                want = TSeq(self._widen_elem(et), max(len(x.v), self.seq_cap or len(x.v) + 8))
            return self.materialize(x, want)
        if isinstance(x.t, TSeq):
            return x
        if isinstance(x.t, TTuple):
            if isinstance(want, TSeq):
                return self.coerce(x, want)
            et = TBottom()
            for e in x.t.elems:
                et = join(et, e)
            cap = max(len(x.t.elems), self.seq_cap or len(x.t.elems))
            return self.coerce(x, TSeq(et, cap))
        raise CompileError(f"sequence expected, got {x.t}")

    def _widen_elem(self, t):
        """Element type for a sequence that starts from constants and grows at run time."""
        if isinstance(t, TAtom):
            mv = any(isinstance(a, ModelValue) for a in t.atoms)
            pool = self.all_mvs if mv else self.all_strings
            return TAtom(sorted(set(pool) | set(t.atoms), key=vkey))
        if isinstance(t, TInt):
            return TInt()
        return t

    def seq_index_reg(self, s: Val, kx, n, trap=True):
        kv = self.as_val(kx, TInt())
        o = self.alloc(1)
        t1 = self.alloc(1)
        ok, bad = Label("sik"), Label("sib")
        self.asm.emit("ADDI", o, kv.loc, -1)
        self.asm.emit("JNEG", o, bad)
        self.asm.emit("LT", t1, o, s.loc)
        self.asm.emit("JNZ", t1, ok)
        self.asm.label(bad)
        if trap:
            self.asm.emit("TRAP", TRAP_EVAL, n.line)
        self.li(o, -1)
        self.asm.label(ok)
        return o

    def seq_index(self, s: Val, kx, n):
        o = self.seq_index_reg(s, kx, n)
        et = s.t.elem
        dst = self.alloc(et.size)
        self.asm.emit("LDX", dst, s.loc + 1, o, et.size)
        return Val(et, dst)

    def seq_builtin(self, name, args, n, env, ctx, base, want):
        if name == "Append":
            s = self._as_seq(self.cx(args[0], env, ctx, base, want), want if isinstance(want, TSeq) else None)
            t = want if isinstance(want, TSeq) else s.t
            s = self.coerce(s, t)
            e = self.coerce(self.cx(args[1], env, ctx, base, t.elem), t.elem)
            dst = self.alloc(t.size)
            self.movn(dst, s.loc, t.size)
            t1 = self.alloc(1)
            ok = Label("apk")
            self.asm.emit("LTI", t1, dst, t.cap)
            self.asm.emit("JNZ", t1, ok)
            self.asm.emit("TRAP", TRAP_OVERFLOW, n.line)
            self.asm.label(ok)
            self.asm.emit("STX", dst + 1, dst, e.loc, t.elem.size)
            self.asm.emit("ADDI", dst, dst, 1)
            return Val(t, dst)
        if name == "Head":
            s = self._as_seq(self.cx(args[0], env, ctx, base))
            return self.seq_index(s, Const(1), n)
        if name == "Tail":
            s = self._as_seq(self.cx(args[0], env, ctx, base, want), want if isinstance(want, TSeq) else None)
            t = s.t
            es = t.elem.size
            dst = self.alloc(t.size)
            ok = Label("tlk")
            t1 = self.alloc(1)
            self.asm.emit("GTI", t1, s.loc, 0)
            self.asm.emit("JNZ", t1, ok)
            self.asm.emit("TRAP", TRAP_EVAL, n.line)
            self.asm.label(ok)
            self.asm.emit("ZERO", dst, t.size)
            self.asm.emit("ADDI", dst, s.loc, -1)
            if t.cap > 1:
                self.movn(dst + 1, s.loc + 1 + es, (t.cap - 1) * es)
            r = Val(t, dst)
            return r
        if name == "SelectSeq":
            s = self._as_seq(self.cx(args[0], env, ctx, base, want), want if isinstance(want, TSeq) else None)
            t = s.t
            es = t.elem.size
            test = self.op_value(args[1], env, ctx)
            dst = self.alloc(t.size)
            self.asm.emit("ZERO", dst, t.size)
            i = self.alloc(1)
            t1 = self.alloc(1)
            ev = self.alloc(es)
            top, done = Label("sel"), Label("sed")
            self.li(i, 0)
            self.asm.label(top)
            self.asm.emit("LT", t1, i, s.loc)
            self.asm.emit("JZ", t1, done)
            self.asm.emit("LDX", ev, s.loc + 1, i, es)
            self.asm.emit("ADDI", i, i, 1)
            env2 = dict(test.env)
            env2[test.params[0][0]] = Val(t.elem, ev)
            m0 = self.mark()
            yes = Label("sey")
            self.cc(test.body, env2, test.ctx, base, yes, top)
            self.asm.label(yes)
            self.asm.emit("STX", dst + 1, dst, ev, es)
            self.asm.emit("ADDI", dst, dst, 1)
            self.release(m0)
            self.asm.emit("JMP", top)
            self.asm.label(done)
            return Val(t, dst)
        if name == "SubSeq":
            s = self._as_seq(self.cx(args[0], env, ctx, base))
            t = want if isinstance(want, TSeq) and want.elem == s.t.elem else s.t
            es = t.elem.size
            lo = self.as_val(self.cx(args[1], env, ctx, base), TInt())
            hi = self.as_val(self.cx(args[2], env, ctx, base), TInt())
            dst = self.alloc(t.size)
            self.asm.emit("ZERO", dst, t.size)
            i = self.alloc(1)
            hi_s = self.alloc(1)
            t1 = self.alloc(1)
            tmp = self.alloc(es)
            top, done, bad, ok = Label("ssl"), Label("ssd"), Label("ssb"), Label("ssk")
            self.asm.emit("MOV", i, lo.loc)
            self.asm.emit("MOV", hi_s, hi.loc)
            self.asm.label(top)
            self.asm.emit("LE", t1, i, hi_s)
            self.asm.emit("JZ", t1, done)
            self.asm.emit("LTI", t1, i, 1)
            self.asm.emit("JNZ", t1, bad)
            self.asm.emit("LE", t1, i, s.loc)
            self.asm.emit("JZ", t1, bad)
            self.asm.emit("LTI", t1, dst, t.cap)
            self.asm.emit("JNZ", t1, ok)
            self.asm.emit("TRAP", TRAP_OVERFLOW, n.line)
            self.asm.label(bad)
            self.asm.emit("TRAP", TRAP_EVAL, n.line)
            self.asm.label(ok)
            self.asm.emit("ADDI", t1, i, -1)
            self.asm.emit("LDX", tmp, s.loc + 1, t1, es)
            self.asm.emit("STX", dst + 1, dst, tmp, es)
            self.asm.emit("ADDI", dst, dst, 1)
            self.asm.emit("ADDI", i, i, 1)
            self.asm.emit("JMP", top)
            self.asm.label(done)
            return Val(t, dst)
        raise CompileError(f"sequence operator {name} is not supported on the device yet")

    def seq_concat(self, ln, rn, env, ctx, base, want):
        a = self._as_seq(self.cx(ln, env, ctx, base, want), want if isinstance(want, TSeq) else None)
        t = want if isinstance(want, TSeq) else a.t
        a = self.coerce(a, t)
        bx = self.cx(rn, env, ctx, base, t)
        b = self.coerce(self._as_seq(bx, t), t)
        es = t.elem.size
        dst = self.alloc(t.size)
        self.movn(dst, a.loc, t.size)
        i = self.alloc(1)
        t1 = self.alloc(1)
        tmp = self.alloc(es)
        top, done, ok = Label("ccl"), Label("ccd"), Label("cck")
        self.li(i, 0)
        self.asm.label(top)
        self.asm.emit("LT", t1, i, b.loc)
        self.asm.emit("JZ", t1, done)
        self.asm.emit("LTI", t1, dst, t.cap)
        self.asm.emit("JNZ", t1, ok)
        self.asm.emit("TRAP", TRAP_OVERFLOW, 0)
        self.asm.label(ok)
        self.asm.emit("LDX", tmp, b.loc + 1, i, es)
        self.asm.emit("STX", dst + 1, dst, tmp, es)
        self.asm.emit("ADDI", dst, dst, 1)
        self.asm.emit("ADDI", i, i, 1)
        self.asm.emit("JMP", top)
        self.asm.label(done)
        return Val(t, dst)

    # ------------------------------------------- compile-time masks over set universes
    @staticmethod
    def flat_and(n):
        if n.k == "and":
            out = []
            for x in n.a[0]:
                out += Lowering.flat_and(x)
            return out
        return [n]

    def elem_truth(self, E, pat, c, env, ctx, base, alive):
        """Evaluate predicate c at compile time for every universe ordinal in `alive` (element bound
        to `pat`).  Returns the list of ordinals where it is TRUE, or None if c depends on run-time
        values (or fails to evaluate) for any of them."""
        vals = self._enum_cached(E)
        keep = []
        for o in alive:
            env2 = dict(env)
            env2[pat] = Const(vals[o])
            r = self.try_const(c, env2, ctx, base)
            if r is None or type(r.v) is not bool:
                return None
            if r.v:
                keep.append(o)
        return keep

    def _enum_cached(self, E):
        cache = self.__dict__.setdefault("_enum_cache", {})
        v = cache.get(E)
        if v is None:
            v = cache[E] = self.codec.enum(E)
        return v

    def mask_words(self, E, ordinals, invert=False):
        n = E.card()
        words = [0] * max(1, (n + 31) // 32)
        s = set(ordinals)
        for o in range(n):
            if (o in s) != invert:
                words[o >> 5] |= 1 << (o & 31)
        return [w - (1 << 32) if w >= (1 << 31) else w for w in words]

    def narrow(self, sv: Val, pat, items, env, ctx, base):
        """Fold the element-only conjuncts of `items` (predicates over the bound element and constants,
        e.g. m.type = "1b" /\\ m.bal = b with b unrolled) into a constant bitmask over the universe:
        returns (sv AND mask, remaining conjuncts).  Conjuncts are tried in order on the elements that
        survive the earlier ones, so guards like `m.type = "1b" /\\ m.acc \\in Q` keep their meaning."""
        E = sv.t.elem
        if not isinstance(pat, str) or isinstance(E, TBottom) or E.card() > 4096:
            return sv, items
        alive = list(getattr(sv, "alive", None) or range(E.card()))
        rest, masked = [], False
        for c in items:
            keep = self.elem_truth(E, pat, c, env, ctx, base, alive)
            if keep is None:
                rest.append(c)
            else:
                alive, masked = keep, True
        if not masked:
            return sv, items
        dst = self.alloc(sv.t.size)
        words = self.mask_words(E, alive)
        base = self.asm.const_table(words)
        if base < (1 << 19) and sv.t.size < 256:
            self.asm.emit("BANDC", dst, sv.loc, (base << 8) | sv.t.size)
        else:
            mloc = self.alloc(sv.t.size)
            self.load_words(mloc, words)
            self.asm.emit("BAND", dst, sv.loc, mloc, sv.t.size)
        return MVal(sv.t, dst, alive), rest

    def forall_val(self, sv: Val, pat, P, env, ctx, base, lf):
        """Emit code for  \\A pat \\in sv : P  -- jumps to lf when violated, falls through when it holds."""
        E = sv.t.elem
        if P.k == "and" and len(P.a[0]) > 1:
            for x in P.a[0]:
                self.forall_val(sv, pat, x, env, ctx, base, lf)
            return
        if P.k == "and":
            P = P.a[0][0]
        if P.k == "bin" and P.a[0] == "=>":
            sv2, rest = self.narrow(sv, pat, self.flat_and(P.a[1]), env, ctx, base)
            if sv2 is not sv:
                if rest:
                    ante = rest[0] if len(rest) == 1 else Node("and", (tuple(rest),), P.line, P.col)
                    P2 = Node("bin", ("=>", ante, P.a[2]), P.line, P.col)
                    self._forall_loop(sv2, pat, P2, env, ctx, base, lf)
                else:
                    self.forall_val(sv2, pat, P.a[2], env, ctx, base, lf)
                return
        if E.card() <= 4096:
            keep = self.elem_truth(E, pat, P, env, ctx, base, list(range(E.card())))
            if keep is not None:
                mloc = self.alloc(sv.t.size)
                self.load_words(mloc, self.mask_words(E, keep))
                t1 = self.alloc(1)
                self.asm.emit("BSUB", t1, sv.loc, mloc, sv.t.size)
                self.asm.emit("JZ", t1, lf)
                return
        self._forall_loop(sv, pat, P, env, ctx, base, lf)

    def _forall_loop(self, sv, pat, P, env, ctx, base, lf):
        def each(xv):
            nxt = Label("fa")
            self.cc(P, self.bind(env, pat, xv), ctx, base, nxt, lf)
            self.asm.label(nxt)
        self.loop_set(sv, each)

    # ------------------------------------------------------------- conditions
    def cc(self, n: Node, env, ctx, base, lt: Label, lf: Label):
        """Compile n in control context: jump to lt if TRUE else lf.  Falls through to neither.
        All temporaries are dead once control has left, so the frame is released on exit."""
        mk = self.mark()
        try:
            self._cc(n, env, ctx, base, lt, lf)
        finally:
            self.release(mk)

    def _cc(self, n: Node, env, ctx, base, lt: Label, lf: Label):
        if n.line:
            self.asm.cur_line = n.line
        c = self.try_const(n, env, ctx, base)
        if c is not None:
            if c.v is True:
                self.asm.emit("JMP", lt)
            elif c.v is False:
                self.asm.emit("JMP", lf)
            else:
                raise CompileError(f"BOOLEAN expected at line {n.line}, got {fmt(c.v)}")
            return
        k = n.k
        if k == "and":
            items = n.a[0]
            for x in items[:-1]:
                nxt = Label("an")
                self.cc(x, env, ctx, base, nxt, lf)
                self.asm.label(nxt)
            self.cc(items[-1], env, ctx, base, lt, lf)
            return
        if k == "or":
            items = n.a[0]
            for x in items[:-1]:
                nxt = Label("on")
                self.cc(x, env, ctx, base, lt, nxt)
                self.asm.label(nxt)
            self.cc(items[-1], env, ctx, base, lt, lf)
            return
        if k == "not":
            self.cc(n.a[0], env, ctx, base, lf, lt)
            return
        if k == "if":
            c1 = self.try_const(n.a[0], env, ctx, base)
            if c1 is not None:
                self.cc(n.a[1] if c1.v else n.a[2], env, ctx, base, lt, lf)
                return
            a, b = Label("cit"), Label("cif")
            self.cc(n.a[0], env, ctx, base, a, b)
            self.asm.label(a)
            self.cc(n.a[1], env, ctx, base, lt, lf)
            self.asm.label(b)
            self.cc(n.a[2], env, ctx, base, lt, lf)
            return
        if k == "case":
            arms, other = n.a
            node = other if other is not None else Node("app", ("__trap_case", ()), n.line, n.col)
            for c2, e in reversed(arms):
                node = Node("if", (c2, e, node), n.line, n.col)
            self.cc(node, env, ctx, base, lt, lf)
            return
        if k == "let":
            self.cc(n.a[1], self.let_env(n.a[0], env, ctx, base, n.a[1]), ctx, base, lt, lf)
            return
        if k == "prime":
            self.cc(n.a[0], env, ctx, "P", lt, lf)
            return
        if k == "unchanged":
            self.cc_eq(Node("prime", (n.a[0],), n.line, n.col), n.a[0], env, ctx, base, lt, lf, n)
            return
        if k == "forall" or k == "exists":
            bounds, body = n.a
            is_all = k == "forall"
            if len(bounds) == 1 and isinstance(bounds[0][0], str) and bounds[0][1] is not None:
                kind = self.set_elements(bounds[0][1], env, ctx, base)
                if kind[0] == "val" and not isinstance(kind[1].t.elem, TBottom):
                    pat, sv = bounds[0][0], kind[1]
                    if is_all:
                        self.forall_val(sv, pat, body, env, ctx, base, lf)
                        self.asm.emit("JMP", lt)
                    else:
                        sv2, rest = self.narrow(sv, pat, self.flat_and(body), env, ctx, base)
                        if not rest:
                            t1 = self.alloc(1)
                            self.asm.emit("BISZ", t1, sv2.loc, sv2.t.size)
                            self.asm.emit("JZ", t1, lt)
                            self.asm.emit("JMP", lf)
                        else:
                            body2 = rest[0] if len(rest) == 1 else Node("and", (tuple(rest),), body.line, body.col)

                            def each1(xv):
                                nxt = Label("qn")
                                self.cc(body2, self.bind(env, pat, xv), ctx, base, lt, nxt)
                                self.asm.label(nxt)
                            self.loop_set(sv2, each1)
                            self.asm.emit("JMP", lf)
                    return

            def each(env2):
                nxt = Label("qn")
                if is_all:
                    self.cc(body, env2, ctx, base, nxt, lf)
                else:
                    self.cc(body, env2, ctx, base, lt, nxt)
                self.asm.label(nxt)
            self.for_each(bounds, env, ctx, base, each)
            self.asm.emit("JMP", lt if is_all else lf)
            return
        if k == "bin":
            op, ln, rn = n.a
            if op == "=>":
                nxt = Label("im")
                self.cc(ln, env, ctx, base, nxt, lt)
                self.asm.label(nxt)
                self.cc(rn, env, ctx, base, lt, lf)
                return
            if op == "<=>":
                a = self.as_val(self.cx(ln, env, ctx, base), TBool())
                b = self.as_val(self.cx(rn, env, ctx, base), TBool())
                t1 = self.alloc(1)
                self.asm.emit("EQ", t1, a.loc, b.loc)
                self.asm.emit("JNZ", t1, lt)
                self.asm.emit("JMP", lf)
                return
            if op in ("=", "#"):
                self.cc_eq(ln, rn, env, ctx, base, lt if op == "=" else lf, lf if op == "=" else lt, n)
                return
            if op in ("<", ">", "<=", ">="):
                a = self.cx(ln, env, ctx, base)
                b = self.cx(rn, env, ctx, base)
                self._int_t(a)
                self._int_t(b)
                t1 = self.alloc(1)
                if type(b) is Const and IMM28_MIN < b.v < IMM28_MAX:
                    av = self.as_val(a, TInt())
                    self.asm.emit({"<": "LTI", ">": "GTI", "<=": "LEI", ">=": "GEI"}[op], t1, av.loc, b.v)
                else:
                    av, bv = self.as_val(a, TInt()), self.as_val(b, TInt())
                    if op == "<":
                        self.asm.emit("LT", t1, av.loc, bv.loc)
                    elif op == "<=":
                        self.asm.emit("LE", t1, av.loc, bv.loc)
                    elif op == ">":
                        self.asm.emit("LT", t1, bv.loc, av.loc)
                    else:
                        self.asm.emit("LE", t1, bv.loc, av.loc)
                self.asm.emit("JNZ", t1, lt)
                self.asm.emit("JMP", lf)
                return
            if op in ("\\in", "\\notin"):
                self.cc_in(ln, rn, env, ctx, base, lt if op == "\\in" else lf, lf if op == "\\in" else lt, n)
                return
            if op in ("\\subseteq", "\\supseteq"):
                if op == "\\supseteq":
                    ln, rn = rn, ln
                self.cc_subseteq(ln, rn, env, ctx, base, lt, lf, n)
                return
        if k == "app" and n.a[0] == "Assert":
            r = self.resolve("Assert", env, ctx)
            if r[0] == "builtin":
                cond, msg = n.a[1]
                ok, bad = Label("ask"), Label("asb")
                self.cc(cond, env, ctx, base, ok, bad)
                self.asm.label(bad)
                mc = self.try_const(msg, env, ctx, base)
                self.asserts.append((mc.v if mc is not None else "<non-constant message>", n.loc()))
                self.asm.emit("ASSERTF", len(self.asserts) - 1)
                self.asm.emit("JMP", lf)
                self.asm.label(ok)
                self.asm.emit("JMP", lt)
                return
        if k == "app" and n.a[0] in ("Print", "PrintT") and self.resolve(n.a[0], env, ctx)[0] == "builtin":
            # printing from the device is not supported; the value of Print(out, v) is v / TRUE
            if n.a[0] == "PrintT":
                self.asm.emit("JMP", lt)
            else:
                self.cc(n.a[1][1], env, ctx, base, lt, lf)
            return
        if k == "app" and n.a[0] == "__trap_case":
            self.asm.emit("TRAP", TRAP_CASE, n.line)
            self.asm.emit("JMP", lf)
            return
        if k == "app" and self.use_subs:
            try:
                r = self.resolve(n.a[0], env, ctx)
            except CompileError:
                r = None
            if r is not None and r[0] == "def" and len(r[1].params) == len(n.a[1]):
                v = self._sub_call(r[1], r[2], n.a[1], env, ctx, base, TBool(), n)
                if v is not None:
                    if type(v) is Const:
                        self.asm.emit("JMP", lt if v.v is True else lf)
                    else:
                        self.asm.emit("JNZ", v.loc, lt)
                        self.asm.emit("JMP", lf)
                    return
        if k in ("id", "app", "sel"):
            # expand user operators in control context (keeps short-circuiting)
            tgt = self._expand(n, env, ctx, base)
            if tgt is not None:
                node2, env2, ctx2, base2 = tgt
                self.cc(node2, env2, ctx2, base2, lt, lf)
                return
        v = self.cx(n, env, ctx, base)
        if type(v) is Const:
            self.asm.emit("JMP", lt if v.v is True else lf)
            return
        if not isinstance(v.t, TBool):
            raise CompileError(f"BOOLEAN expected at line {n.line} col {n.col}, got {v.t}")
        self.asm.emit("JNZ", v.loc, lt)
        self.asm.emit("JMP", lf)

    def _expand(self, n, env, ctx, base):
        """If n is a reference to a user operator / LET definition return (body, env, ctx, base)."""
        if n.k == "sel":
            r = self.ev.resolve_sel(n.a[0], self.eval_env(env), Fr(ctx))
            if r[0] == "def":
                _, od, dctx, args = r
                return (od.body, self.bind_args(od.params, args, env, ctx, base, od.body), dctx, base)
            if r[0] == "expr":
                _, node, dctx, (od, args) = r
                return (node, self.bind_args(od.params, args, env, ctx, base), dctx, base)
            return None
        name = n.a[0]
        args = n.a[1] if n.k == "app" else ()
        try:
            r = self.resolve(name, env, ctx)
        except CompileError:
            return None
        if r[0] == "env":
            x = r[1]
            if type(x) is Lazy and not args:
                return (x.node, x.env, x.ctx, x.base if x.base == "P" else base)
            if type(x) is OpC:
                env2 = dict(x.env)
                env2.update(self.bind_args(x.params, args, env, ctx, base, x.body))
                return (x.body, env2, x.ctx, base)
            return None
        if r[0] == "def":
            d = r[1]
            if len(d.params) != len(args):
                raise CompileError(f"arity mismatch calling {name}")
            return (d.body, self.bind_args(d.params, args, env, ctx, base, d.body), r[2], base)
        if r[0] == "subst" and not args:
            return (r[1], {}, r[2], base)
        return None

    def cc_eq(self, ln, rn, env, ctx, base, lt, lf, n):
        a = self.cx(ln, env, ctx, base)
        b = self.cx(rn, env, ctx, base, a.t if isinstance(a, Val) else None)
        if type(a) is Const and isinstance(b, Val):
            a, b = b, a
        if type(a) is Const:
            from ..front.values import values_equal
            self.asm.emit("JMP", lt if values_equal(a.v, b.v) else lf)
            return
        t1 = self.alloc(1)
        if type(b) is Const:
            if a.t.scalar:
                if isinstance(a.t, TInt) and type(b.v) is int and a.t.lo is not None:
                    if not (a.t.lo <= b.v <= a.t.hi):
                        self.asm.emit("JMP", lf)        # outside the static range of a
                        return
                    if a.t.lo == a.t.hi:
                        self.asm.emit("JMP", lt)
                        return
                if isinstance(a.t, TInt) and type(b.v) is int and IMM28_MIN < b.v < IMM28_MAX:
                    self.asm.emit("EQI", t1, a.loc, b.v)
                elif isinstance(a.t, TAtom) and is_atom(b.v):
                    self.asm.emit("EQI", t1, a.loc, self.atoms.id(b.v))
                elif isinstance(a.t, TBool) and type(b.v) is bool:
                    self.asm.emit("EQI", t1, a.loc, int(b.v))
                else:
                    self.asm.emit("JMP", lf)
                    return
                self.asm.emit("JNZ", t1, lt)
                self.asm.emit("JMP", lf)
                return
            if isinstance(a.t, TSet) and isinstance(b.v, frozenset) and len(b.v) == 0:
                self.asm.emit("BISZ", t1, a.loc, a.t.size)
                self.asm.emit("JNZ", t1, lt)
                self.asm.emit("JMP", lf)
                return
            try:
                tj = join(a.t, self.natural_type(b.v))
            except TypeErr:
                self.asm.emit("JMP", lf)
                return
            av = self.coerce(a, tj)
            bv = self.materialize(b, tj)
        else:
            try:
                tj = join(a.t, b.t)
            except TypeErr:
                self.asm.emit("JMP", lf)
                return
            av = self.coerce(a, tj)
            bv = self.coerce(b, tj)
        if tj.size == 1:
            self.asm.emit("EQ", t1, av.loc, bv.loc)
        else:
            self.asm.emit("EQN", t1, av.loc, bv.loc, tj.size)
        self.asm.emit("JNZ", t1, lt)
        self.asm.emit("JMP", lf)

    def cc_in(self, en, sn, env, ctx, base, lt, lf, n):
        # structural set expressions first (avoid materialising big sets)
        sc = self.try_const(sn, env, ctx, base)
        if sc is None:
            if sn.k == "subset":
                self.cc_subseteq(en, sn.a[0], env, ctx, base, lt, lf, n)
                return
            if sn.k == "bin" and sn.a[0] == "\\cup":
                nxt = Label("iu")
                self.cc_in(en, sn.a[1], env, ctx, base, lt, nxt, n)
                self.asm.label(nxt)
                self.cc_in(en, sn.a[2], env, ctx, base, lt, lf, n)
                return
            if sn.k == "bin" and sn.a[0] == "\\cap":
                nxt = Label("ic")
                self.cc_in(en, sn.a[1], env, ctx, base, nxt, lf, n)
                self.asm.label(nxt)
                self.cc_in(en, sn.a[2], env, ctx, base, lt, lf, n)
                return
            if sn.k == "bin" and sn.a[0] == "\\":
                nxt = Label("id")
                self.cc_in(en, sn.a[1], env, ctx, base, nxt, lf, n)
                self.asm.label(nxt)
                self.cc_in(en, sn.a[2], env, ctx, base, lf, lt, n)
                return
            if sn.k == "bin" and sn.a[0] == "..":
                e = self.as_val(self.cx(en, env, ctx, base), TInt())
                lo = self.as_val(self.cx(sn.a[1], env, ctx, base), TInt())
                hi = self.as_val(self.cx(sn.a[2], env, ctx, base), TInt())
                t1 = self.alloc(1)
                self.asm.emit("LE", t1, lo.loc, e.loc)
                self.asm.emit("JZ", t1, lf)
                self.asm.emit("LE", t1, e.loc, hi.loc)
                self.asm.emit("JNZ", t1, lt)
                self.asm.emit("JMP", lf)
                return
            if sn.k == "funcset":
                # f \in [D -> R] with a constant domain and a state-dependent range: every f[k] \in R
                dc = self.try_const(sn.a[0], env, ctx, base)
                e = self.cx(en, env, ctx, base)
                if dc is not None and isinstance(e, Val) and isinstance(e.t, TFun) \
                        and set(e.t.keys) == set(set_iter(dc.v)):
                    env2 = dict(env)
                    for j in range(len(e.t.keys)):
                        nxt = Label("ifs")
                        env2["__fs_elem"] = Val(e.t.elem, e.loc + j * e.t.elem.size)
                        self.cc_in(Node("id", ("__fs_elem",), sn.line, sn.col), sn.a[1], env2, ctx, base, nxt, lf, n)
                        self.asm.label(nxt)
                    self.asm.emit("JMP", lt)
                    return
            if sn.k == "app" and sn.a[0] == "Seq" and len(sn.a[1]) == 1 and self.resolve("Seq", env, ctx)[0] == "builtin":
                # s \in Seq(S) with a state-dependent S: every element \in S
                e = self.cx(en, env, ctx, base)
                if isinstance(e, Val) and isinstance(e.t, TSeq):
                    es = e.t.elem.size
                    i, t1, ev = self.alloc(1), self.alloc(1), self.alloc(es)
                    top, ok = Label("iql"), Label("iqk")
                    self.li(i, 0)
                    self.asm.label(top)
                    self.asm.emit("LT", t1, i, e.loc)
                    self.asm.emit("JZ", t1, lt)
                    self.asm.emit("LDX", ev, e.loc + 1, i, es)
                    self.asm.emit("ADDI", i, i, 1)
                    env2 = dict(env)
                    env2["__sq_elem"] = Val(e.t.elem, ev)
                    self.cc_in(Node("id", ("__sq_elem",), sn.line, sn.col), sn.a[1][0], env2, ctx, base, top, lf, n)
                    return
            if sn.k == "recset":
                # r \in [f1 : S1, ...]: r has exactly these fields and every r.fi \in Si (no enumeration)
                e = self.cx(en, env, ctx, base)
                names = sorted(f for f, _x in sn.a[0])
                if type(e) is Const:
                    if not (isinstance(e.v, Fcn) and sorted(e.v.d) == names):
                        self.asm.emit("JMP", lf)
                        return
                elif not isinstance(e.t, TRec) or e.t.alt_index(names) < 0:
                    self.asm.emit("JMP", lf)
                    return
                elif e.t.tagged:
                    t1 = self.alloc(1)
                    self.asm.emit("EQI", t1, e.loc, e.t.alt_index(names))
                    self.asm.emit("JZ", t1, lf)
                env2 = dict(env)
                env2["__rs_lhs"] = e
                for f, x in sn.a[0]:
                    nxt = Label("irs")
                    fld = Node("dot", (Node("id", ("__rs_lhs",), sn.line, sn.col), f), sn.line, sn.col)
                    self.cc_in(fld, x, env2, ctx, base, nxt, lf, n)
                    self.asm.label(nxt)
                self.asm.emit("JMP", lt)
                return
            if sn.k == "domain":
                # "f" \in DOMAIN r  for a record / tagged union r (InnerSerial.tla:30): a test on the alternative
                c = self.try_const(en, env, ctx, base)
                if c is not None and isinstance(c.v, str):
                    r = self.cx(sn.a[0], env, ctx, base)
                    if isinstance(r, Val) and isinstance(r.t, TRec):
                        if c.v not in r.t.fields:
                            self.asm.emit("JMP", lf)
                        elif not r.t.tagged:
                            self.asm.emit("JMP", lt)
                        else:
                            mask = sum(1 << j for j, alt in enumerate(r.t.alts) if c.v in alt)
                            mreg, tst = self.alloc(1), self.alloc(1)
                            self.li(mreg, mask)
                            self.asm.emit("BTEST", tst, mreg, r.loc)
                            self.asm.emit("JNZ", tst, lt)
                            self.asm.emit("JMP", lf)
                        return
                    if type(r) is Const and isinstance(r.v, Fcn):
                        self.asm.emit("JMP", lt if c.v in r.v.d else lf)
                        return
            if sn.k == "setfilter":
                (pat, s2), pred = sn.a
                nxt = Label("isf")
                self.cc_in(en, s2, env, ctx, base, nxt, lf, n)
                self.asm.label(nxt)
                e = self.cx(en, env, ctx, base)
                self.cc(pred, self.bind(env, pat, e), ctx, base, lt, lf)
                return
            if sn.k in ("id", "app", "sel"):
                tgt = self._expand(sn, env, ctx, base)
                if tgt is not None and tgt[0].k in ("subset", "bin", "setfilter", "funcset", "recset"):
                    # re-dispatch on the definition body with its own environment
                    node2, env2, ctx2, base2 = tgt
                    e = self.cx(en, env, ctx, base)
                    env3 = dict(env2)
                    env3["__in_lhs"] = e
                    self.cc_in(Node("id", ("__in_lhs",)), node2, env3, ctx2, base2, lt, lf, n)
                    return
        e = self.cx(en, env, ctx, base)
        if sc is not None:
            s = sc.v
            if not is_set(s):
                raise CompileError(f"\\in applied to a non-set at line {n.line}")
            if type(e) is Const:
                self.asm.emit("JMP", lt if set_contains(s, e.v) else lf)
                return
            self._in_const_set(e, s, lt, lf, n)
            return
        if sn.k == "domain":
            f = self.cx(sn.a[0], env, ctx, base)
            if isinstance(f, Val) and isinstance(f.t, TSparse):
                r = self.sp_find(f, e)
                self.asm.emit("JGEZ", r, lt)
                self.asm.emit("JMP", lf)
                return
        sv = self.cx(sn, env, ctx, base)
        if type(sv) is Const:
            self._in_const_set(self.as_val(e), sv.v, lt, lf, n)
            return
        if isinstance(sv.t, TSparse) and sv.t.vt is None:
            r = self.sp_find(sv, e)
            self.asm.emit("JGEZ", r, lt)
            self.asm.emit("JMP", lf)
            return
        if not isinstance(sv.t, TSet):
            raise CompileError(f"\\in applied to non-set type {sv.t}")
        if isinstance(sv.t.elem, TBottom):
            self.asm.emit("JMP", lf)
            return
        t1 = self.alloc(1)
        if type(e) is Const:
            oc = self.codec.ord_of(sv.t.elem, e.v)
            if oc < 0:
                self.asm.emit("JMP", lf)
                return
            self.asm.emit("BTESTI", t1, sv.loc, oc)
        else:
            o = self.ord_in(sv.t.elem, e)
            if self.ord_can_fail(sv.t.elem, e):
                self.asm.emit("JNEG", o, lf)
            self.asm.emit("BTEST", t1, sv.loc, o)
        self.asm.emit("JNZ", t1, lt)
        self.asm.emit("JMP", lf)

    def _in_const_set(self, e: Val, s, lt, lf, n):
        from ..front.values import SetFuncs, SetSubset, SetRecs, SetTimes, SetUnionLazy, SetSeq
        t = e.t
        # structural membership in lazy set values (never enumerate [S -> T], SUBSET S, ...)
        if isinstance(s, SetUnionLazy):
            nxt = Label("mu")
            self._in_const_set(e, s.a, lt, nxt, n)
            self.asm.label(nxt)
            self._in_const_set(e, s.b, lt, lf, n)
            return
        if isinstance(s, SetFuncs) and isinstance(t, (TFun, TTuple)):
            dom = tuple(sorted_vals(to_finite(s.dom)))
            keys = t.keys if isinstance(t, TFun) else tuple(range(1, len(t.elems) + 1))
            if dom != tuple(keys):
                self.asm.emit("JMP", lf)
                return
            for j in range(len(keys)):
                sub = Val(t.elem, e.loc + j * t.elem.size) if isinstance(t, TFun) else Val(t.elems[j], e.loc + t.offs[j])
                nxt = Label("mf")
                self._in_const_set(sub, s.rng, nxt, lf, n)
                self.asm.label(nxt)
            self.asm.emit("JMP", lt)
            return
        if isinstance(s, SetSubset) and isinstance(t, TSet):
            if isinstance(t.elem, TBottom):
                self.asm.emit("JMP", lt)
                return
            vals = self.codec.enum(t.elem)
            words = [0] * t.size
            for i, v in enumerate(vals):
                if set_contains(s.s, v):
                    words[i >> 5] |= 1 << (i & 31)
            words = [w - (1 << 32) if w >= (1 << 31) else w for w in words]
            mloc = self.alloc(t.size)
            self.load_words(mloc, words)
            t2 = self.alloc(1)
            self.asm.emit("BSUB", t2, e.loc, mloc, t.size)
            self.asm.emit("JNZ", t2, lt)
            self.asm.emit("JMP", lf)
            return
        if isinstance(s, SetRecs) and isinstance(t, TRec) and not t.tagged:
            names = tuple(sorted(f for f, _ in s.fields))
            if names != t.alts[0]:
                self.asm.emit("JMP", lf)
                return
            for f, fs in s.fields:
                nxt = Label("mr")
                self._in_const_set(Val(t.fields[f], e.loc + t.off[f]), fs, nxt, lf, n)
                self.asm.label(nxt)
            self.asm.emit("JMP", lt)
            return
        if isinstance(s, SetSeq) and isinstance(t, (TSeq, TTuple)):
            if isinstance(t, TTuple):
                for j in range(len(t.elems)):
                    nxt = Label("mq")
                    self._in_const_set(Val(t.elems[j], e.loc + t.offs[j]), s.s, nxt, lf, n)
                    self.asm.label(nxt)
                self.asm.emit("JMP", lt)
                return
            es = t.elem.size
            for j in range(t.cap):            # element j is checked only if j < Len
                nxt = Label("mq")
                t2 = self.alloc(1)
                self.asm.emit("LEI", t2, e.loc, j)
                self.asm.emit("JNZ", t2, lt)
                self._in_const_set(Val(t.elem, e.loc + 1 + j * es), s.s, nxt, lf, n)
                self.asm.label(nxt)
            self.asm.emit("JMP", lt)
            return
        if isinstance(s, SetTimes) and isinstance(t, TTuple) and len(s.sets) == len(t.elems):
            for j, ss in enumerate(s.sets):
                nxt = Label("mt")
                self._in_const_set(Val(t.elems[j], e.loc + t.offs[j]), ss, nxt, lf, n)
                self.asm.label(nxt)
            self.asm.emit("JMP", lt)
            return
        t1 = self.alloc(1)
        if isinstance(t, TInt) and t.lo is None:
            if isinstance(s, SetNat):
                self.asm.emit("GEI", t1, e.loc, 0)
                self.asm.emit("JNZ", t1, lt)
                self.asm.emit("JMP", lf)
                return
            if isinstance(s, SetInt):
                self.asm.emit("JMP", lt)
                return
            if isinstance(s, frozenset):
                ints = sorted(x for x in s if type(x) is int)
                if ints and ints == list(range(ints[0], ints[-1] + 1)):
                    self.asm.emit("GEI", t1, e.loc, ints[0])
                    self.asm.emit("JZ", t1, lf)
                    self.asm.emit("LEI", t1, e.loc, ints[-1])
                    self.asm.emit("JNZ", t1, lt)
                    self.asm.emit("JMP", lf)
                    return
                for x in ints:
                    self.asm.emit("EQI", t1, e.loc, x)
                    self.asm.emit("JNZ", t1, lt)
                self.asm.emit("JMP", lf)
                return
            raise CompileError("membership of an unbounded integer in a lazy set")
        # enumerable element type: constant bitmask over its universe
        try:
            n_u = t.card()
        except TypeErr as ex:
            raise CompileError(str(ex))
        if n_u > 8192:
            raise CompileError("membership test over a universe larger than 8192 values")
        vals = self.codec.enum(t)
        words = [0] * ((n_u + 31) // 32)
        anyb = False
        for i, v in enumerate(vals):
            if set_contains(s, v):
                words[i >> 5] |= 1 << (i & 31)
                anyb = True
        if not anyb:
            self.asm.emit("JMP", lf)
            return
        words = [w - (1 << 32) if w >= (1 << 31) else w for w in words]
        mloc = self.alloc(len(words))
        self.load_words(mloc, words)
        o = self.ord_in(t, e)
        self.asm.emit("JNEG", o, lf)
        self.asm.emit("BTEST", t1, mloc, o)
        self.asm.emit("JNZ", t1, lt)
        self.asm.emit("JMP", lf)

    def cc_subseteq(self, ln, rn, env, ctx, base, lt, lf, n):
        a = self.cx(ln, env, ctx, base)
        if type(a) is Const:
            vals = list(set_iter(a.v))
            for v in vals:
                nxt = Label("ss")
                env2 = dict(env)
                env2["__ss_elem"] = Const(v)
                self.cc_in(Node("id", ("__ss_elem",)), rn, env2, ctx, base, nxt, lf, n)
                self.asm.label(nxt)
            self.asm.emit("JMP", lt)
            return
        if not isinstance(a.t, TSet):
            raise CompileError(f"\\subseteq on non-set type {a.t}")
        rc = self.try_const(rn, env, ctx, base)
        if rc is not None and not is_enumerable(rc.v):
            # e.g.  S \subseteq Nat : check element-wise
            def each(x):
                nxt = Label("se")
                self._in_const_set(x, rc.v, nxt, lf, n)
                self.asm.label(nxt)
            self.loop_set(a, each)
            self.asm.emit("JMP", lt)
            return
        b = self.cx(rn, env, ctx, base, a.t)
        try:
            bv = self.coerce(b, a.t) if type(b) is Const or b.t != a.t else b
            av = a
        except CompileError:
            tj = join(a.t, b.t if isinstance(b, Val) else self.natural_type(b.v))
            av, bv = self.coerce(a, tj), self.coerce(b, tj)
        t1 = self.alloc(1)
        self.asm.emit("BSUB", t1, av.loc, bv.loc, av.t.size)
        self.asm.emit("JNZ", t1, lt)
        self.asm.emit("JMP", lf)

    # ----------------------------------------------------------------- actions
    def ca(self, n, env, ctx, bound, k, act):
        """Compile action n; `k(bound)` emits the continuation for each satisfying branch.
        Control falls through after all alternatives are exhausted."""
        self.bound = bound
        kind = n.k
        # Segment cuts (compile/sliced.py): `top` is true while nothing but disjunction structure lies
        # between the root of Next and this node, i.e. the code of each alternative below is a self-contained slice of
        # the program (entered by falling in, left by falling out) that can become a kernel of its own.
        top = self._seg_top
        self._seg_top = False
        if kind == "and":
            items = n.a[0]
            # the first conjunct may still be sliced: the conjuncts after it are lowered inside its continuations
            self._seg_top = top
            if len(items) > 1 and act is not None and act[0] == "split":
                act = ("fixed",) + act[1:]

            def chain(i, b):
                if i == len(items):
                    k(b, act)
                    return
                self.ca(items[i], env, ctx, b, lambda b2, _a: chain(i + 1, b2), act)
            chain(0, bound)
            return
        if kind == "abox":        # [A]_v as an action: A \/ UNCHANGED v
            n = Node("or", ((n.a[0], Node("unchanged", (n.a[1],), n.line, n.col)),), n.line, n.col)
            kind = "or"
        if kind == "or":
            for x in n.a[0]:
                self.bound = bound
                m = self.mark()
                if top:
                    top = self._seg_begin()
                self.ca(x, env, ctx, bound, k, act)
                self.release(m)
                if top:
                    self._seg_end()
            return
        if kind == "exists":
            bounds, body = n.a
            if len(bounds) == 1 and isinstance(bounds[0][0], str) and bounds[0][1] is not None:
                sk = self.set_elements(bounds[0][1], env, ctx, "N")
                if sk[0] == "val" and not isinstance(sk[1].t.elem, TBottom):
                    pat = bounds[0][0]
                    sv2, rest = self.narrow(sk[1], pat, self.flat_and(body), env, ctx, "N")
                    body2 = Node("bool", (True,)) if not rest else (
                        rest[0] if len(rest) == 1 else Node("and", (tuple(rest),), body.line, body.col))

                    def each1(xv):
                        m = self.mark()
                        self.bound = bound
                        self.ca(body2, self.bind(env, pat, xv), ctx, bound, k, act)
                        self.release(m)
                    self.loop_set(sv2, each1)
                    return

            topbox = [top]

            def each(env2):
                m = self.mark()
                self.bound = bound
                if topbox[0]:
                    topbox[0] = self._seg_begin()
                self.ca(body, env2, ctx, bound, k, act)
                self.release(m)
                if topbox[0]:
                    self._seg_end()
            self.for_each(bounds, env, ctx, "N", each)
            return
        if kind == "if":
            c1 = self.try_const(n.a[0], env, ctx, "N")
            if c1 is not None:
                self._seg_top = top
                self.ca(n.a[1] if c1.v else n.a[2], env, ctx, bound, k, act)
                return
            lt, lf, end = Label("at"), Label("af"), Label("ae")
            m = self.mark()
            self.cc(n.a[0], env, ctx, "N", lt, lf)
            self.release(m)
            self.asm.label(lt)
            self.ca(n.a[1], env, ctx, bound, k, act)
            self.asm.emit("JMP", end)
            self.asm.label(lf)
            self.ca(n.a[2], env, ctx, bound, k, act)
            self.asm.label(end)
            return
        if kind == "case":
            arms, other = n.a
            node = other if other is not None else Node("bool", (False,), n.line, n.col)
            for c2, e in reversed(arms):
                node = Node("if", (c2, e, node), n.line, n.col)
            self.ca(node, env, ctx, bound, k, act)
            return
        if kind == "let":
            env_l = self.let_env(n.a[0], env, ctx, "N", n.a[1])
            self._seg_top = top
            self.ca(n.a[1], env_l, ctx, bound, k, act)
            return
        if kind in ("id", "app", "sel"):
            is_assert = kind == "app" and n.a[0] == "Assert"
            tgt = None if is_assert else self._expand(n, env, ctx, "N")
            if tgt is not None:
                node2, env2, ctx2, _ = tgt
                act2 = act
                if (act is None or act[0] == "split") and kind != "sel":
                    r = self.resolve(n.a[0], env, ctx)
                    if r[0] == "def":
                        act2 = ("split", r[1].name, r[1].body.loc(), r[2].name)
                self._seg_top = top
                self.ca(node2, env2, ctx2, bound, k, act2)
                return
        if kind == "bin" and n.a[0] in ("=", "\\in"):
            tv = self._assign_target(n.a[1], env, ctx, bound)
            if tv is not None:
                t = self.var_types[tv]
                if n.a[0] == "=":
                    m = self.mark()
                    x = self.cx(n.a[2], env, ctx, "N", t)
                    xv = self.coerce(x, t)
                    self.movn(self.p_off[tv], xv.loc, t.size)
                    self.release(m)
                    b2 = bound | {tv, "*" + tv}
                    self.bound = b2
                    k(b2, act)
                    if self.copy_once:
                        self.movn(self.p_off[tv], self.n_off[tv], t.size)
                    return
                # x' \in S : one alternative per element
                def each(env2):
                    m = self.mark()
                    x = env2["__asg"]
                    xv = self.coerce(x, t)
                    self.movn(self.p_off[tv], xv.loc, t.size)
                    self.release(m)
                    b2 = bound | {tv, "*" + tv}
                    self.bound = b2
                    k(b2, act)
                self.for_each([("__asg", n.a[2])], env, ctx, "N", each)
                if self.copy_once:
                    self.movn(self.p_off[tv], self.n_off[tv], t.size)
                return
        if kind == "unchanged":
            names = []
            if self._unchanged_vars(n.a[0], env, ctx, names):
                b2 = set(bound)
                end = Label("ue")
                for v in names:
                    t = self.var_types[v]
                    if v in b2:
                        t1 = self.alloc(1)
                        if t.size == 1:
                            self.asm.emit("EQ", t1, self.p_off[v], self.n_off[v])
                        else:
                            self.asm.emit("EQN", t1, self.p_off[v], self.n_off[v], t.size)
                        self.asm.emit("JZ", t1, end)
                    else:
                        if not self.copy_once:
                            self.movn(self.p_off[v], self.n_off[v], t.size)
                        b2.add(v)
                b2 = frozenset(b2)
                self.bound = b2
                k(b2, act)
                self.asm.label(end)
                return
        # guard
        lt, lf = Label("gt"), Label("gf")
        m = self.mark()
        self.bound = bound
        self.cc(n, env, ctx, "N", lt, lf)
        self.release(m)
        self.asm.label(lt)
        k(bound, act)
        self.asm.label(lf)

    def _seg_begin(self) -> bool:
        """Start a slice of the Next program here if nothing has been emitted since the last slice boundary (code
        emitted at this level would be shared by the alternatives that follow and has to stay in one slice)."""
        code = self.asm.code
        if code is not self._seg_buf or len(code) != self._seg_clean:
            self._seg_top = False
            return False
        if self._seg_last != len(code):
            L = Label("seg")
            self.asm.label(L)
            self.seg_cuts["next"].append(L)
            self._seg_clean = self._seg_last = len(self.asm.code)
        self._seg_top = True
        return True

    def _seg_end(self):
        if self.asm.code is self._seg_buf:
            self._seg_clean = len(self.asm.code)

    def _assign_target(self, ln, env, ctx, bound):
        if ln.k == "id" and ln.a[0] in env and type(env[ln.a[0]]) is Lazy:
            lz = env[ln.a[0]]
            return self._assign_target(lz.node, lz.env, lz.ctx, bound)
        if ln.k == "prime" and ln.a[0].k == "id":
            v = ln.a[0].a[0]
            if v in env and type(env[v]) is Lazy and env[v].node.k == "id":
                lz = env[v]
                return self._assign_target(Node("prime", (lz.node,)), lz.env, lz.ctx, bound)
            if v in ctx.varset and v not in env and v not in ctx.substs and v not in bound \
                    and v in self.var_types:
                return v
        return None

    def _unchanged_vars(self, e, env, ctx, out):
        if e.k == "id":
            nm = e.a[0]
            if nm in env:
                return False
            if nm in ctx.varset and nm not in ctx.substs:
                out.append(nm)
                return True
            d = ctx.defs.get(nm)
            if d is not None and not d[0].params:
                return self._unchanged_vars(d[0].body, {}, d[1], out)
            return False
        if e.k == "tuple":
            return all(self._unchanged_vars(x, env, ctx, out) for x in e.a[0])
        return False

    # ---------------------------------------------------------------- symmetry
    def _perm_touches(self, t: T, perm) -> bool:
        """Does applying `perm` (dict ModelValue -> ModelValue) change any value of type t?"""
        if isinstance(t, TAtom):
            return any(a in perm and perm[a] != a for a in t.atoms)
        if isinstance(t, (TInt, TBool, TBottom)):
            return False
        if isinstance(t, TRec):
            return any(self._perm_touches(x, perm) for x in t.fields.values())
        if isinstance(t, TTuple):
            return any(self._perm_touches(x, perm) for x in t.elems)
        if isinstance(t, TFun):
            return any(k in perm and perm[k] != k for k in t.keys) or self._perm_touches(t.elem, perm)
        if isinstance(t, (TSet, TSeq)):
            return self._perm_touches(t.elem, perm)
        return True

    def gen_perm(self, t: T, src, dst, perm):
        """Emit code writing the image of the value at frame[src..] under `perm` to frame[dst..]."""
        from ..front.values import permute_value
        if not self._perm_touches(t, perm):
            self.movn(dst, src, t.size)
            return
        if isinstance(t, TAtom):
            tbl = list(range(len(self.atoms.vals)))
            for a in t.atoms:
                if a in perm:
                    tbl[self.atoms.id(a)] = self.atoms.id(perm[a])
            self.asm.emit("TBL", dst, self.asm.const_table(tbl), src)
            return
        if isinstance(t, TRec):
            if t.tagged:
                self.asm.emit("MOV", dst, src)
            for f in t.fnames:
                self.gen_perm(t.fields[f], src + t.off[f], dst + t.off[f], perm)
            return
        if isinstance(t, TTuple):
            for e, o in zip(t.elems, t.offs):
                self.gen_perm(e, src + o, dst + o, perm)
            return
        if isinstance(t, TFun):
            es = t.elem.size
            for i, k in enumerate(t.keys):
                j = t.kindex[perm.get(k, k)] if (is_atom(k) and not isinstance(k, str)) else i
                self.gen_perm(t.elem, src + i * es, dst + j * es, perm)
            return
        if isinstance(t, TSet):
            vals = self._enum_cached(t.elem)
            ptab = [self.codec.ord_of(t.elem, permute_value(v, perm)) for v in vals]
            if any(o < 0 for o in ptab):
                raise CompileError("SYMMETRY: a set universe is not closed under the permutation")
            base = self.asm.const_table(ptab)
            self.asm.emit("ZERO", dst, t.size)
            idx, pidx = self.alloc(1), self.alloc(1)
            top, done = Label("pl"), Label("pd")
            self.li(idx, -1)
            self.asm.label(top)
            self.asm.emit("BNEXT", idx, src, idx, t.nbits)
            self.asm.emit("JNEG", idx, done)
            self.asm.emit("TBL", pidx, base, idx)
            self.asm.emit("BSET", dst, pidx)
            self.asm.emit("JMP", top)
            self.asm.label(done)
            return
        if isinstance(t, TSeq):
            self.asm.emit("MOV", dst, src)
            for j in range(t.cap):
                self.gen_perm(t.elem, src + 1 + j * t.elem.size, dst + 1 + j * t.elem.size, perm)
            return
        raise CompileError(f"SYMMETRY: cannot permute values of type {t}")

    def gen_canonicalize(self, group):
        """Replace the primed state by the least (word-wise lexicographic on the unpacked frame) of its images
        under the symmetry group, so that one representative per orbit reaches the seen-set (K6 of SURVEY §2c)."""
        usz = self.usz
        best, cand = self.alloc(usz), self.alloc(usz)
        p0 = self.p_off[self.m.vars[0]]
        self.movn(best, p0, usz)
        for perm in group:
            mk = self.mark()
            for v in self.m.vars:
                off = self.n_off[v]
                self.gen_perm(self.var_types[v], p0 + off, cand + off, perm)
            t1 = self.alloc(1)
            skip = Label("cs")
            self.asm.emit("LEXLT", t1, cand, best, usz)
            self.asm.emit("JZ", t1, skip)
            self.movn(best, cand, usz)
            self.asm.label(skip)
            self.release(mk)
        self.movn(p0, best, usz)

    # ------------------------------------------------------------------ driver
    def compile(self, init_states) -> CompiledModel:
        """Two passes: a dry pass counts how often each zero-arity state-level definition
        (e.g. Paxos.tla:185 `votes`) is expanded; definitions used more than once and free of
        traps are then evaluated once per state in the program prologue (hoisted)."""
        self.var_types = self.infer_var_types(init_states)
        if self.use_subs:
            return self._compile_with_subs()
        self.dry = True
        try:
            self._compile_pass()
        except CompileError:
            self.dry = False
            raise
        keys = [k for k, c in self.def_uses.items() if c >= 2]
        info = dict(self.def_info)
        # reset the assembler state
        self.dry = False
        self.asm = Asm()
        self.actions, self.asserts = [], []
        self.hoisted, self.def_uses, self.def_info = {}, {}, {}
        self._evenv_cache = {}
        self.__dict__.pop("_univ_cache", None)
        self.__dict__.pop("_field_cache", None)
        self.hoist_keys = [(k, info[k]) for k in keys]
        return self._compile_pass()

    def _reset_pass_state(self):
        self.asm = Asm()
        self.actions, self.asserts = [], []
        self.hoisted, self.def_uses, self.def_info = {}, {}, {}
        self._evenv_cache = {}
        self.__dict__.pop("_univ_cache", None)
        self.__dict__.pop("_field_cache", None)
        self.subs, self.sub_bufs, self.sub_calls = {}, [], {}
        self._sub_stack, self._sub_active = [], set()

    def _compile_with_subs(self):
        """Operator definitions as CALL/RET subroutines (for specifications whose inline expansion explodes).
        Pass 1 discovers the subroutine instances, their frame sizes and the call graph; pass 2 generates the same
        code with the planned static frames."""
        self.hoist_keys = []
        self.sub_plan = None
        self._compile_pass()
        main_high = self._main_high
        plan, total = self._plan_sub_frames(main_high)
        self._reset_pass_state()
        self.sub_plan = plan
        cm = self._compile_pass()
        if self._main_high > main_high:
            raise CompileError("internal: non-deterministic lowering between the subroutine passes")
        cm.frame_words = max(cm.frame_words, total + 4)
        return cm

    def _hoist_prologue(self, program):
        for key, (od, dctx) in self.hoist_keys:
            name, _, base, prog = key
            if prog != program or base != "N":
                continue
            with self.asm.capture() as cap:
                save_top = self.top
                try:
                    v = self.cx(od.body, {}, dctx, "N")
                except CompileError:
                    v = None
                if v is None or type(v) is Const or any(
                        (i[0] == "TRAP" and i[1] != TRAP_OVERFLOW) or i[0] in ("ASSERTF", "TBLT") for i in cap.asm.code):
                    self.top = save_top
                    v = None
            if v is None:
                continue
            self.asm.splice(cap.buf)
            self.hoisted[key] = v

    def _compile_pass(self) -> CompiledModel:
        m = self.m
        self.n_off, self.p_off = {}, {}
        off = 0
        for v in m.vars:
            self.n_off[v] = off
            off += self.var_types[v].size
        usz = off
        self.usz = usz
        for v in m.vars:
            self.p_off[v] = usz + self.n_off[v]
        self.blocks = set()
        for v in m.vars:
            self.blocks.add((self.n_off[v], self.var_types[v].size))
            self.blocks.add((self.p_off[v], self.var_types[v].size))
        self.top = self.high = 2 * usz
        # SYMMETRY: the canonicalisation code is one subroutine (CALL at every EMIT site) with a static scratch region
        # right after the two state copies; its size is measured by a trial lowering
        self._canon = None
        if self.group:
            with self.asm.capture():
                self.gen_canonicalize(self.group)
            base0 = 2 * usz
            ret = base0
            need = self.high - base0
            self._canon = {"label": Label("canon"), "ret": ret, "base": base0 + 1}
            self.top = self.high = base0 + 1 + need
        entries = {}
        # ---- invariants (evaluated on the state being expanded) ----
        linv = Label("inv")
        self.asm.label(linv)
        entries["inv"] = linv
        self.program = "inv"
        self._hoist_prologue("inv")
        self.seg_cuts = {"inv": [], "next": []}
        self._seg_top, self._seg_buf, self._seg_clean, self._seg_last = False, None, -1, -1
        for i, (nm, node, c) in enumerate(m.invariants):
            cut = Label("segi")
            self.asm.label(cut)
            self.seg_cuts["inv"].append(cut)
            ok, bad = Label("iok"), Label("ibad")
            mk = self.mark()
            self.bound = frozenset()
            self.cc(node, {}, c, "N", ok, bad)
            self.release(mk)
            self.asm.label(bad)
            self.asm.emit("INVF", i)
            self.asm.label(ok)
        self.asm.emit("HALT")
        # ---- next ----
        lnext = Label("next")
        self.asm.label(lnext)
        entries["next"] = lnext
        self.program = "next"
        inv_top = self.top
        # Wide states (container models): the primed copy is initialised ONCE per state (primed := current) and kept
        # "clean" -- UNCHANGED is then free, an assignment x' = e restores x' := x when its continuation returns.
        # Per successor this replaces a copy of every unchanged variable (raft: ~500 words of containers) by a copy
        # of the changed ones.  (Not with SYMMETRY: canonicalisation rewrites the whole primed state in place.)
        self.copy_once = (not self.group) and self.usz >= 64
        if self.copy_once:
            self.movn(self.usz, 0, self.usz)
        self._hoist_prologue("next")
        allv = frozenset(m.vars)

        slot_ranges = self._var_slot_ranges() if self.copy_once else None

        def emit_succ(b, aid):
            """EMIT, or EMITD with the packed-slot ranges of the variables assigned on this path (wide states:
            the engine re-packs those over the parent's packed words instead of packing every slot)."""
            if slot_ranges is None or aid > MAXREG:
                self.asm.emit("EMIT", aid)
                return
            rs = []
            for v in m.vars:
                if "*" + v in b:
                    rs += slot_ranges[v]
            rs.sort()
            merged = []
            for first, cnt, pos in rs:
                if merged and merged[-1][0] + merged[-1][1] == first:
                    merged[-1][1] += cnt
                else:
                    merged.append([first, cnt, pos])
            if sum(c for _, c, _ in merged) * 2 > self._n_slots:      # most of the state changed: plain pack
                self.asm.emit("EMIT", aid)
                return
            tbl = [len(merged)]
            for first, cnt, pos in merged:
                tbl += [first, cnt, pos]
            if not self.asm.cpool:             # table index 0 means "no table" to the engines: occupy it
                self.asm.const_table([0])
            base = self.asm.const_table(tbl)
            self.asm.emit("EMITD", aid, base)

        def emit_k(b, act):
            missing = [v for v in m.vars if v not in b]
            if missing:
                raise CompileError(f"action {act[1] if act else 'Next'} does not assign {missing}")
            aid = self._action_id(act)
            # refinement PROPERTYs: every transition must satisfy [Next2]_v2 (checked like TLC's action
            # properties, on every generated successor); a violation is reported through ASSERTF
            for nm, _inits, nxt2, sub2, c2 in getattr(m, "refinements", []):
                if nxt2 is None:
                    continue
                ok, bad = Label("pok"), Label("pbad")
                mk = self.mark()
                self.bound = allv
                step = Node("or", ((nxt2, Node("unchanged", (sub2,))),))
                self.cc(step, {}, c2, "N", ok, bad)
                self.release(mk)
                self.asm.label(bad)
                self.asserts.append(("\x00property:" + nm, nxt2.loc()))
                self.asm.emit("ASSERTF", len(self.asserts) - 1)
                self.asm.label(ok)
            if self.group:
                self.asm.emit("CALL", self._canon["ret"], self._canon["label"])
            if m.constraints or m.action_constraints:
                ok, bad, end = Label("cok"), Label("cbad"), Label("cend")
                mk = self.mark()
                self.bound = allv
                conj = [Node("prime", (Node("id", (nm,)),)) for nm, _, _ in m.constraints]
                conj += [Node("id", (nm,)) for nm, _, _ in m.action_constraints]
                self.cc(Node("and", (tuple(conj),)), {}, self.ctx, "N", ok, bad)
                self.release(mk)
                self.asm.label(bad)
                self.asm.emit("GEN")
                self.asm.emit("JMP", end)
                self.asm.label(ok)
                emit_succ(b, aid)
                self.asm.label(end)
            else:
                emit_succ(b, aid)
        if m.next_node is None:
            raise CompileError("no next-state action")
        # slices of Next: the first one starts right after the prologue (copy of the state, hoisted definitions)
        cut0 = Label("seg")
        self.asm.label(cut0)
        self.seg_cuts["next"].append(cut0)
        self._seg_buf = self.asm.code
        self._seg_clean = self._seg_last = len(self.asm.code)
        self._seg_top = True
        self.ca(m.next_node, {}, m.next_ctx, frozenset(), emit_k, None)
        self._seg_top, self._seg_buf = False, None
        self.asm.emit("HALT")
        self._main_high = self.high
        if self._canon is not None:
            save_top = self.top
            self.top = self._canon["base"]
            self.asm.label(self._canon["label"])
            self.gen_canonicalize(self.group)
            self.asm.emit("RET", self._canon["ret"])
            self.top = save_top
        for buf in self.sub_bufs:            # subroutine bodies (entered by CALL only)
            self.asm.splice(buf)
        code, cpool, ent = self.asm.assemble(entries)
        cm = CompiledModel()
        cm.code, cm.cpool, cm.entries = code, cpool, ent
        cm.segments = {k: sorted(set(int(L.pos) for L in v)) for k, v in self.seg_cuts.items()}
        cm.blocks = sorted(self.blocks) if len(self.blocks) <= 8192 else None
        cm.line_table = self.asm.line_table
        cm.frame_words = self.high + 4
        cm.var_types = self.var_types
        cm.var_off = dict(self.n_off)
        cm.vars = list(m.vars)
        cm.n_off, cm.p_off = 0, usz
        cm.state_words_unpacked = usz
        cm.actions = list(self.actions)
        cm.asserts = list(self.asserts)
        cm.invariants = [nm for nm, _, _ in m.invariants]
        cm.atoms, cm.codec = self.atoms, self.codec
        cm.group = list(self.group)
        cm.warnings = self.warnings
        cm.seq_cap = self.seq_cap
        lay = self._packed_layout()
        import numpy as np
        cm.layout = np.array(lay, dtype=np.int32).reshape(-1, 3)
        bits = int(cm.layout[:, 1].sum())
        cm.W = max(1, (bits + 31) // 32)
        cm.state_bits = bits
        return cm

    def _compile_labels(self, cm, state_preds, edge_preds) -> "LabelImage":
        """compile_labels: the two label programs over cm's frame layout (the offsets of _compile_pass)"""
        m = self.m
        self.n_off, self.p_off = dict(cm.var_off), {v: cm.state_words_unpacked + cm.var_off[v] for v in m.vars}
        self.usz = usz = cm.state_words_unpacked
        self.blocks = set()
        for v in m.vars:
            self.blocks.add((self.n_off[v], self.var_types[v].size))
            self.blocks.add((self.p_off[v], self.var_types[v].size))
        self.top = self.high = 2 * usz
        self._canon = None
        allv = frozenset(m.vars)
        entries = {}
        for prog, preds, bound in (("states", state_preds, frozenset()), ("edges", edge_preds, allv)):
            lab = Label(prog)
            self.asm.label(lab)
            entries[prog] = lab
            self.program = prog
            for j, p in enumerate(preds):
                node = p.node
                if prog == "edges":          # <<A>>_v = A /\ ~UNCHANGED v
                    a, sub = node.a
                    node = Node("and", ((a, Node("not", (Node("unchanged", (sub,)),))),), node.line, node.col)
                ok, bad = Label("lok"), Label("lbad")
                mk = self.mark()
                self.bound = bound
                self.cc(node, _label_env(p.env), p.ctx, "N", ok, bad)
                self.release(mk)
                self.asm.label(bad)
                self.asm.emit("INVF", j)
                self.asm.label(ok)
            self.asm.emit("HALT")
        for buf in self.sub_bufs:
            self.asm.splice(buf)
        code, cpool, ent = self.asm.assemble(entries)
        img = LabelImage()
        img.code, img.cpool, img.entries = code, cpool, ent
        img.frame_words = self.high + 4
        img.n_states, img.n_edges = len(state_preds), len(edge_preds)
        limit = frame_class(cm.frame_words)
        if img.frame_words > limit:
            raise CompileError(f"the liveness labels need a frame of {img.frame_words} words, more than the "
                               f"{limit} words the model's kernels have")
        return img

    def _packed_layout(self):
        """Pack order: (frame offset, bit width, bias) per scalar slot."""
        lay = []
        aw = self.atoms.width()
        for v in self.m.vars:
            for (fo, w, bias) in self.codec.layout(self.var_types[v], self.n_off[v]):
                lay.append((fo, aw if w < 0 else w, bias))
        if any(has_dynamic(self.var_types[v]) for v in self.m.vars):
            lay = self._cluster_slots_last(lay)
        return lay

    def _var_slot_ranges(self):
        """variable -> [(first slot, slot count, bit position of the first slot)] in pack order."""
        lay = self._packed_layout()
        self._n_slots = len(lay)
        pos, bitpos = {}, 0
        for i, (fo, w, _b) in enumerate(lay):
            pos[fo] = (i, bitpos)
            bitpos += w
        out = {}
        for v in self.m.vars:
            t = self.var_types[v]
            idx = sorted(pos[fo] for fo in range(self.n_off[v], self.n_off[v] + t.size) if fo in pos)
            rs = []
            for i, bp in idx:
                if rs and rs[-1][0] + rs[-1][1] == i:
                    rs[-1][1] += 1
                else:
                    rs.append([i, 1, bp])
            out[v] = [tuple(r) for r in rs]
        return out

    def _cluster_slots_last(self, lay):
        """Pack order for models with containers.  The engine clusters each BFS level, and partitions the state
        space over GPUs, by the LAST TWO packed words (tlag_owner, the frontier clustering key).  With containers laid out in
        variable order those words would hold the zero tail of the last container (no entropy: every state on one
        rank).  So the "control" slots -- scalar variables, elements of small per-process functions, container
        lengths, presence flags -- are packed last, up to 64 bits of them."""
        ctrl = []

        def walk(t, off):
            if t.scalar:
                ctrl.append(off)
            elif isinstance(t, TFun):
                for j in range(len(t.keys)):
                    walk(t.elem, off + j * t.elem.size)
            elif isinstance(t, TSet):
                if t.nbits <= 16:
                    ctrl.append(off)
            elif isinstance(t, (TSeq, TSparse)):
                ctrl.append(off)
            elif isinstance(t, TPFun):
                for j in range(len(t.keys)):
                    ctrl.append(off + j * t.stride)
        for v in self.m.vars:
            walk(self.var_types[v], self.n_off[v])
        ctrl = set(ctrl)
        head, tail, used = [], [], 0
        for slot in lay:
            if slot[0] in ctrl and used + slot[1] <= 64:
                tail.append(slot)
                used += slot[1]
            else:
                head.append(slot)
        return head + tail

    def _action_id(self, act):
        if act is None:
            key = ("Next", (0, 0, 0, 0), self.m.module_name)
        else:
            key = (act[1], act[2], act[3])
        for i, a in enumerate(self.actions):
            if a == key:
                return i
        self.actions.append(key)
        return len(self.actions) - 1


class LabelImage:
    """The bytecode of the state-graph labels (DESIGN.md §7h), an image of its own over a model's frame: the program at
    entries["states"] runs on one stored state (current frame) and the one at entries["edges"] on an edge (s in the
    current frame, t in the primed one).  Predicate j of a program that is false raises INVF j."""

    def __init__(self):
        self.code = None
        self.cpool = None
        self.entries = {}
        self.frame_words = 0
        self.n_states = 0
        self.n_edges = 0


def frame_class(words):
    """The frame the interpreter kernels give a model of `words` frame words (vm_frame_class in csrc/tlag_engine.cu)"""
    c = 64
    while c < 8192 and c < words:
        c *= 2
    return c


def compile_labels(m, cm: CompiledModel, state_preds, edge_preds) -> LabelImage:
    """Lower the state predicates and the actions <<A>>_v (front/spec.py Pred) of model m into a label image over cm's
    layout, atom table and frame; cm itself is not touched.  An image that needs more than the frame the model's
    kernels have (frame_class) is a CompileError."""
    lw = Lowering(m, seq_cap=cm.seq_cap)
    lw.atoms, lw.codec = cm.atoms, cm.codec
    lw.var_types = cm.var_types
    lw.group = []
    return lw._compile_labels(cm, state_preds, edge_preds)


def _label_env(env):
    return {k: Const(v) for k, v in env.items()}
