"""Sliced native build: the bytecode of one CompiledModel compiled to C / CUDA C, ONE FUNCTION PER SLICE of the program.

Why (round-1 measurements, DESIGN.md section 4b): the bytecode interpreter is instruction-issue bound (~70 SASS
instructions per bytecode instruction) and the first compiled form -- the whole program as one function, every warp
walking it on its own -- was slower than the interpreter: 354 KB of code against a 32 KB instruction cache, each warp
in a different place.  A BFS level does not need that: the next-state relation is a disjunction of actions and the
invariants are a conjunction, so a level is expanded as a sequence of small kernels

    for every invariant i:   k_inv<i>  over the frontier          (prologue + the code of invariant i)
    for every slice j of Next: k_next<j> over the frontier        (prologue + the code of one disjunct of Next)

Every warp of a launch runs the same few KB of straight-line code (instruction-cache resident, hardware divergence
and reconvergence instead of a software pc election), the packed state is re-read per kernel (44 B for Paxos: the
launches are still three orders of magnitude under the HBM roofline), and successors are handled where they are
produced (pack -> fingerprint -> probe/insert) instead of through an event protocol.

The lowering marks where slices may start (compile/lower.py: `_seg_begin`; `cm.segments`); this module checks that each
slice is closed under its jumps (merging neighbours that are not) and emits, per model, one `.inc` file:

    subroutines (CALL targets)      -> TLAG_SL_SUBQ int  tlag_sl_sub_<pc>(cpool, f, cx)      0 = returned, 1 = trapped
    slices                          -> TLAG_SL_SEGQ void tlag_sl_inv_<i> / tlag_sl_next_<j>(cpool, f, cx)
    TLAG_SL_INV_LIST(X) / TLAG_SL_NEXT_LIST(X), TLAG_SL_W, TLAG_SL_USZ, TLAG_SL_FRAME, program length + FNV-1a

Events are macros the including engine defines: TLAG_SL_EMIT(aid, dirty_table), TLAG_SL_EMITW(aid, words) (scalar
form: the successor already packed), TLAG_SL_GEN(), TLAG_SL_ASSERT(id), TLAG_SL_INVF(i), TLAG_SL_TRAP(code, line).
The CUDA engine (csrc/tlag_engine.cu, -DTLAG_SLICED_INC) and the CPU bytecode engine (oracle/tlag_cpu.c, the
no-GPU semantics check of tests/test_sliced.py) include the same file.

Two forms of the frame:
  * array form (any model): `f[...]` is the per-thread frame array exactly as under the interpreter;
  * scalar form (small call-free models, `scalar=True`): every frame word that is only ever addressed statically is a C
    local of its own (`r113 = r97 & r105;`) -- registers after nvcc's SSA construction, no local-memory frame at all --
    and only the regions that some instruction indexes dynamically (bitset scans, `f[x]` with a run-time x) stay in a
    small array `m[]`; unpack and pack are written out per slot with constant shifts.

The statements restate csrc/tlag_vm_exec.inc op by op: the interpreter and this emitter are two implementations of the
ISA that the fixtures compare bit for bit (fingerprint digests)."""
from __future__ import annotations

import numpy as np

import hashlib

from .bytecode import OP

_NAME = {v: k for k, v in OP.items()}
_COND_J = {"JEQ", "JNE", "JLT", "JGE", "JEQI", "JNEI", "JLTI", "JGEI", "JBT", "JBF", "JBTI", "JBFI"}
_COND_I = {"JZ", "JNZ", "JNEG", "JGEZ"}
_CMP = {"JEQ": "==", "JNE": "!=", "JLT": "<", "JGE": ">=", "JEQI": "==", "JNEI": "!=", "JLTI": "<", "JGEI": ">=",
        "JZ": "==", "JNZ": "!=", "JNEG": "<", "JGEZ": ">="}
_BIN = {"ADD": "(int32_t)((uint32_t){x} + (uint32_t){y})", "SUB": "(int32_t)((uint32_t){x} - (uint32_t){y})",
        "MUL": "(int32_t)((uint32_t){x} * (uint32_t){y})", "LT": "{x} < {y}", "LE": "{x} <= {y}",
        "EQ": "{x} == {y}", "NE": "{x} != {y}", "AND": "({x} != 0) & ({y} != 0)", "OR": "({x} != 0) | ({y} != 0)"}
_BINI = {"ADDI": "(int32_t)((uint32_t){x} + (uint32_t)({J}))", "MULI": "(int32_t)((uint32_t){x} * (uint32_t)({J}))",
         "EQI": "{x} == ({J})", "NEI": "{x} != ({J})", "LTI": "{x} < ({J})", "LEI": "{x} <= ({J})",
         "GTI": "{x} > ({J})", "GEI": "{x} >= ({J})", "SHRI": "(int32_t)((uint32_t){x} >> (({J}) & 31))",
         "ANDI": "{x} & ({J})"}
_WORDWISE = {"BOR": "{x} | {y}", "BAND": "{x} & {y}", "BANDN": "{x} & ~{y}"}
SCALAR_MAX_FRAME = 1024     # scalar form only below this frame size (statements are unrolled word by word)


class SliceError(Exception):
    pass


def model_key(cm) -> str:
    """Identifies the generated code: program words, entry points (the constant pool is folded in through them)."""
    h = hashlib.sha256()
    h.update(np.ascontiguousarray(cm.code, dtype=np.uint64).tobytes())
    h.update(np.ascontiguousarray(cm.cpool, dtype=np.int32).tobytes())
    h.update(repr(sorted(cm.entries.items())).encode())
    return h.hexdigest()[:16]


def _imm28(v: int) -> int:
    v &= 0xFFFFFFF
    return v - (1 << 28) if v & (1 << 27) else v


def _k14(b: int) -> int:
    return b - (1 << 14) if b & (1 << 13) else b


class Ins:
    __slots__ = ("k", "op", "a", "b", "c", "d", "I", "J", "w")

    def __init__(self, k, w):
        self.k, self.w = k, w
        self.op = _NAME.get(w & 0xFF)
        self.a, self.b, self.c, self.d = (w >> 8) & 0x3FFF, (w >> 22) & 0x3FFF, (w >> 36) & 0x3FFF, (w >> 50) & 0x3FFF
        self.I, self.J = _imm28(w >> 22), _imm28(w >> 36)

    def target(self):
        if self.op in _COND_J:
            return self.J
        if self.op in _COND_I or self.op in ("JMP", "CALL"):
            return self.I
        return None


STATIC_WORDS = 16    # scalar form: run-time indexed regions up to this many words are addressed through select chains


def dyn_accesses(ins: Ins):
    """[(base, nwords or None)] of the frame regions instruction `ins` addresses with a run-time index."""
    op = ins.op
    if op == "BNEXT":
        return [(ins.b, (ins.d + 31) // 32)] if ins.d > 32 else []      # one word: written out statically
    if op in ("BSET", "BCLR", "JBT", "JBF", "STX", "SINS"):
        return [(ins.a, None)]
    if op in ("BTEST", "LDX", "SFIND"):
        return [(ins.b, None)]
    return []


MIN_SLICE = 256      # adjacent slices are merged into one kernel until it holds at least this many bytecode instructions


class Plan:
    """Slices of a compiled model: prologues, slice ranges (closed under their jumps), subroutine regions."""

    def __init__(self, cm, min_slice=None):
        self.cm = cm
        self.min_slice = MIN_SLICE if min_slice is None else int(min_slice)
        self.ins = [Ins(k, int(w)) for k, w in enumerate(np.ascontiguousarray(cm.code, dtype=np.uint64))]
        n = len(self.ins)
        halts = [i.k for i in self.ins if i.op == "HALT"]
        e_inv, e_next = int(cm.entries["inv"]), int(cm.entries["next"])
        if len(halts) != 2 or not (e_inv <= halts[0] < e_next <= halts[1]):
            raise SliceError("program is not `inv ... HALT next ... HALT`")
        segs = getattr(cm, "segments", None) or {}
        self.subs = self._subroutines(halts[1] + 1, n)
        self.progs = {}
        for name, entry, halt in (("inv", e_inv, halts[0]), ("next", e_next, halts[1])):
            cuts = sorted(set(c for c in (segs.get(name) or []) if entry <= c <= halt))
            if not cuts:
                cuts = [entry]
            pro, closed = self._close(entry, cuts, halt)
            # Every kernel re-reads the packed frontier (Paxos b4: 15.5 GB per launch at the peak levels) and pays a
            # launch + tail: tiny slices (Phase1a(b): 7 instructions) are merged with their neighbours.  Adjacent
            # slices are consecutive code whose only exit is falling into the next one, so a group is just a coarser cut.
            merged, cur = [], None
            for s_, e_ in closed:
                if cur is None:
                    cur = [s_, e_]
                else:
                    cur[1] = e_
                if cur[1] - cur[0] >= self.min_slice:
                    merged.append(tuple(cur))
                    cur = None
            if cur is not None:
                if merged and cur[1] - cur[0] < self.min_slice // 2:
                    merged[-1] = (merged[-1][0], cur[1])
                else:
                    merged.append(tuple(cur))
            self.progs[name] = (pro, merged)

    def _subroutines(self, lo, hi):
        entries = sorted(set(i.I for i in self.ins if i.op == "CALL"))
        for e in entries:
            if not lo <= e < hi:
                raise SliceError(f"CALL target {e} inside a main program")
        regions = {}
        for j, e in enumerate(entries):
            end = entries[j + 1] if j + 1 < len(entries) else hi
            for i in self.ins[e:end]:
                t = i.target()
                if t is not None and i.op != "CALL" and not e <= t < end:
                    raise SliceError(f"subroutine at {e}: jump from {i.k} to {t} leaves it")
                if i.op in ("EMIT", "EMITD", "GEN", "HALT"):
                    raise SliceError(f"subroutine at {e} contains {i.op}")
            regions[e] = end
        if entries and entries[0] != lo:
            raise SliceError("code between the last HALT and the first subroutine")
        if not entries and lo != hi:
            raise SliceError("unreachable code after the last HALT")
        return regions

    def _close(self, entry, cuts, halt):
        """-> (prologue range, [slice ranges]); neighbours are merged until every jump of a slice stays inside it or
        goes to its end (= falls into the next slice = "this disjunct is done")."""
        bounds = cuts + [halt]
        # the prologue may only fall into the first slice
        for i in self.ins[entry:cuts[0]]:
            t = i.target()
            if t is not None and i.op != "CALL" and not entry <= t <= cuts[0]:
                bounds = [entry, halt]
                break
            if i.op in ("EMIT", "EMITD", "GEN"):
                bounds = [entry, halt]
                break
        changed = True
        while changed:
            changed = False
            for j in range(len(bounds) - 1):
                s, e = bounds[j], bounds[j + 1]
                bad = None
                for i in self.ins[s:e]:
                    t = i.target()
                    if t is not None and i.op != "CALL" and not s <= t <= e:
                        bad = t
                        break
                if bad is None:
                    continue
                if bad > e:
                    bounds = [b for b in bounds if not (e <= b < bad)] if bad <= halt else None
                else:
                    bounds = [b for b in bounds if not (bad < b <= s)] if bad >= bounds[0] else None
                if bounds is None:
                    raise SliceError(f"jump to {bad} leaves the program")
                if bounds[-1] != halt:
                    bounds.append(halt)
                changed = True
                break
        return (entry, bounds[0]), [(bounds[j], bounds[j + 1]) for j in range(len(bounds) - 1)]

    def calls_of(self, ranges):
        """transitive closure of the subroutines called from the given pc ranges"""
        seen, todo = set(), []
        for s, e in ranges:
            todo += [i.I for i in self.ins[s:e] if i.op == "CALL"]
        while todo:
            t = todo.pop()
            if t in seen:
                continue
            seen.add(t)
            todo += [i.I for i in self.ins[t:self.subs[t]] if i.op == "CALL"]
        return seen


class Emitter:
    def __init__(self, cm, scalar=False, min_slice=None):
        self.cm = cm
        # grouping pays in the scalar form (Paxos b4: 0.41 -> 0.39 s per BFS at 256, 0.56 s at 512: register pressure);
        # in the array form a group unpacks the union of its slices' live slots (raft: 0.95 -> 1.02 s), so none there
        self.plan = Plan(cm, (MIN_SLICE if scalar else 0) if min_slice is None else min_slice)
        self.usz = int(cm.state_words_unpacked)
        self.frame = int(cm.frame_words)
        self.layout = [tuple(int(x) for x in r) for r in np.asarray(cm.layout).reshape(-1, 3)]
        self.cpool = [int(x) for x in np.asarray(cm.cpool)]
        self.W = int(cm.W)
        self.scalar = bool(scalar)
        self.dyn_index = {}
        if self.scalar:
            if self.plan.subs:
                raise SliceError("scalar form: the program has subroutines")
            if self.frame > SCALAR_MAX_FRAME:
                raise SliceError("scalar form: frame too large")
            self._find_dyn()

    # ---- scalar form: which words stay in memory ---------------------------------------------------------------
    def _static_ok(self, i: Ins, base, nw) -> bool:
        """scalar form: can this run-time indexed access be written with compile-time word names (a select chain over
        the region's words)?  Then the region needs no memory at all."""
        n = self._extent(i, base, nw)
        if i.op in ("LDX", "STX"):
            return n <= 4 * STATIC_WORDS and n // max(1, i.d) <= STATIC_WORDS
        if i.op in ("SFIND", "SINS"):
            return False
        return n <= STATIC_WORDS

    def _find_dyn(self, ranges=None):
        """Frame words that some instruction of the given pc ranges (default: the whole program) addresses with a
        run-time index in a way that needs memory, widened to the allocation blocks they lie in.  Computed per slice
        function: temporaries are stack-allocated by the lowering, so a word that is a bitset under scan in one slice
        is a plain scalar in the others.  Small regions (<= STATIC_WORDS words) are not in here: their accesses are
        written as select chains over the words' C locals (_static_ok)."""
        blocks = getattr(self.cm, "blocks", None)
        if not blocks:
            raise SliceError("scalar form needs the allocation blocks of the lowering (cm.blocks)")
        dyn = set()
        ins = self.plan.ins if ranges is None else [i for s, e in ranges for i in self.plan.ins[s:e]]
        for i in ins:
            if i.op in ("SFIND", "SINS"):
                raise SliceError("scalar form: sparse containers")
            for base, nw in dyn_accesses(i):
                if self._static_ok(i, base, nw):
                    continue
                dyn.update(range(base, base + self._extent(i, base, nw)))
        self.dyn_index = {w: j for j, w in enumerate(sorted(dyn))}

    def R(self, k: int) -> str:
        """C lvalue of frame word k"""
        if not self.scalar:
            return f"f[{k}]"
        j = self.dyn_index.get(k)
        return f"r{k}" if j is None else f"m[{j}]"

    def SEL(self, base: int, n: int, idx: str) -> str:
        """C rvalue of frame word base + idx for a run-time idx in 0..n-1, as a select chain over the n words"""
        e = self.R(base + n - 1)
        for j in range(n - 2, -1, -1):
            e = f"({idx} == {j}u ? {self.R(base + j)} : {e})"
        return e

    def SEL2(self, base: int, cnt: int, d: int, j: int, idx: str) -> str:
        """word j of element idx (0..cnt-1) of an array of d-word elements at base, as a select chain"""
        e = self.R(base + (cnt - 1) * d + j)
        for k in range(cnt - 2, -1, -1):
            e = f"({idx} == {k}u ? {self.R(base + k * d + j)} : {e})"
        return e

    def D(self, base: int, idx: str) -> str:
        """C lvalue of frame word base + idx (run-time idx): the region is in memory in both forms"""
        if not self.scalar:
            return f"f[{base}u + {idx}]"
        return f"m[{self.dyn_index[base]}u + {idx}]"

    def _run(self, base, n):
        """contiguous words base..base+n: are they one run in memory (array form: always)?"""
        if not self.scalar:
            return True
        js = [self.dyn_index.get(base + i) for i in range(n)]
        return all(j is not None for j in js) and all(js[i] == js[0] + i for i in range(n))

    # ---- liveness (per slice function) ------------------------------------------------------------------------
    # Every slice kernel starts from the packed state; under the interpreter the state was unpacked once and the primed
    # copy initialised once per state, here that would be paid per slice (raft: 589 + 589 word stores x 36 kernels).
    # A backward liveness pass over the slice's control-flow graph finds the frame words a slice actually reads before
    # writing them: only those slots are unpacked, copies / fills of words nobody reads afterwards are trimmed to the
    # live sub-ranges, and pure instructions whose result is dead are dropped.
    def _extent(self, i: Ins, base, nw):
        if nw is not None:
            return nw
        blocks = getattr(self.cm, "blocks", None) or []
        ends = [b + n for b, n in blocks if b <= base < b + n]
        return max(ends) - base if ends else (i.d if i.op in ("LDX", "STX") else 1)

    def _sub_reads(self, e):
        """words a subroutine (and its callees) may read"""
        memo = self.__dict__.setdefault("_sub_reads_memo", {})
        if e not in memo:
            memo[e] = 0
            m = 0
            for i in self.plan.ins[e:self.plan.subs[e]]:
                m |= self.rw(i)[0]
            memo[e] = m
        return memo[e]

    def rw(self, i: Ins):
        """-> (words read, words certainly overwritten, droppable when the overwritten words are dead) as bit masks"""
        mk = lambda base, n: (((1 << n) - 1) << base) if n > 0 else 0
        op, a, b, c, d, I, J = i.op, i.a, i.b, i.c, i.d, i.I, i.J
        dyn = 0
        for base, nw in dyn_accesses(i):
            dyn |= mk(base, self._extent(i, base, nw))
        if op in _BIN:
            return mk(b, 1) | mk(c, 1), mk(a, 1), True
        if op in _BINI or op in ("MOV", "NEG", "NOT"):
            return mk(b, 1), mk(a, 1), True
        if op in ("JEQ", "JNE", "JLT", "JGE"):
            return mk(a, 1) | mk(b, 1), 0, False
        if op in ("JEQI", "JNEI", "JLTI", "JGEI") or op in _COND_I:
            return mk(a, 1), 0, False
        if op in ("JBT", "JBF"):
            return mk(b, 1) | dyn, 0, False
        if op in ("JBTI", "JBFI"):
            return mk(a + (b >> 5), 1), 0, False
        if op in ("JMP", "GEN", "ASSERTF", "INVF", "TRAP", "HALT", "RET"):
            return 0, 0, False
        if op in ("LI", "LIW"):
            return 0, mk(a, 1), True
        if op == "MOVN":
            return mk(b, c), mk(a, c), True
        if op == "ZERO":
            return 0, mk(a, b), True
        if op == "LDC":
            return 0, mk(a, d), True
        if op in ("DIV", "MOD"):
            return mk(b, 1) | mk(c, 1), mk(a, 1), False
        if op == "EQN":
            return mk(b, d) | mk(c, d), mk(a, 1), True
        if op == "LDX":
            return mk(c, 1) | dyn, mk(a, d), True
        if op == "STX":
            return mk(b, 1) | mk(c, d), 0, False
        if op == "TBL":
            return mk(d, 1), mk(a, 1), True
        if op == "TBLT":
            return mk(d, 1), mk(a, 1), False
        if op in ("BSET", "BCLR"):
            return mk(b, 1) | dyn, 0, False
        if op == "BTEST":
            return mk(c, 1) | dyn, mk(a, 1), True
        if op in _WORDWISE:
            return mk(b, d) | mk(c, d), mk(a, d), True
        if op == "BISZ":
            return mk(b, c), mk(a, 1), True
        if op == "BSUB":
            return mk(b, d) | mk(c, d), mk(a, 1), True
        if op == "BCNT":
            return mk(b, c), mk(a, 1), True
        if op == "BNEXT":
            return mk(c, 1) | mk(b, (d + 31) // 32), mk(a, 1), True
        if op == "BFILL":
            return mk(a, (b + 31) // 32), 0, False
        if op == "BSETI":
            return mk(a + ((I & 0xFFFFFFFF) >> 5), 1), 0, False
        if op == "BTESTI":
            return mk(b + ((J & 0xFFFFFFFF) >> 5), 1), mk(a, 1), True
        if op == "UCLAMP":
            return mk(a, 1), 0, False
        if op == "MADI":
            return mk(a, 1) | mk(c, 1), 0, False
        if op == "BANDC":
            return mk(b, J & 0xFF), mk(a, J & 0xFF), True
        if op == "LEXLT":
            return mk(b, d) | mk(c, d), mk(a, 1), True
        if op == "SFIND":
            return mk(c, d & 127) | dyn, mk(a, 1), True
        if op == "SINS":
            return mk(b, d >> 7) | mk(c, 1) | dyn, 0, False
        if op == "CALL":
            return self._sub_reads(I), 0, False
        if op in ("EMIT", "EMITD"):
            p_off = self.usz
            if op == "EMITD" and I > 0:
                n = self.cpool[I]
                slots = [s_ for r in range(n) for s_ in range(self.cpool[I + 1 + 3 * r], self.cpool[I + 1 + 3 * r] + self.cpool[I + 2 + 3 * r])]
            else:
                slots = range(len(self.layout))
            m = 0
            for s_ in slots:
                m |= 1 << (p_off + self.layout[s_][0])
            return m, 0, False
        raise SliceError(f"no read/write description for opcode {op}")

    def liveness(self, pro, seg):
        """live-out word masks per pc for the function `prologue + slice`; also the live-in mask of the function"""
        (p0, p1), (s, e) = pro, seg
        order = list(range(p0, p1)) + list(range(s, e))
        END = -1
        succ = {}
        for k in order:
            i = self.plan.ins[k]
            out = []
            nxt = (k + 1 if k + 1 < p1 else s) if k < p1 and p0 <= k else (k + 1 if k + 1 < e else END)
            if i.op not in ("JMP", "TRAP", "RET", "HALT"):
                out.append(nxt)
            if i.op == "HALT":
                out.append(END)
            t = i.target()
            if t is not None and i.op != "CALL":
                if p0 <= k < p1 and t == p1:
                    t = s
                out.append(END if t == e else t)
            succ[k] = out
        info = {k: self.rw(self.plan.ins[k]) for k in order}
        live_in = {k: 0 for k in order}
        live_in[END] = 0
        live_out = {k: 0 for k in order}
        changed = True
        while changed:
            changed = False
            for k in reversed(order):
                lo = 0
                for t in succ[k]:
                    lo |= live_in[t]
                rd, kl, _ = info[k]
                i = self.plan.ins[k]
                if i.op in ("MOVN", "BANDC") or i.op in _WORDWISE:
                    # element-wise: a source word is read only if the destination word it feeds is read afterwards
                    n_ = i.c if i.op == "MOVN" else ((i.J & 0xFF) if i.op == "BANDC" else i.d)
                    sel = (lo >> i.a) & ((1 << n_) - 1)
                    rd = sel << i.b
                    if i.op in _WORDWISE:
                        rd |= sel << i.c
                li = rd | (lo & ~kl)
                if lo != live_out[k] or li != live_in[k]:
                    live_out[k], live_in[k] = lo, li
                    changed = True
        return live_out, (live_in[order[0]] if order else 0), info

    # ---- one instruction -----------------------------------------------------------------------------------
    @staticmethod
    def _runs(base, n, live):
        """maximal runs (offset, length) of the words base..base+n that are in the live mask (None: all of them)"""
        if live is None:
            return [(0, n)] if n > 0 else []
        out, j = [], 0
        while j < n:
            if (live >> (base + j)) & 1:
                k = j
                while k < n and (live >> (base + k)) & 1:
                    k += 1
                out.append((j, k - j))
                j = k
            else:
                j += 1
        return out

    def stmt(self, i: Ins, goto, rv: str, live=None) -> str:
        """C statement(s) for instruction i.  goto(t) -> text of a jump to pc t; rv: return value text on a trap;
        live: mask of the frame words that are read after this instruction (None = unknown: write everything)."""
        R, D = self.R, self.D
        op, a, b, c, d, I, J = i.op, i.a, i.b, i.c, i.d, i.I, i.J
        runs = lambda n: self._runs(a, n, live)
        words = lambda n: [o + j for o, ln in runs(n) for j in range(ln)]
        trap = lambda code, line: f"{{ TLAG_SL_TRAP({code}, {line}); return{rv}; }}"
        if op in _BIN:
            return f"{R(a)} = {_BIN[op].format(x=R(b), y=R(c))};"
        if op in _BINI:
            return f"{R(a)} = {_BINI[op].format(x=R(b), J=J)};"
        if op in ("JEQ", "JNE", "JLT", "JGE"):
            return f"if ({R(a)} {_CMP[op]} {R(b)}) {goto(J)}"
        if op in ("JEQI", "JNEI", "JLTI", "JGEI"):
            return f"if ({R(a)} {_CMP[op]} ({_k14(b)})) {goto(J)}"
        if op in _COND_I:
            return f"if ({R(a)} {_CMP[op]} 0) {goto(I)}"
        st_ = self.scalar and bool(dyn_accesses(i)) and all(self._static_ok(i, bb, nn) for bb, nn in dyn_accesses(i))
        if st_:
            base_, nw_ = dyn_accesses(i)[0]
            nw_ = self._extent(i, base_, nw_)
            if op in ("JBT", "JBF"):
                return (f"{{ const uint32_t i_ = (uint32_t){R(b)}; const uint32_t w_ = (uint32_t){self.SEL(a, nw_, '(i_ >> 5)')}; "
                        f"if ((((w_ >> (i_ & 31)) & 1u) != 0) == {1 if op == 'JBT' else 0}) {goto(J)} }}")
            if op == "BTEST":
                return (f"{{ const uint32_t i_ = (uint32_t){R(c)}; const uint32_t w_ = (uint32_t){self.SEL(b, nw_, '(i_ >> 5)')}; "
                        f"{R(a)} = (int32_t)((w_ >> (i_ & 31)) & 1u); }}")
            if op in ("BSET", "BCLR"):
                upd = "|= (int32_t)m_" if op == "BSET" else "&= ~(int32_t)m_"
                return (f"{{ const uint32_t i_ = (uint32_t){R(b)}, w_ = i_ >> 5, m_ = 1u << (i_ & 31); "
                        + " ".join(f"if (w_ == {j}u) {R(a + j)} {upd};" for j in range(nw_)) + " }")
            if op == "BNEXT":
                out_ = [f"{{ int32_t cur_ = {R(c)} + 1; int32_t res_ = -1; int done_ = 0;"]
                for j in range(nw_):
                    out_.append(f"if (!done_ && cur_ < {32 * (j + 1)}) {{ const uint32_t sh_ = cur_ > {32 * j} ? (uint32_t)(cur_ - {32 * j}) : 0u; "
                                f"const uint32_t word_ = (uint32_t){R(b + j)} >> sh_; "
                                f"if (word_) {{ const int32_t cand_ = {32 * j} + (int32_t)sh_ + tlag_ffs(word_) - 1; "
                                f"if ((uint32_t)cand_ < {d}u) res_ = cand_; done_ = 1; }} else cur_ = {32 * (j + 1)}; }}")
                out_.append(f"{R(a)} = res_; }}")
                return " ".join(out_)
            if op == "LDX":
                cnt_ = max(1, nw_ // max(1, d))
                return (f"{{ const uint32_t x_ = (uint32_t){R(c)}; "
                        + " ".join(f"{R(a + j)} = {self.SEL2(b, cnt_, d, j, 'x_')};" for j in range(d)) + " }")
            if op == "STX":
                cnt_ = max(1, nw_ // max(1, d))
                return (f"{{ const uint32_t x_ = (uint32_t){R(b)}; "
                        + " ".join(f"if (x_ == {k_}u) {{ " + " ".join(f"{R(a + k_ * d + j)} = {R(c + j)};" for j in range(d)) + " }"
                                   for k_ in range(cnt_)) + " }")
        if op in ("JBT", "JBF"):
            return (f"{{ const uint32_t i_ = (uint32_t){R(b)}; if (((((uint32_t){D(a, '(i_ >> 5)')} >> (i_ & 31)) & 1u) != 0) == "
                    f"{1 if op == 'JBT' else 0}) {goto(J)} }}")
        if op in ("JBTI", "JBFI"):
            return f"if (((((uint32_t){R(a + (b >> 5))} >> {b & 31}) & 1u) != 0) == {1 if op == 'JBTI' else 0}) {goto(J)}"
        if op == "JMP":
            return goto(I)
        if op == "LI":
            return f"{R(a)} = {I};"
        if op == "LIW":           # the constant pool belongs to this model: its words are literals here
            return f"{R(a)} = {self.cpool[I]};"
        if op == "MOV":
            return f"{R(a)} = {R(b)};"
        if op == "MOVN":
            if self.scalar:
                ws = words(c)
                order = ws if a <= b else ws[::-1]
                return " ".join(f"{R(a + j)} = {R(b + j)};" for j in order)
            if a <= b:
                return " ".join(f"for (uint32_t i_ = {o}u; i_ < {o + ln}u; ++i_) f[{a} + i_] = f[{b} + i_];" for o, ln in runs(c))
            return " ".join(f"for (uint32_t i_ = {o + ln}u; i_-- > {o}u;) f[{a} + i_] = f[{b} + i_];" for o, ln in runs(c)[::-1])
        if op == "ZERO":
            if self.scalar:
                return " ".join(f"{R(a + j)} = 0;" for j in words(b))
            return " ".join(f"for (uint32_t i_ = {o}u; i_ < {o + ln}u; ++i_) f[{a} + i_] = 0;" for o, ln in runs(b))
        if op == "LDC":
            if self.scalar or d <= 4:
                return " ".join(f"{R(a + j)} = {self.cpool[I + j]};" for j in words(d))
            return " ".join(f"for (uint32_t i_ = {o}u; i_ < {o + ln}u; ++i_) f[{a} + i_] = tlag_cp(cpool, {I} + (int32_t)i_);"
                            for o, ln in runs(d))
        if op == "NEG":
            return f"{R(a)} = -{R(b)};"
        if op == "NOT":
            return f"{R(a)} = !{R(b)};"
        if op == "EQN":
            if self.scalar:
                return f"{R(a)} = " + " & ".join(f"({R(b + j)} == {R(c + j)})" for j in range(d)) + ";" if d else f"{R(a)} = 1;"
            return f"{{ int32_t e_ = 1; for (uint32_t i_ = 0; i_ < {d}u; ++i_) e_ &= (f[{b} + i_] == f[{c} + i_]); f[{a}] = e_; }}"
        if op == "LDX":
            if self.scalar:
                return (f"{{ const uint32_t x_ = (uint32_t){R(c)} * {d}u; "
                        + " ".join(f"{R(a + j)} = {D(b, f'x_ + {j}u')};" for j in range(d)) + " }")
            return (f"{{ const uint32_t base_ = {b}u + (uint32_t)f[{c}] * {d}u; "
                    f"for (uint32_t i_ = 0; i_ < {d}u; ++i_) f[{a} + i_] = f[base_ + i_]; }}")
        if op == "STX":
            if self.scalar:
                return (f"{{ const uint32_t x_ = (uint32_t){R(b)} * {d}u; "
                        + " ".join(f"{D(a, f'x_ + {j}u')} = {R(c + j)};" for j in range(d)) + " }")
            return (f"{{ const uint32_t base_ = {a}u + (uint32_t)f[{b}] * {d}u; "
                    f"for (uint32_t i_ = 0; i_ < {d}u; ++i_) f[base_ + i_] = f[{c} + i_]; }}")
        if op == "TBL":
            return f"{R(a)} = tlag_cp(cpool, {I} + {R(d)});"
        if op == "TBLT":
            return (f"{{ const int32_t v_ = tlag_cp(cpool, {I} + {R(d)}); if (v_ == (int32_t)0x80000000) {trap(1, 0)} "
                    f"{R(a)} = v_; }}")
        if op == "BSET":
            return f"{{ const uint32_t i_ = (uint32_t){R(b)}; {D(a, '(i_ >> 5)')} |= (int32_t)(1u << (i_ & 31)); }}"
        if op == "BCLR":
            return f"{{ const uint32_t i_ = (uint32_t){R(b)}; {D(a, '(i_ >> 5)')} &= ~(int32_t)(1u << (i_ & 31)); }}"
        if op == "BTEST":
            return (f"{{ const uint32_t i_ = (uint32_t){R(c)}; "
                    f"{R(a)} = (int32_t)(((uint32_t){D(b, '(i_ >> 5)')} >> (i_ & 31)) & 1u); }}")
        if op in _WORDWISE:
            if self.scalar:
                return " ".join(f"{R(a + j)} = {_WORDWISE[op].format(x=R(b + j), y=R(c + j))};" for j in words(d))
            return " ".join(f"for (uint32_t i_ = {o}u; i_ < {o + ln}u; ++i_) f[{a} + i_] = "
                            f"{_WORDWISE[op].format(x=f'f[{b} + i_]', y=f'f[{c} + i_]')};" for o, ln in runs(d))
        if op == "BISZ":
            if self.scalar:
                return f"{R(a)} = ((" + " | ".join(R(b + j) for j in range(c)) + ") == 0);" if c else f"{R(a)} = 1;"
            return f"{{ int32_t z_ = 1; for (uint32_t i_ = 0; i_ < {c}u; ++i_) z_ &= (f[{b} + i_] == 0); f[{a}] = z_; }}"
        if op == "BSUB":
            if self.scalar:
                return (f"{R(a)} = ((" + " | ".join(f"({R(b + j)} & ~{R(c + j)})" for j in range(d)) + ") == 0);"
                        if d else f"{R(a)} = 1;")
            return (f"{{ int32_t z_ = 1; for (uint32_t i_ = 0; i_ < {d}u; ++i_) z_ &= ((f[{b} + i_] & ~f[{c} + i_]) == 0); "
                    f"f[{a}] = z_; }}")
        if op == "BCNT":
            if self.scalar:
                return f"{R(a)} = " + " + ".join(f"tlag_popc((uint32_t){R(b + j)})" for j in range(c)) + ";" if c else f"{R(a)} = 0;"
            return (f"{{ int32_t n_ = 0; for (uint32_t i_ = 0; i_ < {c}u; ++i_) n_ += tlag_popc((uint32_t)f[{b} + i_]); "
                    f"f[{a}] = n_; }}")
        if op == "BNEXT" and d <= 32 and self.scalar:
            return (f"{{ const uint32_t cur_ = (uint32_t)({R(c)} + 1); int32_t res_ = -1; if (cur_ < {d}u) {{ "
                    f"const uint32_t word_ = (uint32_t){R(b)} >> cur_; "
                    f"if (word_) {{ const int32_t cand_ = (int32_t)cur_ + tlag_ffs(word_) - 1; if ((uint32_t)cand_ < {d}u) res_ = cand_; }} }} "
                    f"{R(a)} = res_; }}")
        if op == "BNEXT":
            return (f"{{ int32_t cur_ = {R(c)} + 1; int32_t res_ = -1; "
                    f"while ((uint32_t)cur_ < {d}u) {{ "
                    f"const uint32_t word_ = (uint32_t){D(b, '((uint32_t)cur_ >> 5)')} >> ((uint32_t)cur_ & 31); "
                    f"if (word_) {{ const int32_t cand_ = cur_ + tlag_ffs(word_) - 1; if ((uint32_t)cand_ < {d}u) res_ = cand_; break; }} "
                    f"cur_ = (int32_t)(((uint32_t)cur_ | 31u) + 1u); }} {R(a)} = res_; }}")
        if op == "BFILL":
            nw = (b + 31) // 32
            out = []
            for j in range(nw):
                bits = min(32, b - 32 * j)
                mask = 0xFFFFFFFF if bits == 32 else (1 << bits) - 1
                out.append(f"{R(a + j)} |= (int32_t)0x{mask:x}u;")
            return " ".join(out)
        if op == "BSETI":
            ii = I & 0xFFFFFFFF
            return f"{R(a + (ii >> 5))} |= (int32_t)0x{1 << (ii & 31):x}u;"
        if op == "BTESTI":
            ii = J & 0xFFFFFFFF
            return f"{R(a)} = (int32_t)(((uint32_t){R(b + (ii >> 5))} >> {ii & 31}) & 1u);"
        if op == "UCLAMP":
            return f"if ((uint32_t){R(a)} >= (uint32_t)({I})) {R(a)} = -1;"
        if op == "MADI":
            return f"{R(a)} = (int32_t)((uint32_t){R(a)} * (uint32_t)({_k14(b)}) + (uint32_t){R(c)});"
        if op == "BANDC":
            n_, base = J & 0xFF, (J & 0xFFFFFFFF) >> 8
            if self.scalar:
                # the mask words are compile-time constants of this model: fold them into the code
                return " ".join(f"{R(a + j)} = {R(b + j)} & (int32_t)0x{self.cpool[base + j] & 0xFFFFFFFF:x}u;" for j in words(n_))
            return " ".join(f"for (uint32_t i_ = {o}u; i_ < {o + ln}u; ++i_) f[{a} + i_] = f[{b} + i_] & tlag_cp(cpool, {base} + (int32_t)i_);"
                            for o, ln in runs(n_))
        if op == "DIV":
            return (f"{{ const int32_t x_ = {R(b)}, y_ = {R(c)}; if (y_ == 0) {trap(1, 0)} "
                    f"int32_t q_ = x_ / y_; if ((x_ % y_ != 0) && ((x_ < 0) != (y_ < 0))) --q_; {R(a)} = q_; }}")
        if op == "MOD":
            return (f"{{ const int32_t x_ = {R(b)}, y_ = {R(c)}; if (y_ <= 0) {trap(1, 0)} "
                    f"int32_t r_ = x_ % y_; if (r_ < 0) r_ += y_; {R(a)} = r_; }}")
        if op == "LEXLT":
            if self.scalar:
                expr = "0"
                for j in range(d - 1, -1, -1):
                    expr = f"({R(b + j)} != {R(c + j)} ? ({R(b + j)} < {R(c + j)}) : {expr})"
                return f"{R(a)} = {expr};"
            return (f"{{ int32_t r_ = 0; for (uint32_t i_ = 0; i_ < {d}u; ++i_) {{ const int32_t x_ = f[{b} + i_], y_ = f[{c} + i_]; "
                    f"if (x_ != y_) {{ r_ = x_ < y_; break; }} }} f[{a}] = r_; }}")
        stride, keyw = d >> 7, d & 127
        if op in ("SFIND", "SINS") and self.scalar:
            raise SliceError("scalar form: sparse containers")
        if op == "SFIND":
            return (f"{{ const int32_t n_ = f[{b}]; int32_t r_ = -1; for (int32_t i_ = 0; i_ < n_; ++i_) {{ "
                    f"const uint32_t e_ = {b}u + 1u + (uint32_t)i_ * {stride}u; uint32_t k_ = 0; "
                    f"while (k_ < {keyw}u && f[e_ + k_] == f[{c} + k_]) ++k_; "
                    f"if (k_ == {keyw}u) {{ r_ = i_; break; }} if (f[e_ + k_] > f[{c} + k_]) break; }} f[{a}] = r_; }}")
        if op == "SINS":
            return (f"{{ const int32_t n_ = f[{a}]; const int32_t cap_ = f[{c}]; int32_t pos_ = 0; int32_t hit_ = 0; int full_ = 0; "
                    f"for (; pos_ < n_; ++pos_) {{ const uint32_t e_ = {a}u + 1u + (uint32_t)pos_ * {stride}u; uint32_t k_ = 0; "
                    f"while (k_ < {keyw}u && f[e_ + k_] == f[{b} + k_]) ++k_; "
                    f"if (k_ == {keyw}u) {{ hit_ = 1; break; }} if (f[e_ + k_] > f[{b} + k_]) break; }} "
                    f"if (!hit_) {{ if (n_ >= cap_) {{ f[{c}] = 0; full_ = 1; }} else {{ "
                    f"for (int32_t i_ = n_; i_ > pos_; --i_) {{ const uint32_t dst_ = {a}u + 1u + (uint32_t)i_ * {stride}u; "
                    f"for (uint32_t k_ = 0; k_ < {stride}u; ++k_) f[dst_ + k_] = f[dst_ - {stride}u + k_]; }} f[{a}] = n_ + 1; }} }} "
                    f"if (!full_) {{ const uint32_t e_ = {a}u + 1u + (uint32_t)pos_ * {stride}u; "
                    f"for (uint32_t k_ = 0; k_ < {stride}u; ++k_) f[e_ + k_] = f[{b} + k_]; f[{c}] = 1; }} }}")
        if op == "TRAP":
            return trap(a, I)
        if op == "GEN":
            return "TLAG_SL_GEN();"
        if op == "ASSERTF":
            return f"TLAG_SL_ASSERT({I});"
        if op == "INVF":
            return f"TLAG_SL_INVF({I});"
        if op == "EMIT":
            return self.emit_stmt(I, 0, rv)
        if op == "EMITD":
            return self.emit_stmt(a, I, rv)
        if op == "CALL":
            return f"if (tlag_sl_sub_{I}(cpool, f, cx)) return{rv};"
        if op == "RET":
            return "return 0;"
        raise SliceError(f"no template for opcode {op} at pc {i.k}")

    # ---- pack / unpack written out (scalar form) ------------------------------------------------------------------
    def emit_stmt(self, aid, dirty, rv):
        if not self.scalar:
            return f"TLAG_SL_EMIT({aid}, {dirty});"
        W, p_off = self.W, self.usz
        out = [f"{{ uint32_t o_[{W}];"]
        if dirty > 0:
            n = self.cpool[dirty]
            ranges = [(self.cpool[dirty + 1 + 3 * r], self.cpool[dirty + 2 + 3 * r], self.cpool[dirty + 3 + 3 * r]) for r in range(n)]
            out.append(" ".join(f"o_[{j}] = in_[{j}];" for j in range(W)))
        else:
            ranges = [(0, len(self.layout), 0)]
            out.append(" ".join(f"o_[{j}] = 0u;" for j in range(W)))
        changed = set()         # packed words this site may write (the others are the parent's)
        for first, cnt, bitpos in ranges:
            width = sum(self.layout[s][1] for s in range(first, first + cnt))
            if width:
                changed.update(range(bitpos >> 5, (bitpos + width - 1) // 32 + 1))
        for first, cnt, bitpos in ranges:
            for s in range(first, first + cnt):
                off, width, bias = self.layout[s]
                v = f"(uint32_t)({self.R(p_off + off)} - ({bias}))" if bias else f"(uint32_t){self.R(p_off + off)}"
                wi, sh = bitpos >> 5, bitpos & 31
                mask = 0xFFFFFFFF if width >= 32 else (1 << width) - 1
                st = f"{{ const uint32_t v_ = {v};"
                if width < 32:
                    st += f" if (v_ >> {width}) {{ TLAG_SL_TRAP(2, {s}); return{rv}; }}"
                if dirty > 0:
                    st += f" o_[{wi}] = (o_[{wi}] & ~0x{(mask << sh) & 0xFFFFFFFF:x}u) | (v_ << {sh});"
                    if sh + width > 32:
                        st += f" o_[{wi + 1}] = (o_[{wi + 1}] & ~0x{mask >> (32 - sh):x}u) | (v_ >> {32 - sh});"
                else:
                    st += f" o_[{wi}] |= v_ << {sh};"
                    if sh + width > 32:
                        st += f" o_[{wi + 1}] |= v_ >> {32 - sh};"
                st += " }"
                out.append(st)
                bitpos += width
        # A successor equal to its parent (an action that is enabled but changes nothing) is counted and dropped: the
        # parent is a stored state, so the seen-set probe would only find it there.  The test reads registers only.
        diff = " | ".join(f"(o_[{j}] ^ in_[{j}])" for j in sorted(changed if dirty > 0 else range(W)))
        if diff:
            out.append(f"if (TLAG_SL_SKIPSELF && ({diff}) == 0u) TLAG_SL_GEN(); else TLAG_SL_EMITW({aid}, o_); }}")
        else:
            out.append(f"if (TLAG_SL_SKIPSELF) TLAG_SL_GEN(); else TLAG_SL_EMITW({aid}, o_); }}")
        return "\n    ".join(out)

    def unpack_code(self, live_in=None):
        """frame words of the current state from the packed words in_[0..W); live_in: only the slots whose word the
        function reads before writing it"""
        out = []
        bitpos = 0
        for off, width, bias in self.layout:
            wi, sh = bitpos >> 5, bitpos & 31
            if live_in is not None and not (live_in >> off) & 1:
                bitpos += width
                continue
            e = f"(in_[{wi}] >> {sh})" if sh else f"in_[{wi}]"
            if sh + width > 32:
                e = f"({e} | (in_[{wi + 1}] << {32 - sh}))"
            if width < 32:
                e = f"({e} & 0x{(1 << width) - 1:x}u)"
            out.append(f"  {self.R(off)} = (int32_t){e}{f' + ({bias})' if bias else ''};")
            bitpos += width
        return out

    # ---- functions ----------------------------------------------------------------------------------------------
    def _body(self, ranges, end_pc, rv, leaders_extra=(), redirect=None, live=None):
        """statements of the pc ranges (in order); jumps to end_pc go to L_end; redirect = (from pc, to pc): a jump to
        the first is a jump to the second (end of the prologue -> start of this function's slice); live = (live-out
        masks per pc, rw info per pc) from liveness(): dead pure instructions are dropped, dead words not written."""
        targets = set(leaders_extra)
        for s, e in ranges:
            for i in self.plan.ins[s:e]:
                t = i.target()
                if t is not None and i.op != "CALL":
                    targets.add(t)

        def goto(t):
            if redirect is not None and t == redirect[0]:
                t = redirect[1]
            return "goto L_end;" if t == end_pc else f"goto L{t};"
        lines = []
        for s, e in ranges:
            for i in self.plan.ins[s:e]:
                if i.op == "HALT":
                    text = "goto L_end;"
                elif live is not None:
                    lv = live[0][i.k]
                    _rd, kl, pure = live[1][i.k]
                    text = ";" if (pure and kl and not (kl & lv)) else self.stmt(i, goto, rv, lv)   # ";": result never read
                else:
                    text = self.stmt(i, goto, rv)
                lab = f"L{i.k}: " if i.k in targets and i.k != end_pc and (redirect is None or i.k != redirect[0]) else ""
                if text == ";" and not lab:
                    continue
                lines.append(f"  {lab}{{ {text} }}")
        return lines

    def _decls(self):
        if not self.scalar:
            return []
        words = [k for k in range(self.frame) if k not in self.dyn_index]
        out = []
        for j in range(0, len(words), 16):
            out.append("  int32_t " + ", ".join(f"r{k} = 0" for k in words[j:j + 16]) + ";")
        nd = len(self.dyn_index)
        if nd:
            out.append(f"  int32_t m[{nd}];")
            out.append(f"  for (int i_ = 0; i_ < {nd}; ++i_) m[i_] = 0;")
        return out

    def _cpool_fnv(self):
        h = 0xcbf29ce484222325
        for w in self.cpool:
            h = ((h ^ (w & 0xFFFFFFFF)) * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
        return h

    def pieces(self):
        """-> (defs lines, subroutine declarations, {entry: (weight, lines)}, [(kind, j, weight, lines)])"""
        cm, plan = self.cm, self.plan
        code = [i.w for i in plan.ins]
        fnv = 0xcbf29ce484222325
        for w in code:
            fnv = ((fnv ^ w) * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
        (ip, isegs), (np_, nsegs) = plan.progs["inv"], plan.progs["next"]
        n_inv_prog = len(isegs) if len(getattr(cm, "invariants", [])) else 0
        sig = "(const int32_t* __restrict__ cpool, int32_t* __restrict__ f, tlag_sl_cx* __restrict__ cx)"
        ssig = "(const int32_t* __restrict__ cpool, const uint32_t* __restrict__ in_, tlag_sl_cx* __restrict__ cx)"
        defs = [
            "// generated by tla_rust_b200/compile/sliced.py -- do not edit",
            f"// model key {model_key(cm)}: {len(code)} instructions, {n_inv_prog} invariant slices, {len(nsegs)} slices of Next, "
            f"{len(plan.subs)} subroutines, {'scalar' if self.scalar else 'array'} form",
            f"#define TLAG_NATIVE_CODE_LEN {len(code)}u",
            f"#define TLAG_NATIVE_CODE_FNV 0x{fnv:016x}ULL   /* FNV-1a over the 64-bit program words */",
            f"#define TLAG_NATIVE_CPOOL_FNV 0x{self._cpool_fnv():016x}ULL  /* ... over the constant pool (folded into the code) */",
            f"#define TLAG_SL_W {self.W}", f"#define TLAG_SL_USZ {self.usz}", f"#define TLAG_SL_FRAME {self.frame}",
            f"#define TLAG_SL_SCALAR {1 if self.scalar else 0}",
            "#ifndef TLAG_SL_SKIPSELF        /* scalar form: drop successors equal to their parent (CUDA: a run-time switch) */",
            "#define TLAG_SL_SKIPSELF 1", "#endif",
            f"#define TLAG_SL_NINV {n_inv_prog}", f"#define TLAG_SL_NNEXT {len(nsegs)}",
            "#define TLAG_SL_INV_LIST(X) " + " ".join(f"X({j})" for j in range(n_inv_prog)),
            "#define TLAG_SL_NEXT_LIST(X) " + " ".join(f"X({j})" for j in range(len(nsegs))),
        ]
        decls = [f"TLAG_SL_SUBQ int tlag_sl_sub_{e}{sig};" for e in sorted(plan.subs)]
        subs = {}
        for e in sorted(plan.subs):
            lines = [f"TLAG_SL_SUBQ int tlag_sl_sub_{e}{sig} {{"]
            lines += self._body([(e, plan.subs[e])], -1, " 1")
            lines += ["  return 0;", "}"]
            subs[e] = (plan.subs[e] - e, lines)
        slices = []
        can_live = bool(getattr(cm, "blocks", None))        # extents of dynamic accesses come from the allocation blocks
        for name, pro, segs, cnt in (("inv", ip, isegs, n_inv_prog), ("next", np_, nsegs, len(nsegs))):
            for j, (s, e) in enumerate(segs[:cnt]):
                out = [f"// {name} slice {j}: pcs [{s}, {e}) after the prologue [{pro[0]}, {pro[1]})"]
                ranges = [r for r in (pro, (s, e)) if r[1] > r[0]]
                live, live_in = None, None
                if can_live:
                    lo, live_in, info = self.liveness(pro, (s, e))
                    live = (lo, info)
                out.append(f"TLAG_SL_SEGQ void tlag_sl_{name}_{j}{ssig} {{")
                if self.scalar:
                    self._find_dyn(ranges)
                    out += self._decls()
                else:
                    out.append(f"  int32_t f[{self.frame}];")
                    out.append("#ifdef TLAG_SL_POISON")
                    out.append(f"  for (int i_ = 0; i_ < {self.frame}; ++i_) f[i_] = 0x5A5A5A5A;")
                    out.append("#endif")
                ucode = self.unpack_code(live_in)
                out.append(f"  // unpack: {len(ucode)} of {len(self.layout)} slots are read by this slice")
                out += ucode
                # the prologue falls into its first slice; for the others: jump over the slices in between
                if pro[1] > pro[0]:
                    out += self._body([pro], -1, "", leaders_extra=(), redirect=(pro[1], s), live=live)
                    out.append(f"  goto L{s};")
                out += self._body([(s, e)], e, "", leaders_extra=(s,), live=live)
                out += ["  L_end: return;", "}"]
                slices.append((name, j, (pro[1] - pro[0]) + (e - s) + len(ucode) // 4, out))
        return defs, decls, subs, slices

    def emit(self) -> str:
        """everything in one file (the CPU bytecode engine's test build includes it: oracle/tlag_cpu.c)"""
        defs, decls, subs, slices = self.pieces()
        out = list(defs) + decls
        for e in sorted(subs):
            out += subs[e][1]
        for _n, _j, _w, lines in slices:
            out += lines
        out.append("")
        return "\n".join(out)

    def emit_parts(self, nparts, defs_path):
        """The CUDA build: `defs` (constants, included by the engine's translation unit too) and `nparts` translation
        units that each hold a share of the subroutines and slices (balanced by instruction count) with their kernels
        and launchers -- compiled in parallel (nvcc -dc), linked with the engine unit.  -> (defs text, [part texts])"""
        defs, decls, subs, slices = self.pieces()
        items = [("sub", e, w, lines) for e, (w, lines) in subs.items()] + [("slice", (n, j), w, lines) for n, j, w, lines in slices]
        items.sort(key=lambda t: -t[2])
        nparts = max(1, min(nparts, len(items)))
        bins = [[0, []] for _ in range(nparts)]
        for it in items:
            bmin = min(bins, key=lambda b_: b_[0])
            bmin[0] += it[2] + 50
            bmin[1].append(it)
        parts = []
        for k, (_w, its) in enumerate(bins):
            out = [f"// generated by tla_rust_b200/compile/sliced.py -- part {k} of {nparts}; do not edit",
                   f'#define TLAG_SLICED_DEFS "{defs_path}"', '#include "tlag_dev.cuh"',
                   "#undef TLAG_SL_SUBQ", '#define TLAG_SL_SUBQ extern "C" __device__ __noinline__   /* defined in one part, called from any */']
            out += decls
            for kind, _key, _w2, lines in its:
                if kind == "sub":
                    out += lines
            for kind, _key, _w2, lines in its:
                if kind == "slice":
                    out += lines
            out.append('#include "tlag_dev2.cuh"')
            for kind, key, _w2, _lines in its:
                if kind == "slice":
                    nm = "INV" if key[0] == "inv" else "NEXT"
                    out.append(f"TLAG_SL_KERNEL_{nm}({key[1]}) TLAG_SL_LAUNCH_{nm}({key[1]})")
            out.append("")
            parts.append("\n".join(out))
        return "\n".join(defs) + "\n", parts


def emit_sliced(cm, scalar=False, min_slice=None) -> str:
    return Emitter(cm, scalar=scalar, min_slice=min_slice).emit()


def emit_parts(cm, scalar, nparts, defs_path, min_slice=None):
    return Emitter(cm, scalar=scalar, min_slice=min_slice).emit_parts(nparts, defs_path)
