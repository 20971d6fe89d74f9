"""Generated models with a closed-form state space, at the shapes where the device paths change: packed width W (the
scalar form stages 288 / 64 / 32 slots per warp for W = 1 / <= 12 / 13..26, and none from W = 27: tlag_dev.cuh,
TLAG_SL_STAGE_SLOTS), slots that straddle word boundaries, clustering keys that vary, are constant or equal the rank
set's empty marker, interpreter frame classes, and levels that outgrow their store and are rolled back and redone.

The model: K slots x[1..K], each stepped by D from 0 up to B*D, one slot per action (`\\E i \\in 1..K`).  The reachable
set is the box {0, D, ..., B*D}^K: level L holds the coefficient of t^L in (1 + t + ... + t^B)^K states, and every
state has one successor per slot below its top.  Optional parts:
- a mirror y[i], written by the same action (y' = [y EXCEPT ![i] = x[i] + D]); starting at -1 it packs as 0xFFFFFFFF
  until its slot is first stepped.  With ballast between x and y and most of the state unchanged, the action is compiled
  to an EMITD: the parent's packed words copied, two dirty slot ranges far apart re-packed over them;
- ballast: KB constant 32-bit words, before the mirror or after it (then the clustering key is constant);
- a stuttering step at the top corner (a self-loop, which the scalar form drops before the probe).

The reference (per-level sizes, generated, distinct, depth, and the XOR / SUM digest of the 64-bit fingerprints) is
computed here in numpy from the closed form: the box is enumerated, each state packed from cm.layout and hashed with a
port of fingerprint.fingerprint_words.  Neither the bytecode, the emitted C nor the device takes part in it."""
import os
from collections import namedtuple

import numpy as np
import pytest

import test_sliced
from tla_rust_b200.checker import _frame_of, compile_model, encode_states, pack_words
from tla_rust_b200.compile.sliced import Emitter, SliceError
from tla_rust_b200.fingerprint import fingerprint_words
from tla_rust_b200.front.spec import Model
from tla_rust_b200.front.values import Fcn
from oracle import cpu_engine

# typed: x (and a mirror that does not start at -1) declared in TypeOK as [1..K -> 0..B*D], so a slot has the bits of
# B*D; untyped variables are inferred from a sample of states and get 32-bit slots.  mirror: None, "pos" (starts at 0)
# or "neg" (starts at -1, 32 bits).  order: pack order of x, ballast c and mirror y (the last two words are the key).
# down: a second action steps a slot back by D (no mirror): the box and its levels are the same, every successor it
# generates lies in the previous level, so the seen-set must still hold that level after a rollback
Shape = namedtuple("Shape", "name K B D typed mirror KB order stutter down", defaults=(False,))

SHAPES = [
    # W = 1, 2-bit slots: 288 staging slots; a warp of states with ten enabled slots stages 320 successors
    Shape("w1", 10, 2, 1, True, None, 0, "xcy", False),
    # 10-bit slots straddling words at bits 30, 60, ...; W = 12 (64 slots) with a constant key: one key per level
    Shape("w12", 16, 1, 999, True, "pos", 2, "xyc", True),
    # W = 13 (32 slots), key in the mirror's straddling 10-bit slots
    Shape("w13", 16, 1, 999, True, "pos", 3, "xcy", False),
    # 32-bit slots: W = 25 / 26 are the last staged widths, 27 the first unstaged one
    Shape("w25", 12, 1, 7, False, "neg", 1, "xcy", True),
    Shape("w26", 12, 1, 7, False, "neg", 2, "xcy", False),
    Shape("w27", 12, 1, 7, False, "neg", 3, "xcy", True),
    # W = 34, levels of up to 12 870 states; the key is (y[16], y[15]): all ones while both are unstepped
    Shape("w34", 16, 1, 5, False, "neg", 2, "xcy", False),
    # interpreter frame classes: 64 words or fewer, and just over
    Shape("f64", 5, 2, 3, False, None, 22, "xcy", False),
    Shape("f66", 5, 2, 3, False, None, 23, "xcy", False),
    # EMITD (lower.py emits it where an action changes at most half of 64 or more slots): x and y are 4 slots each, 60
    # ballast words apart; W = 72
    Shape("emitd", 6, 3, 3, False, "pos", 60, "xcy", True),
    # W = 1 with steps back to the previous level
    Shape("back", 10, 2, 1, True, None, 0, "xcy", False, True),
]
BY_NAME = {s.name: s for s in SHAPES}
Ref = namedtuple("Ref", "levels generated distinct depth fp_xor fp_sum words level_of frames")


def _spec(s):
    """(module text, cfg text) of shape s"""
    top = s.B * s.D
    names = {"x": "x", "c": "c", "y": "y"}
    vars_ = [names[v] for v in s.order if (v != "y" or s.mirror) and (v != "c" or s.KB)]
    init = [f"x = [i \\in 1..{s.K} |-> 0]"]
    step = f"x[i] < {top} /\\ x' = [x EXCEPT ![i] = x[i] + {s.D}]"
    types = [f"x \\in [1..{s.K} -> 0..{top}]"] if s.typed else []
    if s.mirror:
        init.append(f"y = [i \\in 1..{s.K} |-> {-1 if s.mirror == 'neg' else 0}]")
        step += f" /\\ y' = [y EXCEPT ![i] = x[i] + {s.D}]"
        if s.typed and s.mirror == "pos":
            types.append(f"y \\in [1..{s.K} -> 0..{top}]")
    if s.KB:
        init.append("c = <<" + ", ".join(str(0x5A5A0000 + 7919 * j) for j in range(s.KB)) + ">>")
        step += " /\\ UNCHANGED c"
    lines = [f"---- MODULE Box_{s.name} ----", "EXTENDS Integers", "VARIABLES " + ", ".join(vars_)]
    if types:       # a type hint only: not checked as an invariant
        lines.append("TypeOK == " + " /\\ ".join(types))
    lines.append("Init == " + " /\\ ".join(init))
    nxt = f"\\E i \\in 1..{s.K} : {step}"
    if s.down:
        assert not s.mirror
        back = f"x[i] > 0 /\\ x' = [x EXCEPT ![i] = x[i] - {s.D}]" + (" /\\ UNCHANGED c" if s.KB else "")
        nxt = f"\\/ {nxt}\n        \\/ \\E i \\in 1..{s.K} : {back}"
    if s.stutter:
        nxt = f"\\/ {nxt}\n        \\/ (\\A i \\in 1..{s.K} : x[i] = {top}) /\\ UNCHANGED <<{', '.join(vars_)}>>"
    lines += [f"Next == {nxt}", "===="]
    cfg = f"INIT Init\nNEXT Next\nCHECK_DEADLOCK {'TRUE' if s.stutter else 'FALSE'}\n"
    return "\n".join(lines) + "\n", cfg


def _model(s, where):
    os.makedirs(where, exist_ok=True)
    path = os.path.join(where, f"Box_{s.name}.tla")
    text, cfg = _spec(s)
    with open(path, "w") as f:
        f.write(text)
    m = Model(path, cfg_text=cfg)
    init = m.initial_states()
    return m, init, compile_model(m, init)


# ---- reference --------------------------------------------------------------------------------------------------
M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def _rotl(x, r):
    return (x << np.uint64(r)) | (x >> np.uint64(64 - r))


def _fmix(k):
    k ^= k >> np.uint64(33)
    k *= np.uint64(0xff51afd7ed558ccd)
    k ^= k >> np.uint64(33)
    k *= np.uint64(0xc4ceb9fe1a85ec53)
    k ^= k >> np.uint64(33)
    return k


def np_fingerprint(words):
    """fingerprint.fingerprint_words over the rows of an (n, W) uint32 array"""
    w = np.asarray(words, dtype=np.uint64)
    n, W = w.shape
    with np.errstate(over="ignore"):
        h = np.full(n, (0x9E3779B97F4A7C15 ^ ((W * 0xD6E8FEB86659FD93) & 0xFFFFFFFFFFFFFFFF)), dtype=np.uint64)
        c1, c2 = np.uint64(0x87c37b91114253d5), np.uint64(0x4cf5ad432745937f)
        i = 0
        while i + 1 < W:
            k = w[:, i] | (w[:, i + 1] << np.uint64(32))
            k = _rotl(k * c1, 31) * c2
            h ^= k
            h = _rotl(h, 27) * np.uint64(5) + np.uint64(0x52dce729)
            i += 2
        if i < W:
            h ^= _rotl(w[:, i] * c1, 31) * c2
        h = _fmix(h ^ np.uint64(W))
    h[h == 0] = 1
    return h


def np_pack(layout, frames, W):
    """tlag_pack over the rows of an (n, frame) int64 array of unpacked states, from the (off, width, bias) layout"""
    n = frames.shape[0]
    out = np.zeros((n, W), dtype=np.uint64)
    bitpos = 0
    for off, width, bias in np.asarray(layout).tolist():
        v = (frames[:, off].astype(np.int64) - bias).astype(np.uint64) & np.uint64(0xFFFFFFFF)
        assert width == 32 or not np.any(v >> np.uint64(width)), ("value outside its slot", off, width)
        wi, sh = bitpos >> 5, bitpos & 31
        out[:, wi] |= (v << np.uint64(sh)) & np.uint64(0xFFFFFFFF)
        if sh + width > 32:
            out[:, wi + 1] |= v >> np.uint64(32 - sh)
        bitpos += width
    return out.astype(np.uint32)


def _offsets(cm, st0, var, K):
    """frame word of var[i] for i = 1..K: the one word that moves when only var[i] changes in the initial state"""
    base = np.array(_frame_of(cm, st0), dtype=np.int64)
    offs = []
    for i in range(1, K + 1):
        st = dict(st0)
        v = st0[var]
        if isinstance(v, tuple):        # a function on 1..K is a sequence
            st[var] = v[:i - 1] + (v[i - 1] + 1,) + v[i:]
        else:
            f = dict(v.items())
            f[i] = f[i] + 1
            st[var] = Fcn(f)
        d = np.nonzero(np.array(_frame_of(cm, st), dtype=np.int64) - base)[0]
        assert len(d) == 1 and _frame_of(cm, st)[d[0]] - base[d[0]] == 1, (var, i, d)
        offs.append(int(d[0]))
    return offs


def reference(s, cm, st0):
    """closed-form counts and the digest of the box, packed and hashed in numpy"""
    K, B, D = s.K, s.B, s.D
    poly = [1]
    for _ in range(K):
        nxt = [0] * (len(poly) + B)
        for a, c in enumerate(poly):
            for b in range(B + 1):
                nxt[a + b] += c
        poly = nxt
    distinct = (B + 1) ** K
    generated = 1 + K * B * (B + 1) ** (K - 1) * (2 if s.down else 1) + (1 if s.stutter else 0)
    digits = np.zeros((distinct, K), dtype=np.int64)
    r = np.arange(distinct, dtype=np.int64)
    for i in range(K):
        digits[:, i] = r % (B + 1)
        r //= (B + 1)
    x = digits * D
    frames = np.tile(np.array(_frame_of(cm, st0), dtype=np.int64), (distinct, 1))
    frames[:, _offsets(cm, st0, "x", K)] = x
    if s.mirror:
        frames[:, _offsets(cm, st0, "y", K)] = np.where(digits == 0, -1 if s.mirror == "neg" else 0, x)
    words = np_pack(cm.layout, frames, cm.W)
    fp = np_fingerprint(words)
    return Ref(poly + [0], generated, distinct, K * B + 1, int(np.bitwise_xor.reduce(fp)), int(fp.sum(dtype=np.uint64)),
               words, digits.sum(axis=1), frames)


_CACHE = {}


def _compiled(s, where):
    """(cm, packed initial states, reference) of shape s, computed once per process"""
    if s.name not in _CACHE:
        m, init, cm = _model(s, where)
        _CACHE[s.name] = (cm, encode_states(cm, init), reference(s, cm, init[0]))
    return _CACHE[s.name]


@pytest.fixture(scope="module")
def shapes_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("shapes"))


def _scalar_ok(cm):
    try:
        Emitter(cm, scalar=True)
        return True
    except SliceError:
        return False


# ---- CPU ----------------------------------------------------------------------------------------------------------
def test_the_shapes_have_the_widths_and_frames_they_are_named_for(shapes_dir):
    from tla_rust_b200.compile.bytecode import OP
    want_w = {"w1": 1, "w12": 12, "w13": 13, "w25": 25, "w26": 26, "w27": 27, "w34": 34, "emitd": 72}
    for s in SHAPES:
        cm, _, ref = _compiled(s, shapes_dir)
        if s.name in want_w:
            assert cm.W == want_w[s.name], (s.name, cm.W)
            assert _scalar_ok(cm), s.name
        assert sum(ref.levels) == ref.distinct
    widths = {w for cm, _, _ in (_compiled(s, shapes_dir) for s in SHAPES) for _, w, _ in cm.layout.tolist()}
    assert {2, 10, 32} <= widths
    # a 10-bit slot straddles a word boundary (bits 30..39)
    assert _compiled(BY_NAME["w12"], shapes_dir)[0].layout[3][1] == 10
    assert _compiled(BY_NAME["f64"], shapes_dir)[0].frame_words <= 64 < _compiled(BY_NAME["f66"], shapes_dir)[0].frame_words
    # the dirty-range emit: in the EMITD shape only
    for s in SHAPES:
        ops = [int(c) & 0xFF for c in _compiled(s, shapes_dir)[0].code]
        assert (OP["EMITD"] in ops) == (s.name == "emitd"), s.name
        assert OP["EMITD"] in ops or OP["EMIT"] in ops
    # clustered levels (>= 8192 states)
    for name in ("w12", "w13", "w34"):
        assert sum(1 for n in _compiled(BY_NAME[name], shapes_dir)[2].levels if n >= 8192) >= 3


def test_numpy_packer_and_hash_match_the_host_and_c_implementations(shapes_dir):
    from tla_rust_b200.checker import unpack_words
    rng = np.random.default_rng(3)
    for name in ("w1", "w13", "w34", "emitd"):
        cm, _, ref = _compiled(BY_NAME[name], shapes_dir)
        pick = rng.choice(len(ref.words), size=min(64, len(ref.words)), replace=False)
        rows = ref.words[pick]
        # the same unpacked frames through the host packer, and back
        for f, w in zip(ref.frames[pick], rows):
            assert pack_words(cm, f.tolist()).tolist() == w.tolist()
            assert unpack_words(cm, w) == f[:cm.state_words_unpacked].tolist()
        assert np_fingerprint(rows).tolist() == [fingerprint_words(w) for w in rows]
        assert [int(v) for v in np_fingerprint(rows)] == [cpu_engine.fingerprint(w) for w in rows]
        fp = np_fingerprint(rows)
        assert cpu_engine.digest(rows, cm.W) == (int(np.bitwise_xor.reduce(fp)), int(fp.sum(dtype=np.uint64)))


def _check(r, ref, what):
    assert r["verdict"] == 0, what
    assert (r["generated"], r["distinct"], r["depth"]) == (ref.generated, ref.distinct, ref.depth), what
    assert r["levels"] == ref.levels, what
    assert (r["fp_xor"], r["fp_sum"]) == (ref.fp_xor, ref.fp_sum), what


@pytest.mark.parametrize("name", [s.name for s in SHAPES])
def test_oracle_and_sliced_c_match_the_closed_form(tmp_path, shapes_dir, name):
    """ORACLE O2 (the C bytecode engine) and the sliced C in both forms inside it"""
    s = BY_NAME[name]
    cm, init, ref = _compiled(s, shapes_dir)
    deadlock = s.stutter
    _check(cpu_engine.run(cm, init, n_threads=2, deadlock=deadlock), ref, (name, "o2"))
    info = {"deadlock": deadlock}
    for scalar in ([False, True] if _scalar_ok(cm) else [False]):
        L = test_sliced._cpu_sliced_lib(tmp_path, cm, scalar)
        _check(test_sliced._run_with(L, cm, init, info), ref, (name, "scalar" if scalar else "array"))


# ---- device ---------------------------------------------------------------------------------------------------------
def _run_device(cm, init, deadlock, native, **kw):
    """the engine to its fixpoint: (engine, per-level sizes, per-level retries, result)"""
    from tla_rust_b200.engine import V_RUNNING, Engine
    e = Engine(cm, deadlock=deadlock, native=native, **kw)
    e.seed(init)
    levels, retries = [int(len(np.unique(init, axis=0)))], []
    while True:
        ws = e.step()
        if ws["expanded"]:
            levels.append(int(ws["discovered"]))
            retries.append(int(ws["retries"]))
        if ws["verdict"] != V_RUNNING:
            break
    return e, levels, retries, e.result()


def _check_device(e, levels, r, ref, what):
    assert r["verdict"] == 0, (what, r)
    assert (r["generated"], r["distinct"], r["depth"]) == (ref.generated, ref.distinct, ref.depth), what
    assert levels == ref.levels, what
    assert e.digest() == (ref.fp_xor, ref.fp_sum), what


# the sliced builds: every shape in the scalar form (staging at 288 / 64 / 32 / 32 / 32 slots, none at W = 27 and 34),
# the array form for the straddling 10-bit slots and the widest shape
SWEEP = [(s.name, "sliced", "scalar") for s in SHAPES if s.name.startswith("w")] + \
        [("w13", "sliced", "array"), ("w34", "sliced", "array"), ("emitd", "sliced", "scalar"),
         ("emitd", "sliced", "array")] + \
        [(s.name, "interp", None) for s in SHAPES]


@pytest.mark.gpu
@pytest.mark.parametrize("name,engine,form", SWEEP)
def test_device_engines_match_the_closed_form(monkeypatch, shapes_dir, name, engine, form):
    s = BY_NAME[name]
    cm, init, ref = _compiled(s, shapes_dir)
    monkeypatch.delenv("TLAG_TIGHT_HEADROOM", raising=False)
    monkeypatch.delenv("TLAG_SL_STAGE", raising=False)
    monkeypatch.delenv("TLAG_SL_SKIPSELF", raising=False)
    if form:
        monkeypatch.setenv("TLAG_SL_FORM", form)
    # staged scalar kernels also with one warp's worth of slots, and with the self-loop filter off
    variants = [{}]
    if form == "scalar" and cm.W <= 26:
        variants += [{"TLAG_SL_STAGE": "32"}, {"TLAG_SL_SKIPSELF": "0"}]
    for env in variants:
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        e, levels, _, r = _run_device(cm, init, s.stutter, "sliced" if engine == "sliced" else False)
        _check_device(e, levels, r, ref, (name, engine, form, env))
        e.close()
        for k in env:
            monkeypatch.delenv(k)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["w12", "w13", "w34"])
def test_clustered_levels_are_ordered_by_key_and_hold_the_closed_form_states(monkeypatch, shapes_dir, name):
    """w12: one key per level (constant ballast); w13: keys from straddling 10-bit slots; w34: some keys are all ones,
    the rank set's empty marker, and sort last"""
    for k in ("TLAG_TIGHT_HEADROOM", "TLAG_RSET_SLOTS", "TLAG_SL_STAGE", "TLAG_SL_SKIPSELF"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("TLAG_SL_FORM", "scalar")
    s = BY_NAME[name]
    cm, init, ref = _compiled(s, shapes_dir)
    e, levels, _, r = _run_device(cm, init, s.stutter, "sliced")
    _check_device(e, levels, r, ref, name)
    W = cm.W
    got = e.read_states(0, r["distinct"])
    rng = np.random.default_rng(11)
    start, prev, clustered, max_keys = 0, (0, 0), 0, 0
    for L, size in enumerate(levels):
        lvl = got[start:start + size]
        want = ref.words[ref.level_of == L]
        assert np.array_equal(lvl[np.lexsort(lvl.T[::-1])], want[np.lexsort(want.T[::-1])]), (name, L)
        if size >= 8192:
            clustered += 1
            key = (lvl[:, W - 1].astype(np.uint64) << np.uint64(32)) | lvl[:, W - 2].astype(np.uint64)
            assert np.all(key[1:] >= key[:-1]), (name, L)
            ones = key == np.uint64(0xFFFFFFFFFFFFFFFF)
            if ones.any():            # the all-ones key is ranked last
                max_keys += 1
                assert np.all(ones[np.argmax(ones):]), (name, L)
        if start > 0:
            for i in rng.choice(size, size=min(size, 100), replace=False):
                row, parent, _, _ = e.read_link(start + int(i))
                assert np.array_equal(np.asarray(row, dtype=np.uint32), lvl[i])
                assert prev[0] <= parent < prev[1], (name, start + int(i), parent, prev)
        prev = (start, start + size)
        start += size
    assert clustered >= 3
    if name == "w12":
        assert len({tuple(r_) for r_ in got[:, W - 2:].tolist()}) == 1
    if name == "w34":
        assert max_keys >= 3
    e.close()


# ---- rollback: levels that outgrow the store or the seen-set --------------------------------------------------------
def _store_overflows(levels):
    """levels (by index) whose wave overflows the store under TLAG_TIGHT_HEADROOM: the store starts at 1024 rows, the
    seed makes room for 1024 more rows than it has states, and each level is given room for as many new states as it
    expands, a rerun for exactly what it discovered"""
    cap = max(1024, levels[0] + 1024)
    hi, out = levels[0], []
    for i in range(len(levels) - 1):
        cap = max(cap, hi + levels[i])
        if hi + levels[i + 1] > cap:
            out.append(i)
            cap = hi + levels[i + 1]
        hi += levels[i + 1]
    return out


TIGHT = [("w1", "sliced", "scalar", 0), ("w13", "sliced", "scalar", 0), ("w27", "sliced", "scalar", 0),
         ("emitd", "sliced", "array", 0), ("emitd", "interp", None, 0), ("back", "sliced", "scalar", 0),
         ("back", "interp", None, 0),
         ("w34", "sliced", "array", 0), ("w13", "interp", None, 0), ("w34", "interp", None, 0),
         ("w1", "sliced", "scalar", 4), ("w1", "interp", None, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,engine,form,table_log2", TIGHT)
def test_levels_rolled_back_and_redone_match_the_closed_form(monkeypatch, shapes_dir, name, engine, form, table_log2):
    """TLAG_TIGHT_HEADROOM: every growing level past the first 1024 states overflows its store (and, from a 16-slot
    table, early levels fill the seen-set) and is redone; the scalar staged kernels then append flush runs that straddle
    the store's capacity, and the rerun fills the store to its last row"""
    for k in ("TLAG_SL_STAGE", "TLAG_SL_SKIPSELF"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("TLAG_TIGHT_HEADROOM", "1")
    if form:
        monkeypatch.setenv("TLAG_SL_FORM", form)
    s = BY_NAME[name]
    cm, init, ref = _compiled(s, shapes_dir)
    e, levels, retries, r = _run_device(cm, init, s.stutter, "sliced" if engine == "sliced" else False,
                                        table_log2=table_log2)
    _check_device(e, levels, r, ref, (name, engine, form, table_log2))
    over = _store_overflows(ref.levels)
    assert len(over) >= 2 and all(retries[i] > 0 for i in over), (retries, over)
    if not table_log2:
        assert [i for i, n in enumerate(retries) if n] == over, (retries, over)
    e.close()


@pytest.mark.gpu
def test_a_full_seen_set_alone_rolls_the_level_back(monkeypatch, shapes_dir):
    """1024 states fit the store the hook starts with: every rerun is one a full 16-slot table caused"""
    monkeypatch.setenv("TLAG_TIGHT_HEADROOM", "1")
    s = Shape("full_table", 10, 1, 1, True, None, 0, "xcy", False)
    m, init, cm = _model(s, os.path.join(shapes_dir, "full_table"))
    ref = reference(s, cm, init[0])
    for native in ("sliced", False):
        e, levels, retries, r = _run_device(cm, encode_states(cm, init), False, native, table_log2=4)
        _check_device(e, levels, r, ref, native)
        assert max(retries) > 0, retries
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,table_log2", [("MCPaxos3_b2", 0), ("MCraft", 1)])
@pytest.mark.parametrize("native", ["sliced", False])
def test_fixtures_rolled_back_and_redone_match_the_oracle(monkeypatch, name, table_log2, native):
    """MCPaxos3_b2 (185 369 states) outgrows the store; MCraft (694 states) fits the store and fills a 2-slot table"""
    from conftest import GOLDEN
    from tla_rust_b200.compiled import load_compiled
    monkeypatch.setenv("TLAG_TIGHT_HEADROOM", "1")
    cm, init, exp, info = load_compiled(os.path.join(GOLDEN, name + ".tlagz"))
    o2 = exp["o2"]
    e, levels, retries, r = _run_device(cm, init, info["deadlock"], native, table_log2=table_log2)
    assert r["verdict"] == o2["verdict"]
    assert (r["generated"], r["distinct"], r["depth"]) == (o2["generated"], o2["distinct"], o2["depth"])
    assert levels == o2["levels"]
    assert e.digest() == (o2["fp_xor"], o2["fp_sum"])
    if table_log2:
        assert any(retries), retries
    else:
        assert all(retries[i] > 0 for i in _store_overflows(o2["levels"])) and len(_store_overflows(o2["levels"])) >= 3
    e.close()


@pytest.mark.gpu
def test_keep_going_under_rollbacks_reports_the_same_first_violation(monkeypatch):
    from conftest import GOLDEN
    from tla_rust_b200.compiled import load_compiled
    cm, init, exp, info = load_compiled(os.path.join(GOLDEN, "demo_race.tlagz"))
    got = []
    for tight in ("0", "1"):
        monkeypatch.setenv("TLAG_TIGHT_HEADROOM", tight)
        for native in ("sliced", False):
            e, levels, retries, r = _run_device(cm, init, info["deadlock"], native, keep_going=True, table_log2=1)
            got.append(((r["verdict"], r["detail"], r["state_idx"], r["generated"], r["distinct"], r["depth"]),
                        e.digest(), levels))
            if tight == "1":
                assert max(retries) > 0, retries
            e.close()
    assert got[0][0][0] == 1 and all(g == got[0] for g in got), got
    o2 = exp["o2"]
    assert got[0][0][4] >= o2["distinct"]          # the whole space: at least what the stopping search had found


def _exact(cm, init, deadlock):
    """TLAG_F_EXACT to the first error: (verdict, generated, distinct, queue, depth), per-level retries"""
    from tla_rust_b200.engine import V_RUNNING, Engine
    e = Engine(cm, deadlock=deadlock, exact=True)
    e.seed(init)
    retries = []
    while True:
        ws = e.step()
        retries.append(int(ws["retries"]))
        if ws["verdict"] != V_RUNNING:
            break
    r = e.result()
    e.close()
    return (r["verdict"], r["generated"], r["distinct"], r["queue_left"], r["depth"]), retries


@pytest.mark.gpu
def test_exact_replay_under_rollbacks_reproduces_the_readme_transcript(monkeypatch):
    from conftest import GOLDEN
    from tla_rust_b200.compiled import load_compiled
    monkeypatch.setenv("TLAG_TIGHT_HEADROOM", "1")
    cm, init, _, info = load_compiled(os.path.join(GOLDEN, "pcal_intro_readme_buggy.tlagz"))
    got, retries = _exact(cm, init, info["deadlock"])
    assert got == (2, 9097, 6164, 999, 7)
    assert any(retries), retries


@pytest.mark.gpu
def test_exact_replay_stopped_in_a_rolled_back_level_keeps_its_error(monkeypatch, shapes_dir):
    """The Assert fails on one of the last states of a level whose successors outgrow the store: the wave that finds it
    is rolled back and redone, and the redone wave must find it again (the stop flag of the first attempt is cleared)."""
    path = os.path.join(shapes_dir, "assert")
    os.makedirs(path, exist_ok=True)
    K = 12              # levels 1, 12, 66, 220, 495, 792, ...: the wave expanding the 495 states outgrows the store
    with open(os.path.join(path, "BoxAssert.tla"), "w") as f:
        f.write("---- MODULE BoxAssert ----\nEXTENDS Integers, TLC\nVARIABLES x\n"
                f"TypeOK == x \\in [1..{K} -> 0..1]\nInit == x = [i \\in 1..{K} |-> 0]\n"
                f"Next == \\E i \\in 1..{K} : x[i] < 1 /\\ Assert(~(x[{K - 3}] = 1 /\\ x[{K - 2}] = 1 /\\ x[{K - 1}] = 1 /\\ x[{K}] = 1), "
                "\"three\") /\\ x' = [x EXCEPT ![i] = 1]\n====\n")
    m = Model(os.path.join(path, "BoxAssert.tla"), cfg_text="INIT Init\nNEXT Next\nCHECK_DEADLOCK FALSE\n")
    init = m.initial_states()
    cm = compile_model(m, init)
    iw = encode_states(cm, init)
    o2 = cpu_engine.run(cm, iw, deadlock=False, exact=True)
    want = (o2["verdict"], o2["generated"], o2["distinct"], o2["queue"], o2["depth"])
    assert want[0] == 2
    assert want[4] == 6 and want[2] > 794 + 495           # stopped in the wave expanding level 5, past its head-room
    monkeypatch.setenv("TLAG_TIGHT_HEADROOM", "0")
    assert _exact(cm, iw, False)[0] == want
    monkeypatch.setenv("TLAG_TIGHT_HEADROOM", "1")
    got, retries = _exact(cm, iw, False)
    assert got == want and retries[-1] > 0, (got, retries)


@pytest.mark.gpu
@pytest.mark.parametrize("native", ["sliced", False])
def test_a_store_cap_below_the_space_fails_the_level_and_drops_nothing_before_it(monkeypatch, shapes_dir, native):
    from tla_rust_b200.engine import V_RUNNING, EngineError, Engine
    monkeypatch.delenv("TLAG_TIGHT_HEADROOM", raising=False)
    monkeypatch.setenv("TLAG_SL_FORM", "scalar")
    s = BY_NAME["w13"]
    cm, init, ref = _compiled(s, shapes_dir)
    e, levels, _, r = _run_device(cm, init, s.stutter, native, max_states=ref.distinct)
    _check_device(e, levels, r, ref, "max_states = the space")
    e.close()
    cap = ref.distinct - 1
    e = Engine(cm, deadlock=s.stutter, native=native, max_states=cap)
    e.seed(init)
    done = [1]
    with pytest.raises(EngineError, match="state store overflow"):
        while True:
            ws = e.step()
            assert ws["verdict"] == V_RUNNING
            done.append(int(ws["discovered"]))
    assert done == ref.levels[:len(done)] and sum(done) <= cap < sum(ref.levels[:len(done) + 1])
    have = e.read_states(0, sum(done))
    want = ref.words[ref.level_of < len(done)]
    assert np.array_equal(have[np.lexsort(have.T[::-1])], want[np.lexsort(want.T[::-1])])
    e.close()
