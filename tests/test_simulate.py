"""Random simulation (`tlc -simulate`, include/tlag.h: tlag_simulate).

CPU side: the CPU walker (tests/sim_walker.c), in its interpreter and sliced-code builds, against ORACLE O1's
transitions, against each other, against a chi-square test of its choices and against a numpy restatement of the draw;
`tlc -simulate` on a CPU shim; the simulation libraries cross-compile.  GPU side (-m gpu): both device engines against the
CPU walker word for word, and `tlc -simulate` end to end."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, REF, ROOT, needs_reference
from oracle.cpu_engine import CpuModel
from tla_rust_b200.compiled import load_compiled
from tla_rust_b200.compile.sliced import Emitter, SliceError, emit_sliced, model_key

WALKER = os.path.join(ROOT, "tests", "sim_walker.c")
MASK = (1 << 64) - 1


# ---- R, restated (csrc/tlag_vm.h: tlag_sim_draw) --------------------------------------------------------------------
def _mix(z):
    z = ((z ^ (z >> 30)) * 0xbf58476d1ce4e5b9) & MASK
    z = ((z ^ (z >> 27)) * 0x94d049bb133111eb) & MASK
    return z ^ (z >> 31)


def draw(seed, w, t, j):
    return _mix(_mix(_mix((seed + 0x9E3779B97F4A7C15) & MASK) ^ w) ^ ((t << 32) | j))


def draw_np(seed, w, t, j):
    """vectorised over w and j (uint64 arithmetic wraps mod 2^64)"""
    def mix(z):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xbf58476d1ce4e5b9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94d049bb133111eb)
        return z ^ (z >> np.uint64(31))
    with np.errstate(over="ignore"):
        s = mix(np.uint64((seed + 0x9E3779B97F4A7C15) & MASK))
        return mix(mix(s ^ np.asarray(w, dtype=np.uint64)) ^ ((np.uint64(t) << np.uint64(32)) | np.asarray(j, dtype=np.uint64)))


# ---- the CPU walker -------------------------------------------------------------------------------------------------
class SimResult(C.Structure):
    _fields_ = [("verdict", C.c_int32), ("detail", C.c_int32), ("detail2", C.c_int32), ("pad", C.c_int32),
                ("walk", C.c_uint64), ("step", C.c_uint64), ("checked", C.c_uint64), ("generated", C.c_uint64),
                ("behaviours", C.c_uint64), ("batch_walks", C.c_uint64)]


_LIBS = {}


def walker_lib(tmp_dir, cm=None, scalar=None):
    """the interpreter build (cm None), or the sliced-code build of cm in the given frame form"""
    key = None if cm is None else (model_key(cm), scalar)
    if key in _LIBS:
        return _LIBS[key]
    flags = []
    name = "walker"
    if cm is not None:
        name = f"walker_{model_key(cm)}{'_s' if scalar else '_a'}"
        inc = os.path.join(tmp_dir, name + ".inc")
        with open(inc, "w") as f:
            f.write(emit_sliced(cm, scalar=scalar))
        flags = [f'-DTLAG_SLICED_INC="{inc}"', "-Wno-unused-label", "-Wno-unused-function"]
    so = os.path.join(tmp_dir, name + ".so")
    subprocess.check_call(["gcc", "-O1", "-std=gnu11", "-fPIC", "-shared", *flags, "-o", so, WALKER])
    L = C.CDLL(so)
    for fn in ("tlagcpu_sim_draw", "tlagcpu_sim_batch", "tlagcpu_sim_term", "tlagcpu_fingerprint"):
        getattr(L, fn).restype = C.c_uint64
    L.tlagcpu_sim_draw.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32]
    L.tlagcpu_sim_batch.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64]
    L.tlagcpu_sim_term.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32, C.c_int32]
    _LIBS[key] = L
    return L


def walk(L, cm, init, seed, num, depth, deadlock=True, first=0):
    """-> (result dict, history [depth, n, W], actions [depth, n], lengths [n]) of the last batch"""
    code = np.ascontiguousarray(cm.code, dtype=np.uint64)
    cpool = np.ascontiguousarray(cm.cpool, dtype=np.int32)
    layout = np.ascontiguousarray(cm.layout, dtype=np.int32)
    init = np.ascontiguousarray(init, dtype=np.uint32).reshape(-1, cm.W)
    m = CpuModel(cm.W, code.ctypes.data, len(code), cm.entries["inv"], cm.entries["next"], cpool.ctypes.data, len(cpool),
                 layout.ctypes.data, layout.shape[0], cm.frame_words, cm.state_words_unpacked, len(cm.invariants),
                 1 if deadlock else 0, 0, 0)
    B = int(L.tlagcpu_sim_batch(cm.W, depth, num))
    n = min(B, num)
    hist = np.zeros((depth, n, cm.W), dtype=np.uint32)
    acts = np.zeros((depth, n), dtype=np.int16)
    lens = np.zeros(n, dtype=np.uint32)
    r = SimResult()
    rc = L.tlagcpu_simulate(C.byref(m), init.ctypes.data_as(C.c_void_p), C.c_uint64(init.shape[0]), C.c_uint64(seed),
                            C.c_uint64(first), C.c_uint64(num), C.c_uint32(depth), C.byref(r),
                            hist.ctypes.data_as(C.c_void_p), acts.ctypes.data_as(C.c_void_p), lens.ctypes.data_as(C.c_void_p))
    assert rc == 0
    res = {f: getattr(r, f) for f, _ in SimResult._fields_ if f != "pad"}
    if r.behaviours % B:        # the last batch was short: its walks are the first behaviours % B columns
        n = r.behaviours % B
        hist, acts, lens = hist[:, :n], acts[:, :n], lens[:n]
    return res, hist, acts, lens


def same_history(a, b):
    """two (result, hist, acts, lens) agree on every state checked"""
    ra, ha, aa, la = a
    rb, hb, ab, lb = b
    assert np.array_equal(la, lb), np.nonzero(la != lb)[0][:8]
    for i in range(len(la)):
        n = int(la[i])
        assert np.array_equal(ha[:n, i], hb[:n, i]), (i, np.nonzero((ha[:n, i] != hb[:n, i]).any(axis=1))[0][:4])
        assert np.array_equal(aa[1:n, i], ab[1:n, i]), i


KEYS = ("verdict", "detail", "walk", "step")
COUNTS = ("checked", "generated", "behaviours")


@pytest.fixture(scope="module")
def libdir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("simwalker"))


def _forms(cm):
    forms = [False]
    try:
        Emitter(cm, scalar=True)
        forms.append(True)
    except SliceError:
        pass
    return forms


def _fixture(name):
    return load_compiled(os.path.join(GOLDEN, name + ".tlagz"))


# ---- 1. every step is a transition of ORACLE O1 ---------------------------------------------------------------------
def _spec_cases():
    cases = [os.path.join(ROOT, "models", "demo", f) for f in ("lock.tla", "race.tla")]
    cases += sorted(os.path.join(ROOT, "tests", "specs", f) for f in os.listdir(os.path.join(ROOT, "tests", "specs"))
                    if f.endswith(".tla") and os.path.exists(os.path.join(ROOT, "tests", "specs", f[:-4] + ".cfg")))
    return cases


def _walks_are_transitions(libdir, path, cfg=None):
    from oracle.tlc_oracle import Oracle
    from tla_rust_b200.checker import compile_model, decode_state, encode_states
    from tla_rust_b200.front.spec import Model
    from tla_rust_b200.front.spec import SpecError
    from tla_rust_b200.front.values import EvalError
    try:
        m = Model(path, cfg_path=cfg)
        m.ev.out = io.StringIO()
        init = [st for st in m.initial_states() if m.in_model(st)]
    except (SpecError, EvalError) as ex:           # specs the checker refuses (tests of its error reports)
        pytest.skip(f"not a checkable spec: {ex}")
    cm = compile_model(m, init)
    o = Oracle(m)
    key = lambda st: o.key(o.canon(st))
    inits = {key(st) for st in init}
    res, hist, acts, lens = walk(walker_lib(libdir), cm, encode_states(cm, init), seed=11, num=64, depth=12,
                                 deadlock=m.check_deadlock)
    seen = 0
    for i in range(len(lens)):
        prev = None
        for t in range(int(lens[i])):
            st = decode_state(cm, hist[t, i])
            if prev is None:
                assert key(st) in inits, (path, i)
            else:
                succ = {key(s) for s, _ in o.successors(prev) if m.in_model(s) and o.in_actions(prev, s)}
                assert key(st) in succ, (path, i, t)
                seen += 1
            prev = st
    assert seen or res["verdict"] != 0 or max(lens) == 1


@pytest.mark.parametrize("path", _spec_cases(), ids=lambda p: os.path.basename(p))
def test_every_step_of_a_walk_is_a_transition_of_the_ast_oracle(libdir, tmp_path, path):
    if "demo" in path:              # PlusCal: translated in a copy
        path = _demo(os.path.basename(path)[:-4], tmp_path)
    _walks_are_transitions(libdir, path)


# the README's bug in pcal_intro.tla: the withdrawal and the deposit in two steps (tests/golden/make_golden.py)
README_BUGGY = (("     alice_account := alice_account - money;", "     A: alice_account := alice_account - money;"),
                ("     bob_account := bob_account + money;", "     B: bob_account := bob_account + money;"))


def _pcal_intro(tmp_path, edits=()):
    from tla_rust_b200.front.pcal import translate_file
    src = open(os.path.join(REF, "pcal_intro.tla")).read()
    for a, b in edits:
        assert a in src
        src = src.replace(a, b)
    path = os.path.join(tmp_path, "pcal_intro.tla")
    with open(path, "w") as f:
        f.write(src)
    with open(os.path.join(tmp_path, "pcal_intro.cfg"), "w") as f:
        f.write("SPECIFICATION Spec\n")
    translate_file(path)
    return path


@needs_reference
def test_pcal_intro_walks_are_transitions_of_the_ast_oracle(libdir, tmp_path):
    _walks_are_transitions(libdir, _pcal_intro(tmp_path))


# ---- 2. interpreter walker == sliced-code walker ----------------------------------------------------------------------
SLICED_FIXTURES = ["atomic_add", "pcal_intro", "pcal_intro_readme_buggy", "demo_race", "demo_lock", "MCInnerFIFO",
                   "MCAlternatingBit", "MCPaxos", "MCPaxos3", "MCPaxos3_sym", "MCVoting", "MCVoting_deadlock", "Containers",
                   "HourClock", "AsynchInterface", "MCPaxos3_b2"]


@pytest.mark.parametrize("name", SLICED_FIXTURES)
def test_sliced_code_walks_like_the_interpreter(libdir, name):
    cm, init, _exp, info = _fixture(name)
    ref = walk(walker_lib(libdir), cm, init, seed=5, num=256, depth=40, deadlock=info["deadlock"])
    for scalar in _forms(cm):
        got = walk(walker_lib(libdir, cm, scalar), cm, init, seed=5, num=256, depth=40, deadlock=info["deadlock"])
        for k in KEYS:
            assert got[0][k] == ref[0][k], (name, scalar, k, got[0], ref[0])
        if ref[0]["verdict"] != 4:      # (after an evaluation trap the counts may differ, DESIGN.md §5)
            for k in COUNTS:
                assert got[0][k] == ref[0][k], (name, scalar, k)
            same_history(got, ref)


def test_the_fixtures_cover_every_verdict(libdir):
    verdicts = {}
    for name in ("demo_race", "pcal_intro_readme_buggy", "MCVoting_deadlock", "demo_lock"):
        cm, init, _exp, info = _fixture(name)
        verdicts[name] = walk(walker_lib(libdir), cm, init, seed=5, num=256, depth=40, deadlock=info["deadlock"])[0]["verdict"]
    assert verdicts == {"demo_race": 1, "pcal_intro_readme_buggy": 2, "MCVoting_deadlock": 3, "demo_lock": 0}


# ---- 3. uniform choices ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 2, 7, 64])
def test_the_pick_among_k_candidates_is_uniform(libdir, tmp_path, k):
    """A generated model whose every state has exactly k candidates (x' = i for i in 0..k-1, the self-loop included):
    over 10^5 walks, the successor chosen at step 0 and at step 3 passes a chi-square test."""
    from scipy.stats import chisquare
    from tla_rust_b200.checker import compile_model, decode_state, encode_states
    from tla_rust_b200.front.spec import Model
    path = tmp_path / f"Pick{k}.tla"
    path.write_text(f"---- MODULE Pick{k} ----\nEXTENDS Naturals\nVARIABLE x\nInit == x = 0\n"
                    f"Next == \\E i \\in 0..{k - 1} : x' = i\n====\n")
    m = Model(str(path), cfg_text="INIT Init\nNEXT Next\n")
    init = m.initial_states()
    cm = compile_model(m, init)
    res, hist, acts, lens = walk(walker_lib(libdir), cm, encode_states(cm, init), seed=1234, num=100000, depth=5)
    assert res["verdict"] == 0 and res["generated"] == 100000 * 4 * k and res["checked"] == 100000 * 5
    for t in (1, 4):
        xs = np.array([decode_state(cm, hist[t, i])["x"] for i in range(hist.shape[1])])
        got = np.bincount(xs, minlength=k)
        assert len(got) == k
        if k > 1:
            assert chisquare(got).pvalue > 1e-4, (t, got)


def test_the_initial_state_is_uniform_over_the_distinct_initial_states(libdir):
    from scipy.stats import chisquare
    cm, init, _exp, info = _fixture("pcal_intro_readme_buggy")
    distinct = np.unique(init, axis=0)
    assert len(distinct) == 400
    res, hist, _a, _l = walk(walker_lib(libdir), cm, init, seed=99, num=100000, depth=1, deadlock=info["deadlock"])
    order = {bytes(r): i for i, r in enumerate(_first_occurrence(init))}
    got = np.bincount([order[bytes(r)] for r in hist[0]], minlength=400)
    assert chisquare(got).pvalue > 1e-4


def _first_occurrence(init):
    seen, out = set(), []
    for r in np.asarray(init, dtype=np.uint32):
        if bytes(r) not in seen:
            seen.add(bytes(r))
            out.append(r)
    return np.array(out)


# ---- 4. determinism -------------------------------------------------------------------------------------------------
def test_a_seed_fixes_the_walks(libdir):
    cm, init, _exp, info = _fixture("MCPaxos3_b2")
    L = walker_lib(libdir)
    a = walk(L, cm, init, seed=7, num=200, depth=30, deadlock=info["deadlock"])
    b = walk(L, cm, init, seed=7, num=200, depth=30, deadlock=info["deadlock"])
    c = walk(L, cm, init, seed=8, num=200, depth=30, deadlock=info["deadlock"])
    assert a[0] == b[0]
    same_history(a, b)
    assert not np.array_equal(a[1], c[1])


def test_a_walk_does_not_depend_on_its_batch(libdir):
    cm, init, _exp, info = _fixture("MCPaxos3_b2")
    L = walker_lib(libdir)
    small = walk(L, cm, init, seed=3, num=32, depth=25, deadlock=info["deadlock"])
    big = walk(L, cm, init, seed=3, num=1024, depth=25, deadlock=info["deadlock"])
    assert small[0]["batch_walks"] == 32 and big[0]["batch_walks"] == 1024
    assert small[0]["verdict"] == big[0]["verdict"] == 0
    for i in range(32):
        n = int(small[3][i])
        assert n == big[3][i] and np.array_equal(small[1][:n, i], big[1][:n, i]), i
    # a walk started at its global id on its own is the same walk too
    one = walk(L, cm, init, seed=3, num=1, depth=25, deadlock=info["deadlock"], first=17)
    n = int(one[3][0])
    assert n == big[3][17] and np.array_equal(one[1][:n, 0], big[1][:n, 17])


def test_the_draw_matches_its_numpy_restatement(libdir):
    L = walker_lib(libdir)
    for seed, w, t, j in [(0, 0, 0, 0), (1, 2, 3, 4), (MASK, MASK, 0xFFFFFFFF, 0xFFFFFFFF), (123456789, 1 << 40, 7, 0xFFFFFFFF)]:
        assert L.tlagcpu_sim_draw(seed, w, t, j) == draw(seed, w, t, j)
    ws = np.arange(1000, dtype=np.uint64)
    assert [int(x) for x in draw_np(42, ws, 5, 3)] == [draw(42, int(w), 5, 3) for w in ws]
    # walk 0's initial state is the restated draw over the distinct initial states
    cm, init, _exp, info = _fixture("pcal_intro_readme_buggy")
    _r, hist, _a, _l = walk(L, cm, init, seed=2024, num=32, depth=1, deadlock=info["deadlock"])
    distinct = _first_occurrence(init)
    k = draw(2024, 0, 0, 0xFFFFFFFF) % len(distinct)
    assert np.array_equal(hist[0, 0], distinct[k])


def test_the_batch_size_depends_on_width_depth_and_count_only(libdir):
    L = walker_lib(libdir)
    assert L.tlagcpu_sim_batch(32, 100, 1 << 20) == (4 << 30) // (100 * 130) // 32 * 32 == 330368
    assert L.tlagcpu_sim_batch(4, 100, 1 << 30) == 1 << 20
    assert L.tlagcpu_sim_batch(1, 1, 1 << 30) == 1 << 20
    assert L.tlagcpu_sim_batch(4, 100, 1000) == 992 and L.tlagcpu_sim_batch(4, 100, 5) == 32


# ---- 5. tlc -simulate on a CPU shim -------------------------------------------------------------------------------
class _CpuSimShim:
    """Stand-in for tla_rust_b200.engine.Engine(simulate=True) backed by the CPU walker (test infrastructure)."""
    lib_dir = None

    def __init__(self, cm, deadlock=True, device=0, native=False, simulate=False, exact=False):
        assert simulate
        self.cm, self.deadlock = cm, deadlock

    def seed(self, iw):
        self.iw = iw

    def simulate(self, seed, num, depth, first=0):
        self.r, self.hist, self.acts, self.lens = walk(walker_lib(self.lib_dir), self.cm, self.iw, seed, num, depth,
                                                       self.deadlock, first)
        self.first = self.r["behaviours"] - len(self.lens) + first
        return dict(self.r, device_ms=0.0)

    def sim_trace(self, w):
        i = w - self.first
        n = int(self.lens[i])
        return self.hist[:n, i].copy(), self.acts[:n, i].astype(np.int32)

    def launches(self):
        return 0

    def close(self):
        pass


@pytest.fixture
def shim(monkeypatch, libdir):
    import tla_rust_b200.engine as eng
    _CpuSimShim.lib_dir = libdir
    monkeypatch.setattr(eng, "Engine", _CpuSimShim)
    monkeypatch.setenv("TLAG_NO_STATES_DIR", "1")


def _tlc(argv, capsys):
    from tla_rust_b200.cli import tlc_main
    rc = tlc_main(argv)
    cap = capsys.readouterr()
    return rc, cap.out, cap.err


def _demo(name, tmp_path):
    import shutil
    for ext in (".tla", ".cfg"):
        shutil.copy(os.path.join(ROOT, "models", "demo", name + ext), tmp_path)
    from tla_rust_b200.front.pcal import translate_file
    translate_file(os.path.join(tmp_path, name + ".tla"), write_cfg=False)
    return os.path.join(tmp_path, name + ".tla")


def test_tlc_simulate_reports_an_invariant_violation_with_a_trace(shim, tmp_path, capsys):
    rc, out, _ = _tlc(["-simulate", "num=500", "-seed", "17", "-engine", "interp", _demo("race", tmp_path)], capsys)
    assert rc == 12
    assert "Running random simulation with seed 17." in out
    assert "Error: Invariant Correct is violated." in out and "State 1: <Initial predicate>" in out
    assert "behaviours simulated" in out and "(seed 17)" in out


def test_tlc_simulate_summary_on_a_correct_spec(shim, tmp_path, capsys):
    rc, out, _ = _tlc(["-simulate", "num=300", "-depth", "20", "-seed", "4", _demo("lock", tmp_path)], capsys)
    assert rc == 0
    assert "Simulation completed. No error has been found." in out
    assert "300 behaviours simulated" in out and "(seed 4)" in out


def test_tlc_simulate_is_reproducible_from_its_seed(shim, tmp_path, capsys):
    spec = _demo("race", tmp_path)
    outs = []
    for _ in range(2):
        rc, out, _ = _tlc(["-simulate", "num=200", "-seed", "99", spec], capsys)
        outs.append([ln for ln in out.splitlines() if not ln.startswith("Finished in")])
    assert outs[0] == outs[1]
    rc, out, _ = _tlc(["-simulate", spec], capsys)         # a seed of its own, printed so that the run can be repeated
    seed = int(out.split("Running random simulation with seed ")[1].split(".")[0])
    assert rc == 12 and f"(seed {seed})" in out


def test_tlc_simulate_refuses_several_gpus(tmp_path, capsys):
    rc, _out, err = _tlc(["-gpus", "2", "-simulate", os.path.join(ROOT, "models", "demo", "lock.tla")], capsys)
    assert rc == 2 and "-simulate" in err


# ---- 6. the simulation libraries cross-compile and keep the C ABI -----------------------------------------------------
@pytest.mark.parametrize("name,scalar", [("MCPaxos3_b2", True), ("MCraft", False)])
def test_simulation_library_cross_compiles_and_keeps_the_c_abi(name, scalar):
    from tla_rust_b200 import engine
    cm, _, _, _ = _fixture(name)
    so = engine.build_sliced_library(cm, scalar=scalar, simulate=True)
    assert so.endswith("_sim.so") and so != engine.sliced_library_path(cm, scalar=scalar)
    L = engine._bind(so)
    assert b"sliced" in L.tlag_version()
    syms = subprocess.run(["nm", "-D", "--defined-only", so], capture_output=True, text=True).stdout
    assert "tlag_sl_sim_launch_next_0" in syms and "tlag_sl_launch_next_0" not in syms


# ---- 7-9. device ----------------------------------------------------------------------------------------------------
DEVICE_FIXTURES = ["demo_race", "pcal_intro_readme_buggy", "MCVoting_deadlock", "MCPaxos3_b2", "MCPaxos3_sym", "MCraft",
                   "MCssi_3x1"]


def _device(cm, init, info, native, seed, num, depth, first=0):
    from tla_rust_b200.engine import Engine
    e = Engine(cm, deadlock=info["deadlock"], native=native, simulate=True)
    e.seed(init)
    r = e.simulate(seed, num, depth, first=first)
    return e, r


@pytest.mark.gpu
@pytest.mark.parametrize("native", [False, "sliced"])
@pytest.mark.parametrize("name", DEVICE_FIXTURES)
def test_device_walks_match_the_cpu_walker(libdir, name, native):
    cm, init, _exp, info = _fixture(name)
    ref = walk(walker_lib(libdir), cm, init, seed=31, num=384, depth=50, deadlock=info["deadlock"])
    e, r = _device(cm, init, info, native, seed=31, num=384, depth=50)
    for k in KEYS:
        assert r[k] == ref[0][k], (name, native, k, r, ref[0])
    if ref[0]["verdict"] != 4:
        for k in COUNTS:
            assert r[k] == ref[0][k], (name, native, k)
        first = r["behaviours"] - len(ref[3])
        same_history((None,) + e.sim_read(first, len(ref[3])), ref)
    if r["verdict"]:
        st, acts = e.sim_trace(r["walk"])
        assert len(st) == r["step"] + 1 and acts[0] == -1
    e.close()


@pytest.mark.gpu
def test_the_two_device_engines_agree_at_scale(libdir):
    cm, init, _exp, info = _fixture("MCPaxos3_b4")
    num = min(1 << 20, (4 << 30) // (100 * (4 * cm.W + 2))) // 32 * 32       # one full batch (include/tlag.h)
    runs = {}
    for native in (False, "sliced"):
        e, r = _device(cm, init, info, native, seed=77, num=num, depth=100)
        B = r["batch_walks"]
        assert B == num and r["behaviours"] == num
        runs[native] = (r, e.sim_digest(), e.sim_read(0, 2), e.sim_read(B - 1, 1))
        e.close()
    (ri, di, a0, al), (rs, ds, b0, bl) = runs[False], runs["sliced"]
    assert ri["behaviours"] == rs["behaviours"] and ri["batch_walks"] == rs["batch_walks"]
    for k in KEYS + COUNTS:
        assert ri[k] == rs[k], k
    assert di == ds
    B = ri["batch_walks"]
    L = walker_lib(libdir)
    ref0 = walk(L, cm, init, seed=77, num=2, depth=100, deadlock=info["deadlock"])
    refl = walk(L, cm, init, seed=77, num=1, depth=100, deadlock=info["deadlock"], first=B - 1)
    for got, ref in ((a0, ref0), (b0, ref0), (al, refl), (bl, refl)):
        same_history((None,) + tuple(got), ref)


def _tlc_gpu(spec, engine):
    import sys
    env = dict(os.environ, TLAG_NO_STATES_DIR="1")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "tlc"), "-simulate", "num=4096", "-seed", "5", "-engine",
                        engine, spec], capture_output=True, text=True, timeout=1200, env=env)
    # (the timing line, and the sliced engine's note that it compiles the model, are not part of the report)
    return p.returncode, [ln for ln in p.stdout.splitlines() if not ln.startswith(("Finished in", "Compiling the model"))]


@pytest.mark.gpu
def test_tlc_simulate_end_to_end_on_the_device(tmp_path):
    spec = _demo("race", tmp_path)
    rc_i, out_i = _tlc_gpu(spec, "interp")
    rc_s, out_s = _tlc_gpu(spec, "sliced")
    assert rc_i == rc_s == 12
    assert "Error: Invariant Correct is violated." in out_i and "State 1: <Initial predicate>" in "\n".join(out_i)
    assert out_i == out_s


@pytest.mark.gpu
@needs_reference
def test_tlc_simulate_finds_the_readme_assert_on_the_device(tmp_path):
    spec = _pcal_intro(tmp_path, README_BUGGY)
    rc_i, out_i = _tlc_gpu(spec, "interp")
    rc_s, out_s = _tlc_gpu(spec, "sliced")
    assert rc_i == rc_s == 12
    assert "The first argument of Assert evaluated to FALSE" in "\n".join(out_i) and "State 1: <Initial predicate>" in out_i
    assert out_i == out_s
