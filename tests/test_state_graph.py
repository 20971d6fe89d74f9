"""The state graph of a search (include/tlag.h: tlag_build_graph) and `tlc -dump` / `tlc -dump dot`.

CPU side: the CPU reference (tests/graph_ref.c) against ORACLE O1's transitions; the edge term against a numpy
restatement; `tlc -dump` on a CPU shim (O2 for the search, graph_ref for the graph); the libraries cross-compile and
export the entry points.  GPU side (-m gpu): both device engines against graph_ref on their own stored states, stopped
searches, chunking and store order, both engines at scale, refusals and release, and `tlc -dump dot` end to end."""
import ctypes as C
import io
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, REF, ROOT
from oracle.cpu_engine import CpuModel
from tla_rust_b200.compiled import load_compiled

GRAPH_REF = os.path.join(ROOT, "tests", "graph_ref.c")
MASK = (1 << 64) - 1


# ---- the CPU reference ----------------------------------------------------------------------------------------------
_LIB = {}


def ref_lib(tmp_dir):
    if "L" not in _LIB:
        so = os.path.join(tmp_dir, "graph_ref.so")
        subprocess.check_call(["gcc", "-O1", "-std=gnu11", "-fPIC", "-shared", "-o", so, GRAPH_REF])
        L = C.CDLL(so)
        L.tlagcpu_graph.restype = C.c_int64
        L.tlagcpu_edge_term.restype = C.c_uint64
        L.tlagcpu_edge_term.argtypes = [C.c_uint64, C.c_uint64, C.c_int32]
        L.tlagcpu_fingerprint.restype = C.c_uint64
        _LIB["L"] = L
    return _LIB["L"]


def ref_graph(L, cm, states, n_expanded):
    """-> (src, dst, act) of the graph over `states` (rows [0, n_expanded) expanded), sorted by (s, t, a)"""
    code = np.ascontiguousarray(cm.code, dtype=np.uint64)
    cpool = np.ascontiguousarray(cm.cpool, dtype=np.int32)
    layout = np.ascontiguousarray(cm.layout, dtype=np.int32)
    st = np.ascontiguousarray(states, dtype=np.uint32).reshape(-1, cm.W)
    m = CpuModel(cm.W, code.ctypes.data, len(code), cm.entries["inv"], cm.entries["next"], cpool.ctypes.data, len(cpool),
                 layout.ctypes.data, layout.shape[0], cm.frame_words, cm.state_words_unpacked, len(cm.invariants), 0, 0, 0)
    cap = max(1024, 4 * st.shape[0])
    while True:
        src, dst, act = (np.zeros(cap, dtype=np.uint32), np.zeros(cap, dtype=np.uint32), np.zeros(cap, dtype=np.int32))
        n = L.tlagcpu_graph(C.byref(m), st.ctypes.data_as(C.c_void_p), C.c_uint64(st.shape[0]), C.c_uint64(n_expanded),
                            src.ctypes.data_as(C.c_void_p), dst.ctypes.data_as(C.c_void_p), act.ctypes.data_as(C.c_void_p),
                            C.c_uint64(cap))
        assert n >= 0, n
        if n <= cap:
            return src[:n], dst[:n], act[:n]
        cap = n


def fingerprints(L, states):
    st = np.ascontiguousarray(states, dtype=np.uint32)
    W = st.shape[1]
    return [int(L.tlagcpu_fingerprint(st[i].ctypes.data_as(C.c_void_p), C.c_int(W))) for i in range(st.shape[0])]


@pytest.fixture(scope="module")
def libdir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("graphref"))


def _fixture(name):
    return load_compiled(os.path.join(GOLDEN, name + ".tlagz"))


# ---- 1. graph_ref against ORACLE O1 ----------------------------------------------------------------------------------
def _demo(name, tmp_path):
    from tla_rust_b200.front.pcal import translate_file
    for ext in (".tla", ".cfg"):
        shutil.copy(os.path.join(ROOT, "models", "demo", name + ext), tmp_path)
    translate_file(os.path.join(tmp_path, name + ".tla"), write_cfg=False)
    return os.path.join(tmp_path, name + ".tla")


def _pcal(name, tmp_path):
    from tla_rust_b200.front.pcal import translate_file
    shutil.copy(os.path.join(REF, name + ".tla"), tmp_path)
    if os.path.exists(os.path.join(REF, name + ".cfg")):
        shutil.copy(os.path.join(REF, name + ".cfg"), tmp_path)
    else:
        (tmp_path / f"{name}.cfg").write_text("SPECIFICATION Spec\n")
    translate_file(os.path.join(tmp_path, name + ".tla"))
    return os.path.join(tmp_path, name + ".tla")


O1_CASES = {
    "demo_lock": lambda tp: _demo("lock", tp),
    "demo_race": lambda tp: _demo("race", tp),
    "atomic_add": lambda tp: _pcal("atomic_add", tp),
    "pcal_intro": lambda tp: _pcal("pcal_intro", tp),
    "HourClock": lambda tp: os.path.join(REF, "examples", "SpecifyingSystems", "HourClock", "HourClock.tla"),
    "MCAlternatingBit": lambda tp: os.path.join(REF, "examples", "SpecifyingSystems", "TLC", "MCAlternatingBit.tla"),
    "MCVoting": lambda tp: os.path.join(REF, "examples", "Paxos", "MCVoting.tla"),
}


def _o1_graph(m):
    """O1's reachable states and transitions: canonical, inside CONSTRAINT and ACTION_CONSTRAINT, no self-loops, each
    (state, state, action) once -> (states, {(index s, index t, (name, location, module))})"""
    from oracle.tlc_oracle import Oracle
    o = Oracle(m)
    key = lambda st: o.key(st)
    states, index, edges = [], {}, set()
    for st in m.initial_states():
        if m.in_model(st):
            st = o.canon(st)
            if key(st) not in index:
                index[key(st)] = len(states)
                states.append(st)
    i = 0
    while i < len(states):
        s = states[i]
        for t, act in o.successors(s):
            if not m.in_model(t) or not o.in_actions(s, t):
                continue
            t = o.canon(t)
            if key(t) not in index:
                index[key(t)] = len(states)
                states.append(t)
            if key(t) != key(s):
                edges.add((i, index[key(t)], tuple(act[1:])))
        i += 1
    return states, edges


@pytest.mark.parametrize("name", list(O1_CASES))
def test_graph_ref_edges_are_the_transitions_of_the_ast_oracle(libdir, tmp_path, name):
    from tla_rust_b200.checker import compile_model, encode_states
    from tla_rust_b200.front.spec import Model
    if name not in ("demo_lock", "demo_race") and not os.path.isdir(REF):
        pytest.skip("no tla-rust spec corpus (oracle/_ref/tla-rust)")
    m = Model(O1_CASES[name](tmp_path))
    m.ev.out = io.StringIO()
    init = [st for st in m.initial_states() if m.in_model(st)]
    cm = compile_model(m, init)
    states, want = _o1_graph(m)
    if name == "pcal_intro":
        assert len(states) == 3800
    words = encode_states(cm, states)
    src, dst, act = ref_graph(ref_lib(libdir), cm, words, len(states))
    # (under SYMMETRY O1's representative of an orbit is not the device's: states are compared as packed words, which
    # encode_states puts in the device's form)
    key = [bytes(w) for w in words]
    assert len(set(key)) == len(states)
    got = {(key[s], key[t], tuple(cm.actions[a])) for s, t, a in zip(src.tolist(), dst.tolist(), act.tolist())}
    assert len(got) == len(src)             # distinct triples
    assert got == {(key[s], key[t], a) for s, t, a in want}, (name, len(got), len(want))
    assert want                             # every case has transitions


# ---- 2. the edge term ------------------------------------------------------------------------------------------------
def _mix(z):
    z = ((z ^ (z >> 30)) * 0xbf58476d1ce4e5b9) & MASK
    z = ((z ^ (z >> 27)) * 0x94d049bb133111eb) & MASK
    return z ^ (z >> 31)


def edge_term(fs, ft, a):
    return _mix(_mix(fs ^ 0x9E3779B97F4A7C15) ^ _mix((ft + (a & 0xFFFFFFFF)) & MASK))


def edge_term_np(fs, ft, a):
    def mix(z):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xbf58476d1ce4e5b9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94d049bb133111eb)
        return z ^ (z >> np.uint64(31))
    with np.errstate(over="ignore"):
        fs, ft = np.asarray(fs, dtype=np.uint64), np.asarray(ft, dtype=np.uint64)
        a = np.asarray(a, dtype=np.int64).astype(np.uint32).astype(np.uint64)
        return mix(mix(fs ^ np.uint64(0x9E3779B97F4A7C15)) ^ mix(ft + a))


def graph_digest_np(fp_s, fp_t, act):
    v = edge_term_np(fp_s, fp_t, act)
    return int(np.bitwise_xor.reduce(v)) if len(v) else 0, int(v.sum(dtype=np.uint64)) if len(v) else 0


def test_the_edge_term_matches_its_numpy_restatement(libdir):
    L = ref_lib(libdir)
    rng = np.random.default_rng(5)
    fs = rng.integers(0, 1 << 63, 500, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    ft = rng.integers(0, 1 << 63, 500, dtype=np.uint64)
    a = rng.integers(-1, 5000, 500)
    got = [int(L.tlagcpu_edge_term(int(x), int(y), int(z))) for x, y, z in zip(fs, ft, a)]
    assert got == [int(v) for v in edge_term_np(fs, ft, a)]
    assert got == [edge_term(int(x), int(y), int(z)) for x, y, z in zip(fs, ft, a)]
    assert edge_term(1, 2, 0) != edge_term(2, 1, 0) and edge_term(1, 2, 0) != edge_term(1, 2, 1)


# ---- 3. tlc -dump on a CPU shim --------------------------------------------------------------------------------------
class _CpuGraphShim:
    """Stand-in for tla_rust_b200.engine.Engine: the search is ORACLE O2's (oracle/cpu_engine.py), handed out one level
    per step; the state graph is graph_ref's over O2's store.  Test infrastructure only."""
    lib_dir = None

    def __init__(self, cm, deadlock=True, device=0, native=False, exact=False, simulate=False):
        self.cm, self.deadlock, self.exact = cm, deadlock, exact

    def seed(self, iw):
        from oracle import cpu_engine
        self.iw = iw
        self.o2 = cpu_engine.run(self.cm, iw, deadlock=self.deadlock, want_states=True, max_states=1 << 17,
                                 exact=self.exact)
        self.levels = self.o2["levels"]
        self.k = 0                       # levels expanded

    def _done(self):
        return self.k >= len(self.levels) or (self.o2["verdict"] != 0 and self.k >= len(self.levels) - 1)

    def result(self):
        r = dict(self.o2, distinct=sum(self.levels[:self.k + 1]), depth=min(self.k + 1, len(self.levels)),
                 queue_left=self.o2.get("queue", 0), device_seconds=0.0)
        if not self._done():
            r["verdict"] = 5
        return r

    def step(self):
        self.k += 1
        disc = self.levels[self.k] if self.k < len(self.levels) else 0
        return {"verdict": self.result()["verdict"], "expanded": self.levels[self.k - 1], "discovered": disc,
                "level": self.k, "generated_total": 0, "distinct_total": sum(self.levels[:self.k + 1])}

    def run(self):
        self.k = len(self.levels)
        return self.result()

    def read_states(self, first, n):
        return self.o2["states"][first:first + n]

    def trace(self, idx):
        return self.o2["states"][idx:idx + 1], np.array([-1])

    def build_graph(self):
        n = sum(self.levels[:self.k + 1])
        n_exp = sum(self.levels[:self.k])
        src, self.dst, self.act = ref_graph(ref_lib(self.lib_dir), self.cm, self.o2["states"][:n], n_exp)
        self.off = np.searchsorted(src, np.arange(n + 1)).astype(np.uint64)
        return {"n_states": n, "n_expanded": n_exp, "n_edges": len(src), "device_ms": 0.0}

    def state_graph(self, first=0, n=None):
        o = self.off[first:first + n + 1]
        return o - o[0], self.dst[int(o[0]):int(o[-1])], self.act[int(o[0]):int(o[-1])]

    def launches(self):
        return 0

    def close(self):
        pass


@pytest.fixture
def shim(monkeypatch, libdir):
    import tla_rust_b200.engine as eng
    _CpuGraphShim.lib_dir = libdir
    monkeypatch.setattr(eng, "Engine", _CpuGraphShim)
    monkeypatch.setenv("TLAG_NO_STATES_DIR", "1")


def _tlc(argv, capsys):
    from tla_rust_b200.cli import tlc_main
    rc = tlc_main(argv)
    cap = capsys.readouterr()
    return rc, cap.out, cap.err


# demo/lock.tla (Peterson's algorithm): its 26 states, numbered by level, then by fingerprint within a level
LOCK_STATES = r'''State 1:
/\ flag = (0 :> FALSE @@ 1 :> FALSE)
/\ turn = 0
/\ pc = (0 :> "a1" @@ 1 :> "a1")

State 2:
/\ flag = (0 :> FALSE @@ 1 :> TRUE)
/\ turn = 0
/\ pc = (0 :> "a1" @@ 1 :> "a2")

State 3:
/\ flag = (0 :> TRUE @@ 1 :> FALSE)
/\ turn = 0
/\ pc = (0 :> "a2" @@ 1 :> "a1")

State 4:
/\ flag = (0 :> FALSE @@ 1 :> TRUE)
/\ turn = 0
/\ pc = (0 :> "a1" @@ 1 :> "a3")

State 5:
/\ flag = (0 :> TRUE @@ 1 :> TRUE)
/\ turn = 0
/\ pc = (0 :> "a2" @@ 1 :> "a2")

State 6:
/\ flag = (0 :> TRUE @@ 1 :> FALSE)
/\ turn = 1
/\ pc = (0 :> "a3" @@ 1 :> "a1")

State 7:
/\ flag = (0 :> TRUE @@ 1 :> TRUE)
/\ turn = 0
/\ pc = (0 :> "a2" @@ 1 :> "a3")

State 8:
/\ flag = (0 :> FALSE @@ 1 :> TRUE)
/\ turn = 0
/\ pc = (0 :> "a1" @@ 1 :> "cs")

State 9:
/\ flag = (0 :> TRUE @@ 1 :> FALSE)
/\ turn = 1
/\ pc = (0 :> "cs" @@ 1 :> "a1")

State 10:
/\ flag = (0 :> TRUE @@ 1 :> TRUE)
/\ turn = 1
/\ pc = (0 :> "a3" @@ 1 :> "a2")

State 11:
/\ flag = (0 :> FALSE @@ 1 :> TRUE)
/\ turn = 0
/\ pc = (0 :> "a1" @@ 1 :> "a4")

State 12:
/\ flag = (0 :> TRUE @@ 1 :> TRUE)
/\ turn = 0
/\ pc = (0 :> "a3" @@ 1 :> "a3")

State 13:
/\ flag = (0 :> TRUE @@ 1 :> TRUE)
/\ turn = 1
/\ pc = (0 :> "a3" @@ 1 :> "a3")

State 14:
/\ flag = (0 :> TRUE @@ 1 :> TRUE)
/\ turn = 0
/\ pc = (0 :> "a2" @@ 1 :> "cs")

State 15:
/\ flag = (0 :> TRUE @@ 1 :> FALSE)
/\ turn = 1
/\ pc = (0 :> "a4" @@ 1 :> "a1")

State 16:
/\ flag = (0 :> TRUE @@ 1 :> TRUE)
/\ turn = 1
/\ pc = (0 :> "cs" @@ 1 :> "a2")

State 17:
/\ flag = (0 :> TRUE @@ 1 :> TRUE)
/\ turn = 0
/\ pc = (0 :> "a2" @@ 1 :> "a4")

State 18:
/\ flag = (0 :> FALSE @@ 1 :> FALSE)
/\ turn = 1
/\ pc = (0 :> "a1" @@ 1 :> "a1")

State 19:
/\ flag = (0 :> TRUE @@ 1 :> TRUE)
/\ turn = 1
/\ pc = (0 :> "a3" @@ 1 :> "cs")

State 20:
/\ flag = (0 :> TRUE @@ 1 :> TRUE)
/\ turn = 1
/\ pc = (0 :> "a4" @@ 1 :> "a2")

State 21:
/\ flag = (0 :> TRUE @@ 1 :> TRUE)
/\ turn = 0
/\ pc = (0 :> "cs" @@ 1 :> "a3")

State 22:
/\ flag = (0 :> TRUE @@ 1 :> TRUE)
/\ turn = 0
/\ pc = (0 :> "a4" @@ 1 :> "a3")

State 23:
/\ flag = (0 :> TRUE @@ 1 :> FALSE)
/\ turn = 1
/\ pc = (0 :> "a2" @@ 1 :> "a1")

State 24:
/\ flag = (0 :> FALSE @@ 1 :> TRUE)
/\ turn = 1
/\ pc = (0 :> "a1" @@ 1 :> "a2")

State 25:
/\ flag = (0 :> TRUE @@ 1 :> TRUE)
/\ turn = 1
/\ pc = (0 :> "a3" @@ 1 :> "a4")

State 26:
/\ flag = (0 :> TRUE @@ 1 :> TRUE)
/\ turn = 1
/\ pc = (0 :> "a2" @@ 1 :> "a2")

'''

LOCK_DOT = r'''digraph StateGraph {
1 [label="/\\ flag = (0 :> FALSE @@ 1 :> FALSE)\n/\\ turn = 0\n/\\ pc = (0 :> \"a1\" @@ 1 :> \"a1\")",style=filled];
2 [label="/\\ flag = (0 :> FALSE @@ 1 :> TRUE)\n/\\ turn = 0\n/\\ pc = (0 :> \"a1\" @@ 1 :> \"a2\")"];
3 [label="/\\ flag = (0 :> TRUE @@ 1 :> FALSE)\n/\\ turn = 0\n/\\ pc = (0 :> \"a2\" @@ 1 :> \"a1\")"];
4 [label="/\\ flag = (0 :> FALSE @@ 1 :> TRUE)\n/\\ turn = 0\n/\\ pc = (0 :> \"a1\" @@ 1 :> \"a3\")"];
5 [label="/\\ flag = (0 :> TRUE @@ 1 :> TRUE)\n/\\ turn = 0\n/\\ pc = (0 :> \"a2\" @@ 1 :> \"a2\")"];
6 [label="/\\ flag = (0 :> TRUE @@ 1 :> FALSE)\n/\\ turn = 1\n/\\ pc = (0 :> \"a3\" @@ 1 :> \"a1\")"];
7 [label="/\\ flag = (0 :> TRUE @@ 1 :> TRUE)\n/\\ turn = 0\n/\\ pc = (0 :> \"a2\" @@ 1 :> \"a3\")"];
8 [label="/\\ flag = (0 :> FALSE @@ 1 :> TRUE)\n/\\ turn = 0\n/\\ pc = (0 :> \"a1\" @@ 1 :> \"cs\")"];
9 [label="/\\ flag = (0 :> TRUE @@ 1 :> FALSE)\n/\\ turn = 1\n/\\ pc = (0 :> \"cs\" @@ 1 :> \"a1\")"];
10 [label="/\\ flag = (0 :> TRUE @@ 1 :> TRUE)\n/\\ turn = 1\n/\\ pc = (0 :> \"a3\" @@ 1 :> \"a2\")"];
11 [label="/\\ flag = (0 :> FALSE @@ 1 :> TRUE)\n/\\ turn = 0\n/\\ pc = (0 :> \"a1\" @@ 1 :> \"a4\")"];
12 [label="/\\ flag = (0 :> TRUE @@ 1 :> TRUE)\n/\\ turn = 0\n/\\ pc = (0 :> \"a3\" @@ 1 :> \"a3\")"];
13 [label="/\\ flag = (0 :> TRUE @@ 1 :> TRUE)\n/\\ turn = 1\n/\\ pc = (0 :> \"a3\" @@ 1 :> \"a3\")"];
14 [label="/\\ flag = (0 :> TRUE @@ 1 :> TRUE)\n/\\ turn = 0\n/\\ pc = (0 :> \"a2\" @@ 1 :> \"cs\")"];
15 [label="/\\ flag = (0 :> TRUE @@ 1 :> FALSE)\n/\\ turn = 1\n/\\ pc = (0 :> \"a4\" @@ 1 :> \"a1\")"];
16 [label="/\\ flag = (0 :> TRUE @@ 1 :> TRUE)\n/\\ turn = 1\n/\\ pc = (0 :> \"cs\" @@ 1 :> \"a2\")"];
17 [label="/\\ flag = (0 :> TRUE @@ 1 :> TRUE)\n/\\ turn = 0\n/\\ pc = (0 :> \"a2\" @@ 1 :> \"a4\")"];
18 [label="/\\ flag = (0 :> FALSE @@ 1 :> FALSE)\n/\\ turn = 1\n/\\ pc = (0 :> \"a1\" @@ 1 :> \"a1\")"];
19 [label="/\\ flag = (0 :> TRUE @@ 1 :> TRUE)\n/\\ turn = 1\n/\\ pc = (0 :> \"a3\" @@ 1 :> \"cs\")"];
20 [label="/\\ flag = (0 :> TRUE @@ 1 :> TRUE)\n/\\ turn = 1\n/\\ pc = (0 :> \"a4\" @@ 1 :> \"a2\")"];
21 [label="/\\ flag = (0 :> TRUE @@ 1 :> TRUE)\n/\\ turn = 0\n/\\ pc = (0 :> \"cs\" @@ 1 :> \"a3\")"];
22 [label="/\\ flag = (0 :> TRUE @@ 1 :> TRUE)\n/\\ turn = 0\n/\\ pc = (0 :> \"a4\" @@ 1 :> \"a3\")"];
23 [label="/\\ flag = (0 :> TRUE @@ 1 :> FALSE)\n/\\ turn = 1\n/\\ pc = (0 :> \"a2\" @@ 1 :> \"a1\")"];
24 [label="/\\ flag = (0 :> FALSE @@ 1 :> TRUE)\n/\\ turn = 1\n/\\ pc = (0 :> \"a1\" @@ 1 :> \"a2\")"];
25 [label="/\\ flag = (0 :> TRUE @@ 1 :> TRUE)\n/\\ turn = 1\n/\\ pc = (0 :> \"a3\" @@ 1 :> \"a4\")"];
26 [label="/\\ flag = (0 :> TRUE @@ 1 :> TRUE)\n/\\ turn = 1\n/\\ pc = (0 :> \"a2\" @@ 1 :> \"a2\")"];
1 -> 2 [label="a1"];
1 -> 3 [label="a1"];
2 -> 4 [label="a2"];
2 -> 5 [label="a1"];
3 -> 5 [label="a1"];
3 -> 6 [label="a2"];
4 -> 7 [label="a1"];
4 -> 8 [label="a3"];
5 -> 7 [label="a2"];
5 -> 10 [label="a2"];
6 -> 9 [label="a3"];
6 -> 10 [label="a1"];
7 -> 13 [label="a2"];
8 -> 11 [label="cs"];
8 -> 14 [label="a1"];
9 -> 15 [label="cs"];
9 -> 16 [label="a1"];
10 -> 12 [label="a2"];
11 -> 1 [label="a4"];
11 -> 17 [label="a1"];
12 -> 21 [label="a3"];
13 -> 19 [label="a3"];
14 -> 17 [label="cs"];
14 -> 19 [label="a2"];
15 -> 18 [label="a4"];
15 -> 20 [label="a1"];
16 -> 20 [label="cs"];
16 -> 21 [label="a2"];
17 -> 3 [label="a4"];
17 -> 25 [label="a2"];
18 -> 23 [label="a1"];
18 -> 24 [label="a1"];
19 -> 25 [label="cs"];
20 -> 22 [label="a2"];
20 -> 24 [label="a4"];
21 -> 22 [label="cs"];
22 -> 4 [label="a4"];
23 -> 6 [label="a2"];
23 -> 26 [label="a1"];
24 -> 4 [label="a2"];
24 -> 26 [label="a1"];
25 -> 6 [label="a4"];
26 -> 7 [label="a2"];
26 -> 10 [label="a2"];
}
'''


def test_tlc_dump_writes_the_states_of_demo_lock(shim, tmp_path, capsys):
    out_file = tmp_path / "lock_states.txt"
    rc, out, _ = _tlc(["-dump", str(out_file), _demo("lock", tmp_path)], capsys)
    assert rc == 0, out
    assert out.splitlines()[-2] == f"Dumped 26 states to {out_file}."
    assert out_file.read_text() == LOCK_STATES


def test_tlc_dump_dot_writes_the_state_graph_of_demo_lock(shim, tmp_path, capsys):
    out_file = tmp_path / "lock.dot"
    rc, out, _ = _tlc(["-dump", "dot,colorize,actionlabels", str(out_file), _demo("lock", tmp_path)], capsys)
    assert rc == 0, out
    assert "Warning" not in out
    text = out_file.read_text()
    assert out.splitlines()[-2] == f"Dumped the state graph (26 states, {text.count(' -> ')} transitions) to {out_file}."
    assert text == LOCK_DOT


def test_tlc_dump_dot_warns_about_an_unknown_qualifier(shim, tmp_path, capsys):
    rc, out, _ = _tlc(["-dump", "dot,pretty", str(tmp_path / "g.dot"), _demo("lock", tmp_path)], capsys)
    assert rc == 0
    assert [ln for ln in out.splitlines() if ln.startswith("Warning:")] == ["Warning: -dump dot: unknown qualifier pretty ignored."]


def _dot_edges(text):
    edges = []
    for ln in text.splitlines():
        if " -> " in ln:
            k, rest = ln.split(" -> ")
            edges.append((int(k), int(rest.split(" ")[0])))
    return edges


def _dot_nodes(text):
    return [int(ln.split(" ")[0]) for ln in text.splitlines() if "[label=" in ln and " -> " not in ln]


def test_tlc_dump_dot_after_a_violation_has_no_edges_out_of_the_last_level(shim, tmp_path, capsys):
    from oracle import cpu_engine
    out_file = tmp_path / "race.dot"
    spec = _demo("race", tmp_path)
    rc, out, _ = _tlc(["-dump", "dot", str(out_file), spec], capsys)
    assert rc == 12 and "Error: Invariant Correct is violated." in out
    text = out_file.read_text()
    nodes, edges = _dot_nodes(text), _dot_edges(text)
    cm, init, _exp, info = _fixture("demo_race")
    levels = [n for n in cpu_engine.run(cm, init, deadlock=info["deadlock"])["levels"] if n]
    assert len(nodes) == sum(levels) and edges
    first_of_last = sum(levels[:-1]) + 1            # states are numbered from 1, level by level
    assert all(k < first_of_last for k, _ in edges)
    assert any(j >= first_of_last for _, j in edges)


def test_tlc_dump_takes_its_file_argument(shim, tmp_path, capsys):
    """`tlc -dump x Spec.tla` checks Spec.tla only and writes x (it used to check x.tla as a second spec)"""
    spec = _demo("lock", tmp_path)
    rc, out, _ = _tlc(["-dump", str(tmp_path / "x"), spec], capsys)
    assert rc == 0, out
    assert out.count("Parsing file") == 1 and (tmp_path / "x").exists()
    rc, out, _ = _tlc(["-dump", "dot", str(tmp_path / "g.dot"), spec], capsys)
    assert rc == 0 and out.count("Parsing file") == 1 and (tmp_path / "g.dot").exists()


def test_tlc_dump_is_refused_with_simulate_and_several_gpus(tmp_path, capsys):
    spec = os.path.join(ROOT, "models", "demo", "lock.tla")
    rc, _out, err = _tlc(["-dump", str(tmp_path / "x"), "-simulate", spec], capsys)
    assert rc == 2 and "-dump" in err
    rc, _out, err = _tlc(["-gpus", "2", "-dump", "dot", str(tmp_path / "g.dot"), spec], capsys)
    assert rc == 2 and "-dump" in err
    assert not os.path.exists(tmp_path / "x") and not os.path.exists(tmp_path / "g.dot")


# ---- 4. the libraries cross-compile and export the entry points -------------------------------------------------------
GRAPH_EXPORTS = ("tlag_build_graph", "tlag_read_graph", "tlag_graph_digest")


def _exports(so):
    syms = subprocess.run(["nm", "-D", "--defined-only", so], capture_output=True, text=True).stdout
    return all(f" T {fn}\n" in syms for fn in GRAPH_EXPORTS), syms


def test_the_engine_library_exports_the_graph_calls():
    from tla_rust_b200 import engine
    ok, _ = _exports(engine.LIB_PATH)
    assert ok
    assert all(fn in engine.EXPORTS for fn in GRAPH_EXPORTS)


@pytest.mark.parametrize("name,scalar", [("MCPaxos3_b2", True), ("MCraft", False)])
def test_sliced_libraries_cross_compile_with_one_edge_kernel(name, scalar):
    from tla_rust_b200 import engine
    cm, _, _, _ = _fixture(name)
    so = engine.build_sliced_library(cm, scalar=scalar)
    ok, syms = _exports(so)
    assert ok
    engine._bind(so)
    # one instantiation of the interpreter's edge pass, the variant of the model's frame class
    assert len([ln for ln in syms.splitlines() if "k_graphILi" in ln and "device_stub" not in ln]) == 1


# ---- 5-10. device -----------------------------------------------------------------------------------------------------
DEVICE_FIXTURES = ["demo_race", "pcal_intro_readme_buggy", "MCVoting_deadlock", "MCPaxos3_b2", "MCPaxos3_sym", "MCraft",
                   "MCssi_3x1", "MCInnerFIFO"]
# fixtures whose search stops at a violation or never ends
STOPPED = {"demo_race", "pcal_intro_readme_buggy", "MCssi_3x1"}


def _search(cm, init, native, deadlock, depth=0):
    from tla_rust_b200.engine import Engine
    e = Engine(cm, deadlock=deadlock, native=native)
    e.seed(init)
    while True:
        if depth and e.result()["depth"] >= depth:
            break
        if e.step()["verdict"] != 5:
            break
    return e


def _triples(L, states, off, dst, act):
    fps = fingerprints(L, states)
    src = np.repeat(np.arange(len(off) - 1), np.diff(off.astype(np.int64)))
    return sorted((fps[s], fps[t], a) for s, t, a in zip(src.tolist(), dst.tolist(), act.tolist()))


def _check_against_ref(libdir, e, cm, g):
    L = ref_lib(libdir)
    states = e.read_states(0, g["n_states"])
    off, dst, act = e.state_graph()
    assert len(off) == g["n_states"] + 1 and int(off[-1]) == g["n_edges"] == len(dst)
    assert (np.diff(off.astype(np.int64)) >= 0).all()
    assert int(off[g["n_expanded"]]) == g["n_edges"]        # no edge leaves an unexpanded row
    assert (dst < g["n_states"]).all()
    src = np.repeat(np.arange(g["n_states"]), np.diff(off.astype(np.int64)))
    assert (src != dst).all()
    # CSR order, within a row by (t, a), each triple once: graph_ref's edges are sorted and distinct
    rs, rd, ra = ref_graph(L, cm, states, g["n_expanded"])
    assert np.array_equal(src, rs) and np.array_equal(dst, rd) and np.array_equal(act, ra)
    fps = fingerprints(L, states)
    assert e.graph_digest() == graph_digest_np([fps[s] for s in src], [fps[t] for t in dst], act)
    return states, off, dst, act


@pytest.mark.gpu
@pytest.mark.parametrize("native", [False, "sliced"])
@pytest.mark.parametrize("name", [n for n in DEVICE_FIXTURES if n not in STOPPED])
def test_device_graph_at_the_fixpoint_matches_graph_ref(libdir, name, native):
    cm, init, _exp, info = _fixture(name)
    e = _search(cm, init, native, deadlock=False)
    assert e.result()["verdict"] == 0
    g = e.build_graph()
    assert g["n_expanded"] == g["n_states"] == e.result()["distinct"]
    _states, off, dst, act = _check_against_ref(libdir, e, cm, g)
    # every parent link is an edge
    for idx in range(g["n_states"]):
        _st, par, a, _rank = e.read_link(idx)
        if par >= 0:
            row = slice(int(off[par]), int(off[par + 1]))
            assert ((dst[row] == idx) & (act[row] == a)).any(), (name, idx)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("native", [False, "sliced"])
@pytest.mark.parametrize("name", sorted(STOPPED))
def test_device_graph_of_a_stopped_search_leaves_the_expanded_rows_only(libdir, name, native):
    cm, init, _exp, info = _fixture(name)
    depth = 6 if name == "MCssi_3x1" else 0
    e = _search(cm, init, native, deadlock=info["deadlock"], depth=depth)
    r = e.result()
    first, count = e.frontier()
    g = e.build_graph()
    assert g["n_states"] == r["distinct"] and g["n_expanded"] == first and first + count == r["distinct"]
    # (demo_race's violating level discovers nothing new: its frontier is empty)
    assert 0 < g["n_expanded"] <= g["n_states"] and (g["n_expanded"] < g["n_states"] or name == "demo_race")
    _check_against_ref(libdir, e, cm, g)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("native", [False, "sliced"])
def test_chunking_and_store_order_do_not_change_the_graph(libdir, monkeypatch, native):
    cm, init, _exp, info = _fixture("MCPaxos3_b2")
    L = ref_lib(libdir)
    runs = []
    for env in ({}, {"TLAG_GRAPH_EDGES": "4096"}, {"TLAG_NO_SORT": "1"}):
        for k in ("TLAG_GRAPH_EDGES", "TLAG_NO_SORT"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        e = _search(cm, init, native, deadlock=False)
        g = e.build_graph()
        assert g["n_edges"] > 4 * 4096
        states = e.read_states(0, g["n_states"])
        runs.append((g["n_edges"], e.graph_digest(), _triples(L, states, *e.state_graph())))
        e.close()
    assert runs[0] == runs[1] == runs[2]


@pytest.mark.gpu
@pytest.mark.parametrize("native", [False, "sliced"])
def test_a_buffer_smaller_than_one_states_edges_grows(libdir, monkeypatch, native):
    """TLAG_GRAPH_EDGES=1: chunks halve down to one row, and a row with more edges than the buffer gets a bigger one"""
    cm, init, _exp, info = _fixture("MCInnerFIFO")
    L = ref_lib(libdir)
    runs = []
    for edges in (None, "1"):
        monkeypatch.delenv("TLAG_GRAPH_EDGES", raising=False)
        if edges:
            monkeypatch.setenv("TLAG_GRAPH_EDGES", edges)
        e = _search(cm, init, native, deadlock=False)
        g = e.build_graph()
        states = e.read_states(0, g["n_states"])
        off, dst, act = e.state_graph()
        assert int(np.diff(off.astype(np.int64)).max()) > 1
        runs.append((g["n_edges"], e.graph_digest(), _triples(L, states, off, dst, act)))
        e.close()
    assert runs[0] == runs[1]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["MCPaxos3_b4", "MCraft_t4l3"])
def test_both_engines_build_the_same_graph_at_scale(name):
    cm, init, _exp, info = _fixture(name)
    got = {}
    for native in (False, "sliced"):
        e = _search(cm, init, native, deadlock=info["deadlock"])
        r = e.result()
        g = e.build_graph()
        assert g["n_expanded"] == g["n_states"] == r["distinct"]
        got[native] = (g["n_edges"], e.graph_digest())
        # a random sample of 10^5 parent links are all edges
        rng = np.random.default_rng(1)
        n_init = r["init_states"]
        sample = rng.integers(n_init, r["distinct"], min(10 ** 5, r["distinct"] - n_init))
        parents = {}
        for idx in sample.tolist():
            _st, par, a, _rank = e.read_link(idx)
            parents[idx] = (par, a)
        for idx, (par, a) in parents.items():
            off, dst, act = e.state_graph(par, 1)
            assert ((dst == idx) & (act == a)).any(), (name, native, idx)
        e.close()
    assert got[False] == got["sliced"]


@pytest.mark.gpu
def test_refusals_and_release():
    from tla_rust_b200.engine import Engine, EngineError
    cm, init, _exp, info = _fixture("demo_race")
    e = Engine(cm, deadlock=info["deadlock"], native=False)
    with pytest.raises(EngineError, match="rc=-7"):          # not seeded
        e.build_graph()
    e.seed(init)
    e.step()
    e.build_graph()
    e.state_graph()
    e.step()
    with pytest.raises(EngineError, match="rc=-7"):          # released by the step
        e.state_graph()
    e.close()
    e = Engine(cm, deadlock=info["deadlock"], native=False, exact=True)
    e.seed(init)
    e.run()
    with pytest.raises(EngineError, match="rc=-1"):
        e.build_graph()
    e.close()
    e = Engine(cm, deadlock=info["deadlock"], native="sliced", simulate=True)
    e.seed(init)
    with pytest.raises(EngineError, match="rc=-1"):
        e.build_graph()
    e.close()


def _tlc_gpu(spec, engine, out_file):
    env = dict(os.environ, TLAG_NO_STATES_DIR="1")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "tlc"), "-dump", "dot", out_file, "-engine", engine, spec],
                       capture_output=True, text=True, timeout=1200, env=env)
    return p.returncode, open(out_file).read()


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["race", "pcal_intro"])
def test_tlc_dump_dot_end_to_end_on_the_device(libdir, tmp_path, monkeypatch, capsys, which):
    if which == "pcal_intro" and not os.path.isdir(REF):
        pytest.skip("no tla-rust spec corpus")
    spec = _demo("race", tmp_path) if which == "race" else _pcal("pcal_intro", tmp_path)
    rc_i, dot_i = _tlc_gpu(spec, "interp", str(tmp_path / "i.dot"))
    rc_s, dot_s = _tlc_gpu(spec, "sliced", str(tmp_path / "s.dot"))
    assert rc_i == rc_s and dot_i == dot_s and " -> " in dot_i
    import tla_rust_b200.engine as eng
    _CpuGraphShim.lib_dir = libdir
    monkeypatch.setattr(eng, "Engine", _CpuGraphShim)
    monkeypatch.setenv("TLAG_NO_STATES_DIR", "1")
    rc_c, _out, _ = _tlc(["-dump", "dot", str(tmp_path / "c.dot"), spec], capsys)
    assert rc_c == rc_i and (tmp_path / "c.dot").read_text() == dot_i
