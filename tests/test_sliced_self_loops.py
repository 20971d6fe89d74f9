"""Self-loop filter of the sliced native build (scalar form): a successor whose packed words equal its parent's is
counted (generated, the parent's has-a-successor flag) and dropped before the fingerprint and the seen-set probe.  The
parent is a stored state, so the probe could only have found it: counts, per-level sizes and digests must not move,
with the filter on (the default) or off (TLAG_SL_SKIPSELF=0, read when the engine is created).  On the CPU the same generated C runs
inside the CPU bytecode engine with the filter compiled in or out (and, filter on, in tests/test_sliced.py)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from tla_rust_b200.compiled import load_compiled
from tla_rust_b200.compile.sliced import Emitter, emit_sliced


def test_every_scalar_emit_site_tests_for_a_self_loop():
    cm, _, _, _ = load_compiled(os.path.join(GOLDEN, "MCPaxos3_b4.tlagz"))
    src = emit_sliced(cm, scalar=True)
    body = src.split("#define TLAG_SL_NEXT_LIST")[1]
    sites = body.count("TLAG_SL_EMITW(")
    assert sites > 0 and body.count("if (TLAG_SL_SKIPSELF") == sites
    # a full pack compares every packed word with the parent's
    assert all(f"(o_[{j}] ^ in_[{j}])" in body for j in range(cm.W))


def test_a_dirty_range_emit_compares_only_the_words_it_writes():
    cm, _, _, _ = load_compiled(os.path.join(GOLDEN, "MCPaxos3_b4.tlagz"))
    e = Emitter(cm, scalar=True)
    # the first slot alone (bit 0 of word 0), as an EMITD dirty table in a copy of the constant pool
    width = e.layout[0][1]
    assert width <= 32
    e.cpool = e.cpool + [1, 0, 1, 0]
    text = e.emit_stmt(5, len(e.cpool) - 4, "")
    assert "(o_[0] ^ in_[0])" in text and "(o_[1] ^ in_[1])" not in text
    assert text.rstrip().endswith("TLAG_SL_EMITW(5, o_); }")


@pytest.mark.parametrize("skip_self", ["0", "1"])
def test_generated_c_matches_the_oracle_on_the_cpu_with_and_without_the_filter(tmp_path, skip_self):
    """The scalar form's generated C inside the CPU bytecode engine (oracle/tlag_cpu.c), the filter compiled in or out:
    a site that dropped a successor it should have kept, or kept the wrong one, moves the counts or the digest."""
    import ctypes as C
    import subprocess
    from conftest import ROOT
    from oracle import cpu_engine
    for name in ("MCPaxos3", "pcal_intro", "pcal_intro_readme_buggy", "demo_race", "demo_lock", "MCInnerFIFO"):
        cm, init, exp, info = load_compiled(os.path.join(GOLDEN, name + ".tlagz"))
        inc = tmp_path / f"{name}_{skip_self}.inc"
        inc.write_text(emit_sliced(cm, scalar=True))
        so = tmp_path / f"{name}_{skip_self}.so"
        subprocess.check_call(["gcc", "-O1", "-std=gnu11", "-fPIC", "-shared", "-pthread", "-Wno-unused-label",
                               "-Wno-unused-function", f"-DTLAG_SL_SKIPSELF={skip_self}", f'-DTLAG_SLICED_INC="{inc}"',
                               "-o", str(so), os.path.join(ROOT, "oracle", "tlag_cpu.c")])
        cpu_engine.lib()
        saved, cpu_engine._LIB = cpu_engine._LIB, C.CDLL(str(so))
        try:
            r = cpu_engine.run(cm, init, n_threads=2, deadlock=info["deadlock"])
        finally:
            cpu_engine._LIB = saved
        for k in ("verdict", "generated", "distinct", "depth", "fp_xor", "fp_sum", "levels"):
            assert r[k] == exp["o2"][k], (name, skip_self, k)


# scalar form (Paxos, PlusCal: ok, an Assert failure, an invariant violation) and array form (Paxos with SYMMETRY, Voting with a deadlock, raft, SSI with eight
# invariants: models with subroutines), where the switch must change nothing
CASES = [("MCPaxos3_b3", 0), ("pcal_intro", 0), ("pcal_intro_readme_buggy", 0), ("demo_race", 0), ("MCPaxos3_sym", 0),
         ("MCVoting_deadlock", 0), ("MCraft_t4l3", 0), ("MCssi_4x3", 8)]


@pytest.mark.gpu
@pytest.mark.parametrize("skip_self", ["0", "1"])
@pytest.mark.parametrize("name,max_levels", CASES)
def test_sliced_kernels_match_the_oracle_with_and_without_the_filter(monkeypatch, name, max_levels, skip_self):
    from tla_rust_b200.engine import V_RUNNING, Engine
    monkeypatch.setenv("TLAG_SL_SKIPSELF", skip_self)
    cm, init, exp, info = load_compiled(os.path.join(GOLDEN, name + ".tlagz"))
    o2 = exp["o2"]
    e = Engine(cm, deadlock=info["deadlock"], native="sliced")
    e.seed(init)
    levels = [int(len(np.unique(init, axis=0)))]
    while not max_levels or len(levels) < max_levels:
        ws = e.step()
        if ws["expanded"]:
            levels.append(int(ws["discovered"]))
        if ws["verdict"] != V_RUNNING:
            break
    r = e.result()
    if max_levels:
        x, sm, gen = o2["level_digests"][max_levels - 1]
        assert (r["generated"], r["distinct"], r["depth"]) == (gen, sum(o2["levels"][:max_levels]), max_levels)
        assert levels == o2["levels"][:max_levels]
        assert e.digest() == (x, sm)
    else:
        assert r["verdict"] == o2["verdict"], (r, o2)
        assert (r["generated"], r["distinct"], r["depth"]) == (o2["generated"], o2["distinct"], o2["depth"])
        assert levels == o2["levels"]
        assert e.digest() == (o2["fp_xor"], o2["fp_sum"])
    e.close()
