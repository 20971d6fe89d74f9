"""Command-line front ends replacing the two external commands the reference's Makefile shells out to
(Makefile:3-7): `pcal2tla FILE.tla...` and `tlc FILE.tla...` (several files per invocation, FILE.cfg
looked up next to FILE.tla, TLC-format report on stdout, non-zero exit status on any error so that
`make` stops).  The search itself runs on the GPU through the C ABI; there is no CPU backend."""
from __future__ import annotations

import os
import sys
import time

from .front.spec import Model, SpecError
from .front.parser import ParseError
from .front.lexer import LexError
from .front.values import EvalError
from .front.pcal import translate_file, PcalError
from .front.report import format_result, OK, CheckResult, PROPERTY
from .compile.lower import CompileError
from .compile.types import TypeErr

# `tlc -engine auto`: programs of at least this many bytecode instructions are compiled to sliced kernels (about 10 s of
# nvcc per thousand instructions, cached per model); smaller ones run on the interpreter kernel at once.
AUTO_SLICED_MIN_CODE = int(os.environ.get("TLAG_AUTO_SLICED_MIN_CODE", "1500"))
# an Assert failure / deadlock found within this many states is replayed sequentially for TLC-exact counts and trace
EXACT_REPLAY_MAX_STATES = int(os.environ.get("TLAG_EXACT_REPLAY_MAX_STATES", "200000"))


def pcal2tla_main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    files = [a for a in argv if not a.startswith("-")]
    nocfg = "-nocfg" in argv
    if not files:
        print("usage: pcal2tla [-nocfg] FILE.tla ...", file=sys.stderr)
        return 2
    rc = 0
    for f in files:
        if not f.endswith(".tla"):
            f += ".tla"
        try:
            had = translate_file(f, write_cfg=not nocfg)
            if had:
                print(f"pcal2tla: translated {f}")
            else:
                print(f"pcal2tla: no PlusCal algorithm in {f}; file unchanged")
        except (PcalError, LexError, OSError) as ex:
            print(f"pcal2tla: {f}: {ex}", file=sys.stderr)
            rc = 1
    return rc


def check_file(path, deadlock=True, cfg_path=None, out=None, device=0, seq_cap=None, verbose=True, lib_dirs=(),
               engine="auto", max_depth=0, simulate=None, dump=None):
    """engine: "interp" = bytecode interpreter kernel, "sliced" = the model compiled to one CUDA kernel per slice of its
    program (nvcc at run time, cached in csrc/native/), "auto" = sliced for programs big enough to repay the compile.
    max_depth = L: stop after level L exists (levels 1..L-1 expanded) and report the prefix.
    simulate = (num, seed): random simulation instead of the search, num behaviours of at most max_depth states (100 when
    0) from the given seed (include/tlag.h: tlag_simulate).
    dump = (path, dot qualifiers or None): after the report, write every stored state to path (TLC's -dump), or with
    qualifiers the state graph in Graphviz form (TLC's -dump dot)."""
    from .checker import compile_model, encode_states, result_from_engine
    from .engine import Engine
    t0 = time.time()
    if out is None:
        out = sys.stdout
    lib_dirs = list(lib_dirs) + [d for d in os.environ.get("TLA_LIBRARY", "").split(os.pathsep) if d]
    m = Model(path, cfg_path=cfg_path, extra_dirs=lib_dirs)
    m.ev.out = out
    for w in m.warnings:
        print(f"Warning: {w}", file=out)
    m.check_assumes()
    if m.next_node is None and not m.init_nodes:
        print("Model checking completed. No error has been found.", file=out)
        print("  (the module has no behaviour specification; only its assumptions were checked)", file=out)
        return 0
    init = m.initial_states()
    for st in init:      # Init => Init2 of each refinement PROPERTY (the step obligation is checked on the device)
        pbad = m.check_refinement_init(st)
        if pbad is not None:
            res = CheckResult()
            res.verdict, res.invariant, res.trace = PROPERTY, pbad, [(st, None)]
            res.generated = res.distinct = res.init_states = len(init)
            res.depth = 1
            res.error_text = f"Property {pbad} is violated by the initial state"
            print(format_result(res, m.vars, m.module_name), file=out)
            return 12
    # CONSTRAINT on initial states (TLC, ORACLE O1 oracle/tlc_oracle.py:158): an initial state outside the constraint is
    # generated and counted but never explored -- it is not handed to the engine, the counts are adjusted below
    init_all = init
    if m.constraints:
        init = [st for st in init_all if m.in_model(st)]
    n_out = len(init_all) - len(init)
    from .compile import types as _types
    base_sparse = _types.SPARSE_CAP
    try:
        for attempt in range(4):
            cm = compile_model(m, init, seq_cap=seq_cap)
            for w in cm.warnings:
                print(f"Warning: {w}", file=out)
            iw = encode_states(cm, init)
            native = "sliced" if (engine == "sliced" or (engine == "auto" and len(cm.code) >= AUTO_SLICED_MIN_CODE)) else False
            if native == "sliced" and verbose:
                print("Compiling the model to sm_90a kernels (one per invariant / disjunct of Next) ...", file=out)
            if simulate is not None:
                e = Engine(cm, deadlock=deadlock and m.check_deadlock, device=device, native=native, simulate=True)
                e.seed(iw)
                r = e.simulate(simulate[1], simulate[0], max_depth or 100)
                if r["verdict"] == 4 and r["detail"] == 2 and attempt < 3:
                    _types.SPARSE_CAP *= 2
                    seq_cap = 2 * (seq_cap or getattr(cm, "seq_cap", None) or 4)
                    print(f"Note: a default container capacity was exceeded; retrying with sparse capacity "
                          f"{_types.SPARSE_CAP} and sequence capacity {seq_cap}.", file=out)
                    e.close()
                    continue
                break
            world = int(os.environ.get("WORLD_SIZE", "1"))
            if world > 1:                   # `tlc -gpus N`: this process is one rank of N (see tlc_main)
                r, trace, e = _check_distributed(cm, iw, deadlock and m.check_deadlock, native, max_depth, out)
                if r["verdict"] == 4 and r["detail"] == 2 and attempt < 3:
                    _types.SPARSE_CAP *= 2
                    seq_cap = 2 * (seq_cap or getattr(cm, "seq_cap", None) or 4)
                    e.close()
                    continue
                break
            e = Engine(cm, deadlock=deadlock and m.check_deadlock, device=device, native=native)
            e.seed(iw)
            r0 = e.result()
            levels = [r0["distinct"]]            # states per BFS level, in store order (the order -dump numbers them in)
            print(f"Finished computing initial states: {r0['distinct']} distinct state"
                  f"{'s' if r0['distinct'] != 1 else ''} generated.", file=out)
            while True:
                if max_depth and e.result()["depth"] >= max_depth:
                    print(f"Depth bound {max_depth} reached: the states of the last level were not expanded.", file=out)
                    break
                ws = e.step()
                if ws.get("discovered"):
                    levels.append(ws["discovered"])
                if ws["verdict"] != 5:
                    break
                if verbose and ws["expanded"]:
                    print(f"Progress({ws['level']}): {ws['generated_total']} states generated, {ws['distinct_total']} "
                          f"distinct states found, {ws['discovered']} states left on queue.", file=out)
            r = e.result()
            # a container / sequence capacity chosen by default (not by the model's TypeOK) was too small: the run
            # stopped with a capacity trap (never a wrong answer) -- double the defaults and search again
            if r["verdict"] == 4 and r["detail"] == 2 and attempt < 3:
                _types.SPARSE_CAP *= 2
                seq_cap = 2 * (seq_cap or getattr(cm, "seq_cap", None) or 4)
                print(f"Note: a default container capacity was exceeded; retrying with sparse capacity "
                      f"{_types.SPARSE_CAP} and sequence capacity {seq_cap}.", file=out)
                e.close()
                continue
            break
    finally:
        _types.SPARSE_CAP = base_sparse
    if simulate is not None:
        if m.obligations:
            print("Warning: the temporal properties are not checked in simulation mode.", file=out)
        return _report_simulation(path, m, cm, r, e, simulate[1], t0, out)
    live = None
    if m.obligations and r["verdict"] == 0:
        live = _check_liveness(e, m, cm, r, max_depth, out)
    dumped = _dump(e, cm, m, levels, *dump) if dump is not None else None
    if int(os.environ.get("WORLD_SIZE", "1")) == 1:
        # The parallel search reports an error with the counts of the whole level it was found in, and with whichever of
        # several shortest behaviours won the race.  TLC's single worker stops AT the first Assert failure / deadlock
        # (README.md:319: 9097 generated / 6164 distinct / 999 on queue).  For a model small enough, replay the search as
        # one sequential worker on the device (TLAG_F_EXACT) and report that run: TLC's counts and TLC's trace.
        if r["verdict"] in (2, 3) and r["distinct"] <= EXACT_REPLAY_MAX_STATES and not max_depth:
            e.close()
            e = Engine(cm, deadlock=deadlock and m.check_deadlock, device=device, native=False, exact=True)
            e.seed(iw)
            r = e.run()
        trace = None
        if r["verdict"] != 0:
            trace = e.trace(r["state_idx"])
    if n_out:
        r = dict(r, generated=r["generated"] + n_out, distinct=r["distinct"] + n_out, init_states=r.get("init_states", 0) + n_out)
    res = result_from_engine(cm, r, trace)
    if live is not None:
        res = live(res)
    text = format_result(res, m.vars, m.module_name)
    print(text, file=out)
    _write_reports(path, m, res, text)
    if dumped is not None:
        print(dumped(), file=out)
    print(f"Finished in {time.time() - t0:.2f}s ({r['device_seconds']:.4f}s in GPU wave kernels, "
          f"{e.launches()} kernel launches).", file=out)
    e.close()
    return 0 if res.verdict == OK else 12


def _check_liveness(e, m, cm, r, max_depth, out):
    """The temporal obligations of the model on the search's state graph (DESIGN.md §7h), after a search that reached
    its fixpoint without an error.  -> None when they hold or were not checked, else the function that turns the
    search's result into the violation's report"""
    from . import liveness
    from .checker import decode_state
    from .front.report import INVARIANT, LIVENESS
    why = None
    if m.fairness_unknown:
        why = "(the fairness of the SPECIFICATION is not fully understood, see the warning above)"
    elif m.symmetry:
        why = "under SYMMETRY (unsound there, as in TLC)"
    elif int(os.environ.get("WORLD_SIZE", "1")) > 1:
        why = "on a search spread over several GPUs"
    elif max_depth and r["queue_left"]:
        why = "after a depth-bounded search"
    if why is not None:
        print(f"Warning: the temporal properties are not checked {why}.", file=out)
        return None
    print(f"Checking temporal properties for the complete state space with {r['distinct']} total distinct states.",
          file=out)
    found = liveness.check(e, m, cm, lambda w: print(f"Warning: {w}", file=out))
    if found is None:
        return None
    ob, lr = found
    trace, back, back_act = liveness.lasso(e, lr)

    def label(a):
        if a is None or a < 0:
            return None
        nm, loc, mod = cm.actions[a]
        return ("fixed", nm, loc, mod)

    def report(res):
        res.trace = [(decode_state(cm, w), label(a)) for w, a in trace]
        if ob.kind == "always":
            res.verdict, res.invariant = INVARIANT, ob.name
        else:
            res.verdict = LIVENESS
            res.back_to = None if back is None else (back + 1, label(back_act))
        return res
    return report


def _dump(e, cm, m, levels, path, dot):
    """`tlc -dump`: reads what the dump needs from the search's engine now (before an exact replay closes it) and returns
    the function that writes it (after the report) and says so.  States are numbered from 1 by BFS level, then by
    ascending 64-bit fingerprint within a level; with `dot` (the qualifiers) the nodes are those numbers, initial states
    filled, and the edges come from the state graph the engine builds in device memory."""
    from .checker import decode_state
    from .engine import EngineError
    from .fingerprint import fingerprint_words
    from .front.report import format_state
    n = sum(levels)
    words = e.read_states(0, n) if n else []
    order, a = [], 0
    for size in levels:
        order += sorted(range(a, a + size), key=lambda i: fingerprint_words(words[i]))
        a += size
    num = {row: k for k, row in enumerate(order, 1)}
    text = {row: format_state(decode_state(cm, words[row]), m.vars) for row in order}
    edges = None
    if dot is not None:
        try:
            e.build_graph()
            off, dst, act = e.state_graph(0, n)
        except EngineError as ex:
            return lambda: f"The state graph was not dumped: {ex}"
        edges = sorted((num[s], num[int(dst[j])], int(act[j])) for s in range(n) for j in range(int(off[s]), int(off[s + 1])))

    def write():
        with open(path, "w") as f:
            if edges is None:
                for row in order:
                    f.write(f"State {num[row]}:\n{text[row]}\n\n")
                return f"Dumped {n} states to {path}."
            f.write("digraph StateGraph {\n")
            for row in order:
                label = text[row].replace("\\", "\\\\").replace('"', '\\"').replace("\n", "\\n")
                f.write(f'{num[row]} [label="{label}"{",style=filled" if row < levels[0] else ""}];\n')
            for k, j, a_ in edges:
                f.write(f'{k} -> {j} [label="{cm.actions[a_][0]}"];\n')
            f.write("}\n")
        return f"Dumped the state graph ({n} states, {len(edges)} transitions) to {path}."
    return write


def _write_reports(path, m, res, text):
    # TLC keeps its metadata (fingerprint set, trace file) under ./states/ (reference .gitignore:2); the state store of
    # this checker lives in HBM, what is worth keeping on disk is the report: states/<module>.out, and the behaviour
    # leading to an error as states/<module>.trace
    if int(os.environ.get("RANK", "0")) == 0 and os.environ.get("TLAG_NO_STATES_DIR") != "1":
        try:
            sd = os.path.join(os.path.dirname(os.path.abspath(path)), "states")
            os.makedirs(sd, exist_ok=True)
            with open(os.path.join(sd, m.module_name + ".out"), "w") as f:
                f.write(text + "\n")
            tr = os.path.join(sd, m.module_name + ".trace")
            lines = text.splitlines()
            if res.trace and any(ln.startswith("State 1:") for ln in lines):
                first = next(i for i, ln in enumerate(lines) if ln.startswith("State 1:"))
                last = max(i for i, ln in enumerate(lines) if ln.startswith("/\\") or ln.startswith("State "))
                with open(tr, "w") as f:
                    f.write("\n".join(lines[first:last + 1]) + "\n")
            elif os.path.exists(tr):
                os.remove(tr)
        except Exception:  # noqa: BLE001 -- the files are a convenience: never let them fail a check
            pass


def _report_simulation(path, m, cm, r, e, seed, t0, out):
    """`tlc -simulate`: the first error's behaviour in TLC's format, or the summary; the report files as for a search"""
    from .checker import result_from_engine
    trace = e.sim_trace(r["walk"]) if r["verdict"] != 0 else None
    res = result_from_engine(cm, dict(r, distinct=r["checked"], depth=len(trace[0]) if trace else 0), trace)
    stats = (f"{r['behaviours']} behaviours simulated, {r['checked']} states checked, {r['generated']} successors "
             f"generated (seed {seed}).")
    if res.verdict == OK:
        text = "Simulation completed. No error has been found.\n" + stats
    else:
        # the search's statistics lines do not apply: a walk has no queue and no search depth
        text = "\n".join(format_result(res, m.vars, m.module_name).splitlines()[:-2] + [stats])
    print(text, file=out)
    _write_reports(path, m, res, text)
    print(f"Finished in {time.time() - t0:.2f}s ({r['device_ms'] * 1e-3:.4f}s in GPU kernels, {e.launches()} kernel "
          f"launches).", file=out)
    e.close()
    return 0 if res.verdict == OK else 12


def _check_distributed(cm, iw, deadlock, native, max_depth, out):
    """One rank of `tlc -gpus N` (torchrun environment): the state space is partitioned over the N GPUs
    (tla_rust_b200/dist.py); every rank computes, rank 0 reports.  -> (result dict, trace or None, engine)"""
    import torch
    import torch.distributed as dist
    from .dist import DistributedBFS
    from .engine import Engine
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if not dist.is_initialized():
        dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    if native:                              # one rank compiles the model's kernels, the others wait for the library
        if rank == 0:
            from .engine import build_sliced_library
            build_sliced_library(cm)
        dist.barrier()
    e = Engine(cm, deadlock=deadlock, device=local, native=native)
    d = DistributedBFS(e, cm, rank, world, f"cuda:{local}", cap_records=1 << 24, chunk_states=1 << 21)
    d.seed(iw)
    import numpy as np
    n_init = int(len(np.unique(np.asarray(iw).reshape(-1, cm.W), axis=0)))
    print(f"Finished computing initial states: {n_init} distinct state{'s' if n_init != 1 else ''} generated "
          f"({world} GPUs, exchange: {d.exchange}).", file=out)
    res = d.run(max_levels=(max_depth - 1) if max_depth else 1 << 20)
    cex = d.counterexample()
    r = dict(verdict=res["verdict"] if res["verdict"] != 5 else 0, detail=0, detail2=0, generated=res["generated"],
             distinct=res["distinct"], depth=res["depth"], queue_left=0, init_states=n_init, state_idx=0,
             device_seconds=res["local"]["device_seconds"])
    trace = None
    if cex is not None:
        r["verdict"], r["detail"] = cex[0], cex[1]
        trace = (cex[2], cex[3])
    return r, trace, e


def _free_port():
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def tlc_main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    files, deadlock, cfg, dev, libs, seq_cap, engine, depth, gpus = [], True, None, 0, [], None, "auto", 0, 1
    sim_num, seed, dump = None, None, None
    i = 0
    while i < len(argv):
        a = argv[i]
        if a == "-deadlock":
            deadlock = False
        elif a == "-config":
            i += 1
            cfg = argv[i]
        elif a == "-I":                     # module search path (TLC: -DTLA-Library=...); also $TLA_LIBRARY
            i += 1
            libs.append(argv[i])
        elif a == "-seqcap":                # capacity of Seq(S)-typed variables (bounded by the model's CONSTRAINT)
            i += 1
            seq_cap = int(argv[i])
        elif a == "-engine":                # interp | sliced | auto
            i += 1
            engine = argv[i]
        elif a == "-depth":                 # depth-bounded prefix of the breadth-first search; with -simulate: behaviour length
            i += 1
            depth = int(argv[i])
        elif a == "-simulate":              # random behaviours instead of the search: -simulate [num=K]
            sim_num = 1 << 20
            if i + 1 < len(argv) and argv[i + 1].startswith("num="):
                i += 1
                sim_num = int(argv[i][4:])
        elif a == "-seed":
            i += 1
            seed = int(argv[i])
        elif a == "-dump":                  # -dump FILE: the states; -dump dot[,qualifiers] FILE: the state graph
            i += 1
            if argv[i] == "dot" or argv[i].startswith("dot,"):
                dump = (argv[i + 1], argv[i].split(",")[1:])
                # TLC's qualifiers are accepted so that its command lines work; the edges always carry their action
                for q in dump[1]:
                    if q not in ("actionlabels", "colorize", "snapshot"):
                        print(f"Warning: -dump dot: unknown qualifier {q} ignored.")
                i += 1
            else:
                dump = (argv[i], None)
        elif a == "-gpus":                  # partition the state space over N GPUs of this box (one process per GPU)
            i += 1
            gpus = int(argv[i])
        elif a in ("-workers", "-device", "-fpmem", "-coverage", "-checkpoint"):
            i += 1
            if a == "-device":
                dev = int(argv[i])
        elif a.startswith("-"):
            pass
        else:
            files.append(a)
        i += 1
    if not files:
        print("usage: tlc [-deadlock] [-config FILE.cfg] [-I DIR] [-seqcap N] [-engine interp|sliced|auto] [-depth N] [-gpus N] "
              "[-simulate [num=K] [-seed S]] [-dump [dot[,...]] FILE] FILE.tla ...", file=sys.stderr)
        return 2
    if dump is not None and (sim_num is not None or gpus > 1):
        print("tlc: -dump writes the states of a search on one GPU: drop -simulate and -gpus", file=sys.stderr)
        return 2
    if sim_num is not None and gpus > 1:
        print("tlc: -simulate runs on one GPU: drop -gpus", file=sys.stderr)
        return 2
    if sim_num is not None and sim_num < 1:
        print("tlc: -simulate num=K needs K >= 1", file=sys.stderr)
        return 2
    if sim_num is not None and seed is None:
        seed = int.from_bytes(os.urandom(8), "little") >> 1
    if gpus > 1 and "RANK" not in os.environ:
        # re-run this command as N ranks (torch.distributed.run is plumbing: rendezvous + one process per GPU)
        import subprocess
        import tempfile
        # the ranks leave the exit status (0 / 12 violation / 150 spec error ...) in a file and exit 0 themselves: a
        # non-zero rank makes the launcher print a failure report of its own on top of the TLC-format one
        with tempfile.NamedTemporaryFile(prefix="tlag_rc_", delete=False) as tf:
            rc_file = tf.name
        launcher = subprocess.call(
            [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={gpus}", "--master-addr", "127.0.0.1",
             "--master-port", str(_free_port()), "-m", "tla_rust_b200.cli"] + argv,
            env=dict(os.environ, TLAG_RC_FILE=rc_file, PYTHONPATH=os.pathsep.join(
                [os.path.dirname(os.path.dirname(os.path.abspath(__file__)))] +
                [x for x in os.environ.get("PYTHONPATH", "").split(os.pathsep) if x])))
        try:
            txt = open(rc_file).read().strip()
            os.remove(rc_file)
        except OSError:
            txt = ""
        return int(txt) if txt else (launcher or 255)
    quiet = int(os.environ.get("RANK", "0")) != 0
    if quiet:                               # ranks other than 0 compute but do not report
        sys.stdout = open(os.devnull, "w")
    rc = 0
    for f in files:
        if not f.endswith(".tla"):
            f += ".tla"
        print(f"Parsing file {os.path.abspath(f)}")
        if sim_num is not None:
            print(f"Running random simulation with seed {seed}.")
        try:
            r = check_file(f, deadlock=deadlock, cfg_path=cfg, device=dev, lib_dirs=libs, seq_cap=seq_cap,
                           engine=engine, max_depth=depth, simulate=None if sim_num is None else (sim_num, seed),
                           dump=dump)
        except (SpecError, ParseError, LexError, EvalError, CompileError, TypeErr) as ex:
            print(f"Error: {type(ex).__name__}: {ex}")
            r = 150
        except Exception as ex:  # noqa: BLE001 -- e.g. EngineUnavailable: no CUDA device (there is no CPU backend)
            print(f"Error: {type(ex).__name__}: {ex}")
            r = 255
        if r != 0:
            rc = r
            break      # `make` semantics: TLC exits non-zero at the first failing module
    if "RANK" in os.environ and os.environ.get("TLAG_RC_FILE"):
        try:
            import torch.distributed as dist
            if dist.is_initialized():
                dist.destroy_process_group()
        except Exception:  # noqa: BLE001
            pass
        if not quiet:
            with open(os.environ["TLAG_RC_FILE"], "w") as f:
                f.write(str(rc))
        return 0
    return rc


if __name__ == "__main__":
    sys.exit(tlc_main())
