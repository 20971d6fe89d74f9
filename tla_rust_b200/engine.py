"""ctypes binding of the C-ABI engine library (include/tlag.h, csrc/libtlag.so).

The product path has no CPU fallback: if the CUDA extension is missing or no GPU is
visible, construction fails loudly (EngineUnavailable)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("TLAG_LIB") or os.path.join(_HERE, "csrc", "libtlag.so")   # TLAG_LIB: tuning builds
_LIB = None
# target of every native build (csrc/Makefile: ARCH): H100, Hopper
NVCC_ARCH = ("-gencode", "arch=compute_90a,code=sm_90a")

F_DEADLOCK_CHECK = 1
F_KEEP_GOING = 2
F_EXACT = 4
V_OK, V_INVARIANT, V_ASSERT, V_DEADLOCK, V_EVAL_ERROR, V_RUNNING = 0, 1, 2, 3, 4, 5


class EngineUnavailable(RuntimeError):
    pass


class EngineError(RuntimeError):
    pass


class TlagModel(C.Structure):
    _fields_ = [("words_per_state", C.c_uint32), ("code", C.c_void_p), ("code_len", C.c_uint32),
                ("entry_inv", C.c_uint32), ("entry_next", C.c_uint32),
                ("cpool", C.c_void_p), ("cpool_len", C.c_uint32),
                ("layout", C.c_void_p), ("n_slots", C.c_uint32),
                ("frame_words", C.c_uint32), ("unpacked_words", C.c_uint32),
                ("n_invariants", C.c_uint32), ("n_actions", C.c_uint32),
                ("table_slots_log2", C.c_uint32), ("max_states", C.c_uint64),
                ("flags", C.c_uint32), ("device", C.c_int32)]


class WaveStats(C.Structure):
    _fields_ = [("level", C.c_uint64), ("expanded", C.c_uint64), ("generated", C.c_uint64),
                ("discovered", C.c_uint64), ("distinct_total", C.c_uint64), ("generated_total", C.c_uint64),
                ("kernel_ms", C.c_float), ("verdict", C.c_int32), ("cluster_ms", C.c_float),
                ("retries", C.c_uint32)]

    def as_dict(self):
        return {f: getattr(self, f) for f, _ in self._fields_}


class TlagResult(C.Structure):
    _fields_ = [("verdict", C.c_int32), ("detail", C.c_int32), ("detail2", C.c_int32), ("reserved", C.c_int32),
                ("state_idx", C.c_uint64), ("generated", C.c_uint64), ("distinct", C.c_uint64),
                ("queue_left", C.c_uint64), ("depth", C.c_uint64), ("init_states", C.c_uint64),
                ("fp_collision_estimate", C.c_double), ("device_seconds", C.c_double)]

    def as_dict(self):
        return {f: getattr(self, f) for f, _ in self._fields_}


class GraphInfo(C.Structure):
    _fields_ = [("n_states", C.c_uint64), ("n_expanded", C.c_uint64), ("n_edges", C.c_uint64), ("device_ms", C.c_float)]

    def as_dict(self):
        return {f: getattr(self, f) for f, _ in self._fields_}


class LabelProgram(C.Structure):
    _fields_ = [("code", C.c_void_p), ("code_len", C.c_uint32), ("entry_states", C.c_uint32), ("entry_edges", C.c_uint32),
                ("n_state_preds", C.c_uint32), ("n_edge_preds", C.c_uint32), ("cpool", C.c_void_p), ("cpool_len", C.c_uint32),
                ("en_bit", C.c_uint8 * 32), ("nen_bit", C.c_uint8 * 32)]


class GraphDev(C.Structure):
    _fields_ = [("n_states", C.c_uint64), ("n_edges", C.c_uint64), ("off", C.c_uint64), ("dst", C.c_uint64),
                ("state_label", C.c_uint64), ("edge_label", C.c_uint64), ("n_init", C.c_uint64), ("device", C.c_int32)]


class SimParams(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("first_walk", C.c_uint64), ("num_walks", C.c_uint64), ("depth", C.c_uint32),
                ("flags", C.c_uint32)]


class SimResult(C.Structure):
    _fields_ = [("verdict", C.c_int32), ("detail", C.c_int32), ("detail2", C.c_int32), ("reserved", C.c_int32),
                ("walk", C.c_uint64), ("step", C.c_uint64), ("checked", C.c_uint64), ("generated", C.c_uint64),
                ("behaviours", C.c_uint64), ("batch_walks", C.c_uint64), ("device_ms", C.c_double)]

    def as_dict(self):
        return {f: getattr(self, f) for f, _ in self._fields_}


EXPORTS = ["tlag_create", "tlag_seed", "tlag_step", "tlag_run", "tlag_result_now", "tlag_trace",
           "tlag_read_states", "tlag_digest", "tlag_probe_batch", "tlag_probe_batch_device", "tlag_reset_table", "tlag_restart",
           "tlag_kernel_launches", "tlag_destroy", "tlag_last_error", "tlag_version",
           "tlag_frontier", "tlag_expand_route", "tlag_insert_records", "tlag_advance_level",
           "tlag_p2p_init", "tlag_p2p_attach", "tlag_p2p_level", "tlag_p2p_rollback", "tlag_read_link", "tlag_set_rank", "tlag_set_owner_words",
           "tlag_simulate", "tlag_sim_trace", "tlag_sim_read", "tlag_sim_digest",
           "tlag_build_graph", "tlag_read_graph", "tlag_graph_digest", "tlag_label_graph", "tlag_graph_view"]


def build_library(verbose=False):
    """nvcc cross-compiles for sm_90a without a GPU."""
    subprocess.check_call(["make", "-C", os.path.join(_HERE, "csrc")] + ([] if verbose else ["-s"]))


def _bind(path):
    L = C.CDLL(path)
    L.tlag_last_error.restype = C.c_char_p
    L.tlag_version.restype = C.c_char_p
    L.tlag_kernel_launches.restype = C.c_uint64
    L.tlag_destroy.restype = None
    for fn in EXPORTS:
        getattr(L, fn)
    return L


def load_library():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise EngineUnavailable(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                                    f"(the product has no CPU fallback)")
        _LIB = _bind(LIB_PATH)
    return _LIB


NATIVE_DIR = os.path.join(_HERE, "csrc", "native")
_NATIVE_LIBS = {}


def _sliced_tag(cm, scalar, simulate=False):
    import hashlib
    from .compile.sliced import model_key
    h = hashlib.sha256()
    for rel in ("csrc/tlag_engine.cu", "csrc/tlag_dev.cuh", "csrc/tlag_dev2.cuh", "csrc/tlag_vm.h", "csrc/tlag_vm_exec.inc",
                "compile/sliced.py", "../include/tlag.h"):
        with open(os.path.join(_HERE, rel), "rb") as f:
            h.update(f.read())
    h.update(repr((getattr(cm, "segments", None), os.environ.get("TLAG_SL_OCC", ""), os.environ.get("TLAG_SL_BLOCK", ""),
                   os.environ.get("TLAG_SL_MIN_SLICE", ""))).encode())
    if os.environ.get("TLAG_CSRC_DIR"):                 # experiments built from a modified copy of csrc/
        h.update(os.environ["TLAG_CSRC_DIR"].encode())
    return f"sl_{model_key(cm)}_{h.hexdigest()[:8]}{'_s' if scalar else ''}{'_sim' if simulate else ''}"


def sliced_form(cm):
    """scalar form (frame words as C locals) when the model allows it, else the array form; TLAG_SL_FORM overrides."""
    from .compile.sliced import Emitter, SliceError
    want = os.environ.get("TLAG_SL_FORM", "auto")
    if want == "array":
        return False
    try:
        Emitter(cm, scalar=True)
        return True
    except SliceError:
        if want == "scalar":
            raise
        return False


def sliced_library_path(cm, scalar=None, simulate=False):
    if scalar is None:
        scalar = sliced_form(cm)
    return os.path.join(NATIVE_DIR, f"libtlag_{_sliced_tag(cm, scalar, simulate)}.so")


def build_sliced_library(cm, force=False, verbose=False, scalar=None, jobs=None, simulate=False):
    """Model-specialised engine library, sliced form (compile/sliced.py): one kernel per invariant and per disjunct of
    Next, same engine source and C ABI.  The slices are spread over several translation units that nvcc compiles in
    parallel (-dc) next to the engine's own unit; built in-tree (csrc/native/) so that it travels with the snapshot.
    simulate=True: the model's simulation library instead (tlag_simulate; the same slices compiled with -DTLAG_SL_SIM
    into the simulation kernels, no BFS), a library of its own."""
    from concurrent.futures import ThreadPoolExecutor
    from .compile.sliced import emit_parts
    if scalar is None:
        scalar = sliced_form(cm)
    os.makedirs(NATIVE_DIR, exist_ok=True)
    tag = _sliced_tag(cm, scalar, simulate)
    so = os.path.join(NATIVE_DIR, f"libtlag_{tag}.so")
    if os.path.exists(so) and not force:
        return so
    # translation units the program is split into; `jobs` (default: as many) only bounds the nvcc processes run at once
    max_parts = int(os.environ.get("TLAG_BUILD_JOBS", "0")) or min(8, os.cpu_count() or 1)
    jobs = jobs or max_parts
    work = os.path.join(NATIVE_DIR, tag)
    os.makedirs(work, exist_ok=True)
    defs_path = os.path.join(work, "defs.h")
    nparts = max(1, min(max_parts, 1 + len(cm.code) // 1500))
    ms = os.environ.get("TLAG_SL_MIN_SLICE")
    defs, parts = emit_parts(cm, scalar, nparts, defs_path, min_slice=int(ms) if ms else None)
    with open(defs_path, "w") as f:
        f.write(defs)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    csrc = os.environ.get("TLAG_CSRC_DIR") or os.path.join(_HERE, "csrc")      # (experiments: a modified copy of csrc/)
    base = [nvcc, "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", *NVCC_ARCH, "-I", csrc, "-dc"]
    if not scalar and cm.frame_words > 512:
        base.append("-DTLAG_SL_SEG_NOINLINE")
    if simulate:
        base.append("-DTLAG_SL_SIM")
    for k in ("TLAG_SL_OCC", "TLAG_SL_BLOCK"):
        if os.environ.get(k):
            base.append(f"-D{k}={int(os.environ[k])}")
    # subroutines are compiled apart from the kernels that call them (relocatable device code): give them the register
    # budget of the kernels' __launch_bounds__ (tlag_dev.cuh: 256 threads x 4 CTAs per SM by default)
    regcap = 65536 // (int(os.environ.get("TLAG_SL_BLOCK", "256")) * int(os.environ.get("TLAG_SL_OCC", "4")))
    base.append(f"-maxrregcount={min(255, regcap)}")
    units = []
    for k, text in enumerate(parts):
        src = os.path.join(work, f"part{k}.cu")
        with open(src, "w") as f:
            f.write(text)
        units.append((base + ["-o", src[:-3] + ".o", src], src[:-3] + ".o"))
    units.append((base + [f'-DTLAG_SLICED_INC="{defs_path}"', "-o", os.path.join(work, "engine.o"),
                          os.path.join(csrc, "tlag_engine.cu")], os.path.join(work, "engine.o")))

    def run(cmd):
        p = subprocess.run(cmd, capture_output=not verbose, text=True)
        if p.returncode != 0:
            raise EngineError(f"nvcc failed for the sliced build of model {tag}: {(p.stderr or '')[-3000:]}")
    with ThreadPoolExecutor(max_workers=jobs) as ex:
        list(ex.map(run, [u[0] for u in units]))
    run([nvcc, "-shared", *NVCC_ARCH, "-o", so + ".tmp"] + [u[1] for u in units])
    os.replace(so + ".tmp", so)
    if os.environ.get("TLAG_KEEP_BUILD") != "1":       # generated sources + objects (regenerated from the model at will)
        import shutil
        shutil.rmtree(work, ignore_errors=True)
    return so


def load_sliced_library(cm, build=True, simulate=False):
    if os.environ.get("TLAG_NO_BUILD") == "1":      # GPU sessions: never spend box time in nvcc
        build = False
    so = sliced_library_path(cm, simulate=simulate)
    if so not in _NATIVE_LIBS:
        if not os.path.exists(so):
            if not build:
                raise EngineUnavailable(f"{so} is missing (sliced native build of this model)")
            build_sliced_library(cm, simulate=simulate)
        _NATIVE_LIBS[so] = _bind(so)
    return _NATIVE_LIBS[so]


class Engine:
    """One BFS engine instance on one GPU (mirrors tlag_engine)."""

    def __init__(self, cm, deadlock=True, device=0, table_log2=0, max_states=0, keep_going=False, native=None, exact=False,
                 simulate=False):
        """native="sliced" (or True): the model-specialised sliced build -- one kernel per invariant / disjunct of Next,
        compile/sliced.py; built on demand with nvcc and cached in csrc/native/; False: the bytecode interpreter kernel;
        None: follow the environment variable TLAG_NATIVE (sliced / 0).
        simulate=True with the sliced build: the model's simulation library, which runs simulate() and no search (the
        interpreter library runs both)."""
        if native is None:
            native = "sliced" if os.environ.get("TLAG_NATIVE", "0") in ("sliced", "1") else False
        if exact:               # TLAG_F_EXACT: TLC's single worker replayed on the device (interpreter kernel, one warp)
            native = False
        self.native = "sliced" if native else False
        self.deadlock = deadlock
        self.L = load_sliced_library(cm, simulate=simulate) if self.native else load_library()
        self.cm = cm
        self._code = np.ascontiguousarray(cm.code, dtype=np.uint64)
        self._cpool = np.ascontiguousarray(cm.cpool, dtype=np.int32)
        self._layout = np.ascontiguousarray(cm.layout, dtype=np.int32)
        flags = (F_DEADLOCK_CHECK if deadlock else 0) | (F_KEEP_GOING if keep_going else 0) | (F_EXACT if exact else 0)
        m = TlagModel(cm.W, self._code.ctypes.data, len(self._code), cm.entries["inv"], cm.entries["next"],
                      self._cpool.ctypes.data, len(self._cpool), self._layout.ctypes.data, self._layout.shape[0],
                      cm.frame_words, cm.state_words_unpacked, len(cm.invariants), len(cm.actions),
                      table_log2, max_states, flags, device)
        self.h = C.c_void_p()
        rc = self.L.tlag_create(C.byref(m), C.byref(self.h))
        if rc != 0:
            msg = self.L.tlag_last_error(self.h).decode() if self.h else "tlag_create failed"
            if self.h:
                self.L.tlag_destroy(self.h)
                self.h = None
            if rc == -3:
                raise EngineUnavailable(f"CUDA engine unavailable: {msg}")
            raise EngineError(f"tlag_create: {msg}")

    def _ck(self, rc, what):
        if rc != 0:
            raise EngineError(f"{what}: rc={rc}: {self.L.tlag_last_error(self.h).decode()}")

    def close(self):
        if getattr(self, "h", None):
            self.L.tlag_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def seed(self, init_words: np.ndarray):
        a = np.ascontiguousarray(init_words, dtype=np.uint32).reshape(-1, self.cm.W)
        self._ck(self.L.tlag_seed(self.h, a.ctypes.data_as(C.c_void_p), C.c_uint64(a.shape[0])), "tlag_seed")

    def step(self) -> dict:
        ws = WaveStats()
        self._ck(self.L.tlag_step(self.h, C.byref(ws)), "tlag_step")
        return ws.as_dict()

    def run(self) -> dict:
        r = TlagResult()
        self._ck(self.L.tlag_run(self.h, C.byref(r)), "tlag_run")
        return r.as_dict()

    def result(self) -> dict:
        r = TlagResult()
        self._ck(self.L.tlag_result_now(self.h, C.byref(r)), "tlag_result_now")
        return r.as_dict()

    def trace(self, state_idx: int, cap=4096):
        W = self.cm.W
        states = np.zeros((cap, W), dtype=np.uint32)
        acts = np.zeros(cap, dtype=np.int32)
        n = C.c_uint32(cap)
        self._ck(self.L.tlag_trace(self.h, C.c_uint64(state_idx), states.ctypes.data_as(C.c_void_p),
                                   acts.ctypes.data_as(C.c_void_p), C.byref(n)), "tlag_trace")
        return states[:n.value].copy(), acts[:n.value].copy()

    def read_states(self, first: int, n: int) -> np.ndarray:
        out = np.zeros((n, self.cm.W), dtype=np.uint32)
        self._ck(self.L.tlag_read_states(self.h, C.c_uint64(first), C.c_uint64(n), out.ctypes.data_as(C.c_void_p)),
                 "tlag_read_states")
        return out

    def read_link(self, idx: int):
        """-> (state words, parent index or -1 for an initial state, action id, rank holding the parent)"""
        st = np.zeros(self.cm.W, dtype=np.uint32)
        par, meta = C.c_uint32(), C.c_uint32()
        self._ck(self.L.tlag_read_link(self.h, C.c_uint64(idx), st.ctypes.data_as(C.c_void_p), C.byref(par), C.byref(meta)),
                 "tlag_read_link")
        root = par.value == 0xFFFFFFFF
        return st, (-1 if root else par.value), (-1 if root else meta.value >> 8), meta.value & 0xFF

    def digest(self):
        x, s_ = C.c_uint64(), C.c_uint64()
        self._ck(self.L.tlag_digest(self.h, C.byref(x), C.byref(s_)), "tlag_digest")
        return int(x.value), int(s_.value)

    def probe_batch(self, states: np.ndarray) -> np.ndarray:
        a = np.ascontiguousarray(states, dtype=np.uint32).reshape(-1, self.cm.W)
        flags = np.zeros(a.shape[0], dtype=np.uint8)
        self._ck(self.L.tlag_probe_batch(self.h, a.ctypes.data_as(C.c_void_p), C.c_uint64(a.shape[0]),
                                         flags.ctypes.data_as(C.c_void_p)), "tlag_probe_batch")
        return flags

    def probe_batch_device(self, d_states_ptr: int, n: int, d_flags_ptr: int) -> float:
        ms = C.c_float()
        self._ck(self.L.tlag_probe_batch_device(self.h, C.c_uint64(d_states_ptr), C.c_uint64(n),
                                                C.c_uint64(d_flags_ptr), C.byref(ms)), "tlag_probe_batch_device")
        return ms.value

    def reset_table(self):
        self._ck(self.L.tlag_reset_table(self.h), "tlag_reset_table")

    def restart(self):
        self._ck(self.L.tlag_restart(self.h), "tlag_restart")

    def launches(self) -> int:
        return int(self.L.tlag_kernel_launches(self.h))

    # random simulation (include/tlag.h: tlag_simulate)
    def simulate(self, seed, num, depth, first=0) -> dict:
        """`num` random behaviours of at most `depth` states, walks first..first + num - 1 of the run with this seed
        (deadlocks checked as the engine was created).  -> dict(verdict, detail, detail2, walk, step, checked,
        generated, behaviours, batch_walks, device_ms)"""
        r = SimResult()
        self._sim_depth = depth
        sp = SimParams(seed & 0xFFFFFFFFFFFFFFFF, first, num, depth, F_DEADLOCK_CHECK if self.deadlock else 0)
        self._ck(self.L.tlag_simulate(self.h, C.byref(sp), C.byref(r)), "tlag_simulate")
        return r.as_dict()

    def sim_trace(self, walk, cap=1 << 20):
        """-> (states, action ids) of a walk of the last batch, as trace() returns them"""
        W = self.cm.W
        n = C.c_uint32(cap)
        self._ck(self.L.tlag_sim_trace(self.h, C.c_uint64(walk), None, None, C.byref(n)), "tlag_sim_trace")
        states = np.zeros((n.value, W), dtype=np.uint32)
        acts = np.zeros(n.value, dtype=np.int32)
        self._ck(self.L.tlag_sim_trace(self.h, C.c_uint64(walk), states.ctypes.data_as(C.c_void_p),
                                       acts.ctypes.data_as(C.c_void_p), C.byref(n)), "tlag_sim_trace")
        return states, acts

    def sim_read(self, walk, n):
        """History of walks [walk, walk + n) of the last batch: (states [depth, n, W], action ids [depth, n], lengths [n])"""
        L, W = self.L, self.cm.W
        lens = np.zeros(n, dtype=np.uint32)
        self._ck(L.tlag_sim_read(self.h, C.c_uint64(walk), C.c_uint64(n), None, None, lens.ctypes.data_as(C.c_void_p)),
                 "tlag_sim_read")
        depth = self._sim_depth
        states = np.zeros((depth, n, W), dtype=np.uint32)
        acts = np.zeros((depth, n), dtype=np.int16)
        self._ck(L.tlag_sim_read(self.h, C.c_uint64(walk), C.c_uint64(n), states.ctypes.data_as(C.c_void_p),
                                 acts.ctypes.data_as(C.c_void_p), None), "tlag_sim_read")
        return states, acts, lens

    def sim_digest(self):
        x, s_ = C.c_uint64(), C.c_uint64()
        self._ck(self.L.tlag_sim_digest(self.h, C.byref(x), C.byref(s_)), "tlag_sim_digest")
        return int(x.value), int(s_.value)

    # state graph (include/tlag.h: tlag_build_graph)
    def build_graph(self) -> dict:
        """The state graph of the store, built in device memory.  -> dict(n_states, n_expanded, n_edges, device_ms)"""
        gi = GraphInfo()
        self._ck(self.L.tlag_build_graph(self.h, C.byref(gi)), "tlag_build_graph")
        self._graph_states = gi.n_states
        return gi.as_dict()

    def state_graph(self, first=0, n=None):
        """Edges out of rows [first, first + n) (default: to the last row) -> (off [n + 1] uint64 relative to row
        `first`, dst [off[n]] uint32 rows, act [off[n]] int32 action ids)"""
        if n is None:
            n = getattr(self, "_graph_states", 0) - first
        off = np.zeros(n + 1, dtype=np.uint64)
        self._ck(self.L.tlag_read_graph(self.h, C.c_uint64(first), C.c_uint64(n), off.ctypes.data_as(C.c_void_p), None, None),
                 "tlag_read_graph")
        dst = np.zeros(int(off[-1]), dtype=np.uint32)
        act = np.zeros(int(off[-1]), dtype=np.int32)
        self._ck(self.L.tlag_read_graph(self.h, C.c_uint64(first), C.c_uint64(n), off.ctypes.data_as(C.c_void_p),
                                        dst.ctypes.data_as(C.c_void_p), act.ctypes.data_as(C.c_void_p)), "tlag_read_graph")
        return off, dst, act

    def label_graph(self, img, en=None, nen=None) -> float:
        """Label the state graph with a label image (compile/lower.py compile_labels).  en / nen: {edge bit: state bit} of
        the ENABLED bits and their complements derived from the edge labels.  -> device ms"""
        code = np.ascontiguousarray(img.code, dtype=np.uint64)
        cpool = np.ascontiguousarray(img.cpool if len(img.cpool) else [0], dtype=np.int32)
        eb, nb = (C.c_uint8 * 32)(*([0xFF] * 32)), (C.c_uint8 * 32)(*([0xFF] * 32))
        for b, sb in (en or {}).items():
            eb[b] = sb
        for b, sb in (nen or {}).items():
            nb[b] = sb
        lp = LabelProgram(code.ctypes.data, len(code), img.entries["states"], img.entries["edges"], img.n_states,
                          img.n_edges, cpool.ctypes.data, len(img.cpool), eb, nb)
        ms = C.c_float()
        self._ck(self.L.tlag_label_graph(self.h, C.byref(lp), C.byref(ms)), "tlag_label_graph")
        return float(ms.value)

    def graph_view(self) -> GraphDev:
        """The state graph and its labels as device pointers (include/tlag.h: tlag_graph_view)"""
        v = GraphDev()
        self._ck(self.L.tlag_graph_view(self.h, C.byref(v)), "tlag_graph_view")
        return v

    def graph_digest(self):
        x, s_ = C.c_uint64(), C.c_uint64()
        self._ck(self.L.tlag_graph_digest(self.h, C.byref(x), C.byref(s_)), "tlag_graph_digest")
        return int(x.value), int(s_.value)

    # multi-GPU building blocks
    def frontier(self):
        a, b = C.c_uint64(), C.c_uint64()
        self._ck(self.L.tlag_frontier(self.h, C.byref(a), C.byref(b)), "tlag_frontier")
        return int(a.value), int(b.value)

    def set_owner_words(self, k):
        self._ck(self.L.tlag_set_owner_words(self.h, C.c_uint32(k)), "tlag_set_owner_words")

    def set_rank(self, n_ranks, rank):
        self._ck(self.L.tlag_set_rank(self.h, C.c_uint32(n_ranks), C.c_uint32(rank)), "tlag_set_rank")

    def expand_route(self, n_ranks, first, count, d_send_ptr, cap_records):
        counts = (C.c_uint64 * n_ranks)()
        ws = WaveStats()
        self._ck(self.L.tlag_expand_route(self.h, C.c_uint32(n_ranks), C.c_uint64(first), C.c_uint64(count),
                                          C.c_uint64(d_send_ptr), C.c_uint64(cap_records), counts, C.byref(ws)),
                 "tlag_expand_route")
        return [int(c) for c in counts], ws.as_dict()

    def insert_records(self, d_recv_ptr, n_records) -> int:
        nn = C.c_uint64()
        self._ck(self.L.tlag_insert_records(self.h, C.c_uint64(d_recv_ptr), C.c_uint64(n_records), C.c_uint32(0),
                                            C.byref(nn)), "tlag_insert_records")
        return int(nn.value)

    # peer-memory exchange (include/tlag.h: tlag_p2p_*)
    def p2p_init(self, n_ranks, rank, cap_records) -> bytes:
        h = (C.c_uint8 * 64)()
        self._ck(self.L.tlag_p2p_init(self.h, C.c_uint32(n_ranks), C.c_uint32(rank), C.c_uint64(cap_records), h), "tlag_p2p_init")
        return bytes(h)

    def p2p_attach(self, peer, handle: bytes):
        h = (C.c_uint8 * 64).from_buffer_copy(handle)
        self._ck(self.L.tlag_p2p_attach(self.h, C.c_uint32(peer), h), "tlag_p2p_attach")

    def p2p_level(self, n_chunks, chunk_states, expect_inbound=0):
        """-> wave stats dict, or None when one of this rank's send regions overflowed (see p2p_rollback)"""
        ws = WaveStats()
        rc = self.L.tlag_p2p_level(self.h, C.c_uint64(n_chunks), C.c_uint64(chunk_states), C.c_uint64(expect_inbound),
                                   C.byref(ws))
        if rc == -5:            # TLAG_EOVERFLOW
            return None
        self._ck(rc, "tlag_p2p_level")
        return ws.as_dict()

    def p2p_rollback(self):
        self._ck(self.L.tlag_p2p_rollback(self.h), "tlag_p2p_rollback")

    def advance_level(self) -> dict:
        ws = WaveStats()
        self._ck(self.L.tlag_advance_level(self.h, C.byref(ws)), "tlag_advance_level")
        return ws.as_dict()


# ---- liveness building blocks on a caller-provided state graph (include/tlag.h: tlag_scc, tlag_fair_cycles)
NO_SCC = 0xFFFFFFFF             # scc id of a state outside the mask / outside every accepted SCC
FAIR_KINDS = {"WF": 0, "SF": 1}


class TlagGraph(C.Structure):
    _fields_ = [("n_states", C.c_uint64), ("n_edges", C.c_uint64), ("src", C.c_void_p), ("dst", C.c_void_p),
                ("edge_label", C.c_void_p), ("state_label", C.c_void_p), ("state_mask", C.c_void_p),
                ("edge_mask", C.c_void_p), ("device", C.c_int32)]


class TlagFairness(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("enabled_bit", C.c_uint32), ("action_bit", C.c_uint32), ("reserved", C.c_uint32)]


class TlagFairQuery(C.Structure):
    _fields_ = [("fair", C.c_void_p), ("n_fair", C.c_uint32), ("need_clear", C.c_uint32), ("seeds", C.c_void_p)]


class TlagFairResult(C.Structure):
    _fields_ = [("violated", C.c_int32), ("witness", C.c_uint32), ("fair_sccs", C.c_uint64), ("rounds", C.c_uint32),
                ("device_ms", C.c_float)]


def _graph_lib():
    L = load_library()
    if not hasattr(L, "_graph_bound"):
        L.tlag_graph_last_error.restype = C.c_char_p
        L._graph_bound = True
    return L


def _graph_call(L, rc, what):
    if rc != 0:
        raise EngineError(f"{what}: rc={rc}: {L.tlag_graph_last_error().decode()}")


def _graph_struct(n_states, src, dst, edge_label, state_label, state_mask, edge_mask, device):
    """-> (tlag_graph, arrays it points into: keep them alive for the call)"""
    src = np.ascontiguousarray(src, dtype=np.uint32)
    dst = np.ascontiguousarray(dst, dtype=np.uint32)
    if src.shape != dst.shape or src.ndim != 1:
        raise ValueError("src and dst must be 1-D arrays of one length")
    if src.size and max(int(src.max()), int(dst.max())) >= n_states:
        raise ValueError("edge endpoint >= n_states")
    keep = [src, dst]

    def arr(a, dtype, size, what):
        if a is None:
            return None
        a = np.ascontiguousarray(a, dtype=dtype)
        if a.shape != (size,):
            raise ValueError(f"{what} must have shape ({size},)")
        keep.append(a)
        return a.ctypes.data

    g = TlagGraph(n_states, src.size, src.ctypes.data, dst.ctypes.data,
                  arr(edge_label, np.uint32, src.size, "edge_label"), arr(state_label, np.uint32, n_states, "state_label"),
                  arr(state_mask, np.uint8, n_states, "state_mask"), arr(edge_mask, np.uint8, src.size, "edge_mask"), device)
    return g, keep


def scc(n_states, src, dst, state_mask=None, edge_mask=None, device=0):
    """SCC decomposition on the GPU of the graph restricted to the masks (self-loops ignored).
    -> (component id per state, NO_SCC outside the mask; number of components; device ms)"""
    L = _graph_lib()
    g, keep = _graph_struct(n_states, src, dst, None, None, state_mask, edge_mask, device)
    out = np.empty(n_states, dtype=np.uint32)
    n, ms = C.c_uint64(), C.c_float()
    _graph_call(L, L.tlag_scc(C.byref(g), out.ctypes.data_as(C.c_void_p), C.byref(n), C.byref(ms)), "tlag_scc")
    return out, int(n.value), float(ms.value)


def fair_cycles(n_states, src, dst, edge_label=None, state_label=None, state_mask=None, edge_mask=None, fairness=(),
                need_clear=0, seeds=None, device=0):
    """Fair-cycle search (Emerson-Lei) on the GPU; see tlag_fair_cycles in include/tlag.h.
    fairness: (kind "WF"/"SF", ENABLED bit of state_label, action bit of edge_label) triples.
    -> dict(violated, witness, fair_sccs, rounds, device_ms, scc = accepted SCC id per state or NO_SCC)"""
    L = _graph_lib()
    g, keep = _graph_struct(n_states, src, dst, edge_label, state_label, state_mask, edge_mask, device)
    fair = (TlagFairness * max(1, len(fairness)))(*[TlagFairness(FAIR_KINDS[k], en, act, 0) for k, en, act in fairness])
    sd = None
    if seeds is not None:
        sd = np.ascontiguousarray(seeds, dtype=np.uint8)
        if sd.shape != (n_states,):
            raise ValueError(f"seeds must have shape ({n_states},)")
    q = TlagFairQuery(C.addressof(fair), len(fairness), need_clear, None if sd is None else sd.ctypes.data)
    out = np.empty(n_states, dtype=np.uint32)
    r = TlagFairResult()
    _graph_call(L, L.tlag_fair_cycles(C.byref(g), C.byref(q), out.ctypes.data_as(C.c_void_p), C.byref(r)),
                "tlag_fair_cycles")
    return {"violated": bool(r.violated), "witness": None if r.witness == NO_SCC else int(r.witness),
            "fair_sccs": int(r.fair_sccs), "rounds": int(r.rounds), "device_ms": float(r.device_ms), "scc": out}


class TlagLiveQuery(C.Structure):
    _fields_ = [("fair", C.c_void_p), ("n_fair", C.c_uint32), ("flags", C.c_uint32), ("keep_set", C.c_uint32),
                ("keep_clear", C.c_uint32), ("edge_drop", C.c_uint32), ("need_clear", C.c_uint32), ("seed_set", C.c_uint32),
                ("seed_clear", C.c_uint32), ("seed_rows", C.c_uint64)]


class TlagLiveResult(C.Structure):
    _fields_ = [("violated", C.c_int32), ("witness", C.c_uint32), ("fair_sccs", C.c_uint64), ("rounds", C.c_uint32),
                ("prefix_len", C.c_uint32), ("cycle_len", C.c_uint32), ("reserved", C.c_uint32), ("check_ms", C.c_float),
                ("lasso_ms", C.c_float)]


LIVE_SEEDS, LIVE_ANY_SEED = 1, 2


def live_check(view, fairness=(), keep_set=0, keep_clear=0, edge_drop=0, need_clear=0, seed_set=0, seed_clear=0,
               seed_rows=0, flags=0, lasso_cap=1 << 16):
    """Obligation check on an engine's labelled graph (include/tlag.h: tlag_live_check).  view: Engine.graph_view();
    fairness: (kind "WF"/"SF", ENABLED state bit, action edge bit) triples.
    -> dict(violated, witness, fair_sccs, rounds, check_ms, lasso_ms, prefix [rows], cycle [rows])"""
    L = _graph_lib()
    fair = (TlagFairness * max(1, len(fairness)))(*[TlagFairness(FAIR_KINDS[k], en, act, 0) for k, en, act in fairness])
    q = TlagLiveQuery(C.addressof(fair), len(fairness), flags, keep_set, keep_clear, edge_drop, need_clear, seed_set,
                      seed_clear, seed_rows)
    while True:
        lasso = np.zeros(lasso_cap, dtype=np.uint32)
        r = TlagLiveResult()
        rc = L.tlag_live_check(C.byref(view), C.byref(q), lasso.ctypes.data_as(C.c_void_p), C.c_uint32(lasso_cap),
                               C.byref(r))
        if rc == -5 and r.prefix_len + r.cycle_len > lasso_cap:     # TLAG_EOVERFLOW: the lasso's length is set
            lasso_cap = int(r.prefix_len + r.cycle_len)
            continue
        _graph_call(L, rc, "tlag_live_check")
        break
    p, c = int(r.prefix_len), int(r.cycle_len)
    return {"violated": bool(r.violated), "witness": None if r.witness == NO_SCC else int(r.witness),
            "fair_sccs": int(r.fair_sccs), "rounds": int(r.rounds), "check_ms": float(r.check_ms),
            "lasso_ms": float(r.lasso_ms), "prefix": lasso[:p].tolist(), "cycle": lasso[p:p + c].tolist()}


class ProbeOnlyModel:
    """Minimal stand-in CompiledModel for K1-only use (tlag_probe_batch on W-word states)."""

    def __init__(self, W):
        self.W = W
        self.code = np.zeros(2, dtype=np.uint64)  # HALT, HALT
        self.cpool = np.zeros(1, dtype=np.int32)
        self.layout = np.array([[i, 32, 0] for i in range(W)], dtype=np.int32)
        self.entries = {"inv": 0, "next": 1}
        self.frame_words = 2 * W + 4
        self.state_words_unpacked = W
        self.invariants = []
        self.actions = []
