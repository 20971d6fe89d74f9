"""Cost of the state graph pass (tlag_build_graph) on the device: for each model (compiled fixtures) and both engines, a
search to the fixpoint, one warm-up build, one timed build and one build under torch.profiler.  Prints per run the
graph's size, the build's device time and edges per second, the device time of the index pass, of the edge kernel and
of the sort / dedup / append (kernels by name, from the profiled build), and the high-water mark of the device memory
pool during the timed build (store and seen-set included), with the card's name and power limit read in the same
process.

    python tools/graph_profile.py [--models MCPaxos3_b4,MCraft_t4l3] [--engines interp,sliced]
"""
import argparse
import ctypes as C
import glob
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def _cudart():
    import torch
    cands = glob.glob(os.path.join(os.path.dirname(torch.__file__), "..", "nvidia", "cuda_runtime", "lib", "libcudart.so*"))
    cands += glob.glob("/usr/local/cuda/lib64/libcudart.so*")
    return C.CDLL(cands[0])


class PoolHigh:
    """High-water mark of the device's default memory pool (cudaMemPoolAttrUsedMemHigh), where the engine allocates"""
    USED_CURRENT, USED_HIGH = 7, 8

    def __init__(self, device=0):
        self.rt = _cudart()
        self.pool = C.c_void_p()
        assert self.rt.cudaDeviceGetDefaultMemPool(C.byref(self.pool), device) == 0

    def _get(self, attr):
        v = C.c_uint64()
        assert self.rt.cudaMemPoolGetAttribute(self.pool, attr, C.byref(v)) == 0
        return v.value

    def reset(self):
        z = C.c_uint64(0)
        assert self.rt.cudaMemPoolSetAttribute(self.pool, self.USED_HIGH, C.byref(z)) == 0
        return self._get(self.USED_CURRENT)

    def high(self):
        return self._get(self.USED_HIGH)


def kernel_ms(prof):
    """device ms of the profiled build: index pass, edge kernel, the rest (sort, dedup, offsets, append, copies)"""
    out = {"index_ms": 0.0, "edge_kernel_ms": 0.0, "sort_append_ms": 0.0}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if not t or ev.key.startswith(("ProfilerStep", "cuda", "aten")):
            continue
        if "k_graph_index" in ev.key:
            out["index_ms"] += t / 1e3
        elif "k_graph<" in ev.key:
            out["edge_kernel_ms"] += t / 1e3
        elif "k_graph_digest" not in ev.key:
            out["sort_append_ms"] += t / 1e3
    return {k: round(v, 3) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="MCPaxos3_b4,MCraft_t4l3")
    ap.add_argument("--engines", default="interp,sliced")
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from tla_rust_b200.compiled import load_compiled
    from tla_rust_b200.engine import Engine
    torch.zeros(1, device="cuda")
    pool = PoolHigh()
    print(f"card: {card()}", flush=True)
    for name in a.models.split(","):
        cm, init, _exp, info = load_compiled(os.path.join(ROOT, "tests", "golden", name + ".tlagz"))
        for eng in a.engines.split(","):
            e = Engine(cm, deadlock=info["deadlock"], native="sliced" if eng == "sliced" else False)
            e.seed(init)
            r = e.run()
            e.build_graph()                                  # warm-up: modules loaded, pool grown
            before = pool.reset()
            g = e.build_graph()
            peak = pool.high()
            dig = e.graph_digest()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                e.build_graph()
            out = dict(model=name, engine=eng, W=cm.W, verdict=r["verdict"], n_states=g["n_states"],
                       n_expanded=g["n_expanded"], n_edges=g["n_edges"], generated=r["generated"],
                       device_ms=round(g["device_ms"], 3),
                       edges_per_s=round(g["n_edges"] / (g["device_ms"] * 1e-3)) if g["device_ms"] else None,
                       pool_before_gib=round(before / 2 ** 30, 3), pool_peak_gib=round(peak / 2 ** 30, 3),
                       digest=[hex(dig[0]), hex(dig[1])], **kernel_ms(prof))
            print(json.dumps(out), flush=True)
            e.close()
    print(f"card: {card()}", flush=True)


if __name__ == "__main__":
    main()
