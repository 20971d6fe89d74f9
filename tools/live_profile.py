"""Time the device liveness building blocks (tlag_scc, tlag_fair_cycles) on a generated state graph.

The graph is the state graph of K counters modulo B, one action per counter ("A_k: c_k' = (c_k + 1) % B"): B^K states,
K * B^K edges, one strongly connected component.  Each action is always enabled and labels its edges with bit k.
The queries are the ones a liveness check of this model under WF_c(A_k) for every k would ask:
  scc        the decomposition of the whole graph;
  holds      []<>(c_0 = 0): the graph restricted to c_0 # 0 has no fair SCC (A_0 leaves every component);
  fails      []<>(c_0 = 0) without fairness on A_0: every restricted component is fair (a violation);
  sf_split   SF on an action enabled only where c_1 = 0 and never taken: Emerson-Lei drops those states and splits.
That graph is shallow (forward diameter K * (B - 1)) and has one SCC, the best case for the decomposition.  The deep
case is a chain of --depth SCCs of 3 states each ("deep"; the states numbered at random), the case where every search
takes about one pass per SCC along the chain and colouring needs many rounds: timed for the decomposition and for a
fair-cycle query (WF on the in-cycle action: every SCC is fair).
Prints one JSON line with the device times (CUDA events, median of --repeat runs) and the GPU they were taken on.

    python tools/live_profile.py --counters 7 --modulus 10 --depth 10000 --repeat 3
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tla_rust_b200 import engine  # noqa: E402


def counters_graph(K, B):
    n = B ** K
    v = np.arange(n, dtype=np.int64)
    src, dst, lab = [], [], []
    for k in range(K):
        step = B ** k
        ck = (v // step) % B
        src.append(v)
        dst.append(v + np.where(ck == B - 1, -(B - 1) * step, step))
        lab.append(np.full(n, 1 << k, np.uint32))
    c0 = v % B
    c1 = (v // B) % B if K > 1 else np.zeros(n, np.int64)
    return (n, np.concatenate(src).astype(np.uint32), np.concatenate(dst).astype(np.uint32), np.concatenate(lab),
            c0, c1)


def chain_graph(L, seed=1):
    """L SCCs {3i, 3i+1, 3i+2} (a 3-cycle, edge label bit 0), SCC i -> SCC i+1 (label bit 1); states renumbered at random"""
    n = 3 * L
    base = 3 * np.arange(L, dtype=np.int64)
    src = np.concatenate([base, base + 1, base + 2, base[:-1] + 2])
    dst = np.concatenate([base + 1, base + 2, base, base[1:]])
    lab = np.concatenate([np.ones(3 * L, np.uint32), np.full(L - 1, 2, np.uint32)])
    perm = np.random.default_rng(seed).permutation(n)
    return n, perm[src].astype(np.uint32), perm[dst].astype(np.uint32), lab


def timed(runs, fn):
    """-> (median device ms, median call s, last result) over runs after one warm-up run"""
    res = []
    for _ in range(runs + 1):
        t = time.perf_counter()
        r = fn()
        res.append((r[-1] if isinstance(r, tuple) else r["device_ms"], time.perf_counter() - t, r))
    return float(np.median([x[0] for x in res[1:]])), float(np.median([x[1] for x in res[1:]])), res[-1][2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--counters", type=int, default=7)
    ap.add_argument("--modulus", type=int, default=10)
    ap.add_argument("--depth", type=int, default=10000)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    K, B = a.counters, a.modulus
    n, src, dst, elab, c0, c1 = counters_graph(K, B)
    all_en = np.full(n, (1 << K) - 1, np.uint32)
    wf_all = [("WF", k, k) for k in range(K)]
    not_c0 = (c0 != 0).astype(np.uint8)
    # SF on a "never taken" action (edge bit K, on no edge) enabled where c_1 = 0 (state bit K)
    sf_lab = all_en | np.where(c1 == 0, 1 << K, 0).astype(np.uint32)
    queries = {
        "holds": dict(state_label=all_en, state_mask=not_c0, fairness=wf_all),
        "fails": dict(state_label=all_en, state_mask=not_c0, fairness=wf_all[1:]),
        "sf_split": dict(state_label=sf_lab, fairness=[("SF", K, K)]),
    }
    expect = {"holds": False, "fails": True, "sf_split": True}
    out = {"graph": f"{K} counters mod {B}", "states": n, "edges": int(src.size)}
    times = []
    for _ in range(a.repeat + 1):          # the first run warms up module loading and allocations
        t = time.perf_counter()
        ids, k, ms = engine.scc(n, src, dst, device=a.device)
        times.append((ms, time.perf_counter() - t))
    assert k == 1, k
    out["scc_ms"] = float(np.median([t[0] for t in times[1:]]))
    out["scc_call_s"] = float(np.median([t[1] for t in times[1:]]))
    for name, q in queries.items():
        runs = []
        for _ in range(a.repeat + 1):
            t = time.perf_counter()
            r = engine.fair_cycles(n, src, dst, edge_label=elab, device=a.device, **q)
            runs.append((r["device_ms"], time.perf_counter() - t, r))
        r = runs[-1][2]
        assert r["violated"] == expect[name], (name, r["violated"])
        out[name] = {"device_ms": float(np.median([t[0] for t in runs[1:]])),
                     "call_s": float(np.median([t[1] for t in runs[1:]])),
                     "violated": r["violated"], "fair_sccs": r["fair_sccs"], "rounds": r["rounds"]}
    if a.depth > 1:
        L = a.depth
        dn, dsrc, ddst, dlab = chain_graph(L)
        ms, call_s, (ids, k, _) = timed(a.repeat, lambda: engine.scc(dn, dsrc, ddst, device=a.device))
        assert k == L, k
        out["deep"] = {"sccs": L, "states": dn, "edges": int(dsrc.size), "scc_ms": ms, "scc_call_s": call_s}
        ms, call_s, r = timed(a.repeat, lambda: engine.fair_cycles(
            dn, dsrc, ddst, edge_label=dlab, state_label=np.full(dn, 1, np.uint32), fairness=[("WF", 0, 0)],
            device=a.device))
        assert r["violated"] and r["fair_sccs"] == L, r["fair_sccs"]
        out["deep"].update({"fair_ms": ms, "fair_call_s": call_s})
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        out["gpu"] = q.stdout.strip().splitlines()[a.device] if q.returncode == 0 else "unknown"
    except (OSError, subprocess.SubprocessError, IndexError):
        out["gpu"] = "unknown"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
