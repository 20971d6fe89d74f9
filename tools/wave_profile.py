"""Where a BFS job's time goes, level by level, on the sliced native kernels: one fixture (tests/golden/*.tlagz) run
with tlag_step, after `--warmup` untimed runs of the same job on the same engine.  Prints ONE JSON line: per level the
states expanded, successors generated, states discovered, the wave kernels' time (CUDA events around the level's
invariant, Next and deadlock kernels) and the time of the frontier clustering pass that reorders the level's new states
(`cluster_ms`, with the bytes a reorder cannot avoid -- every record of W words + parent + meta read once and written
once -- and the rate that gives), the level's reruns after a store overflow (`retries`), the job's wall time, whether
the counts and the digest match the oracle's record, the TLAG_SL_* switches in effect, and the GPU's name, power limit
and maximum SM clock.  With --kernels the timed job runs under torch.profiler instead, and the line gets the device
time of every kernel over the job (`kernels`, ms by name); its wall time then includes the tracing.

    python tools/wave_profile.py [MCPaxos3_b4] [--warmup 1] [--max-levels L] [--kernels]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tla_rust_b200.compiled import load_compiled  # noqa: E402
from tla_rust_b200.engine import V_RUNNING, Engine  # noqa: E402


def gpu_info(dev):
    """name, power limit and maximum SM clock of device `dev` (a query only)"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(dev)], capture_output=True, text=True, timeout=20).stdout.strip()
        name, power, clock = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as ex:  # noqa: BLE001
        return {"error": str(ex)[:200]}


def switches():
    """the TLAG_SL_* settings in effect: the run-time switch with its default when unset, and any build knob that is set"""
    out = {k: os.environ[k] for k in sorted(os.environ) if k.startswith("TLAG_SL_")}
    v = os.environ.get("TLAG_SL_SKIPSELF", "")
    lead = re.match(r"\s*[+-]?\d+", v)            # as tlag_create reads it: unset or empty = on, else atoi() != 0
    out["TLAG_SL_SKIPSELF"] = "1" if not v or (lead and int(lead.group()) != 0) else "0"
    v = os.environ.get("TLAG_SL_STAGE", "")        # unset or empty = every compiled staging slot, else max(0, atoi())
    lead = re.match(r"\s*[+-]?\d+", v)
    out["TLAG_SL_STAGE"] = "all" if not v else str(max(0, int(lead.group())) if lead else 0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("fixture", nargs="?", default="MCPaxos3_b4")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--max-levels", type=int, default=0, help="stop after this many levels (default: the fixture's bound)")
    ap.add_argument("--kernels", action="store_true", help="per-kernel device times of the timed job (torch.profiler)")
    args = ap.parse_args()
    if args.max_levels < 0:
        ap.error("--max-levels must be at least 1 (0: the fixture's bound)")
    cm, init, exp, info = load_compiled(os.path.join(ROOT, "tests", "golden", args.fixture + ".tlagz"))
    o2 = exp["o2"]
    ml = args.max_levels or o2.get("max_levels", 0)
    if ml > len(o2.get("level_digests") or []):
        ap.error(f"--max-levels {ml}: the oracle's record of {args.fixture} has no per-level digests that deep "
                 f"({len(o2.get('level_digests') or [])} levels)")
    if ml:          # depth-bounded prefix: the oracle's cumulative record after level `ml`
        x, sm, gen = o2["level_digests"][ml - 1]
        o2 = dict(o2, generated=gen, distinct=sum(o2["levels"][:ml]), depth=ml, fp_xor=x, fp_sum=sm)
    e = Engine(cm, deadlock=info["deadlock"], native="sliced")
    e.seed(init)

    def job(record):
        levels = []
        lv = 1
        while not ml or lv < ml:
            ws = e.step()
            lv += 1
            if ws["expanded"]:
                # levels the pass sorts (an unclustered level is copied in discovery order, or appended to the store
                # when no discovery buffer fitted: not counted as a reorder)
                sorted_ = (ws["cluster_ms"] > 0 and ws["discovered"] >= 8192 and ws["verdict"] == V_RUNNING
                           and not os.environ.get("TLAG_NO_SORT"))
                reorder = 2 * (cm.W + 2) * 4 * ws["discovered"] if sorted_ else 0
                levels.append({k: ws[k] for k in ("level", "expanded", "generated", "discovered")}
                              | {"retries": ws["retries"],
                                 "kernel_ms": round(ws["kernel_ms"], 3), "cluster_ms": round(ws["cluster_ms"], 3),
                                 "reorder_bytes": reorder,
                                 "reorder_gb_s": round(reorder / ws["cluster_ms"] * 1e-6, 1) if reorder else 0.0})
            if ws["verdict"] != V_RUNNING:
                break
        return levels if record else None

    for _ in range(max(0, args.warmup)):
        job(False)
        e.restart()
    kernels = None
    t0 = time.perf_counter()
    if args.kernels:
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            levels = job(True)
            torch.cuda.synchronize()
        kernels = {}
        for a in prof.key_averages():     # device time per kernel / copy / memset name, microseconds -> ms
            us = getattr(a, "self_device_time_total", None) or getattr(a, "self_cuda_time_total", 0)
            if us > 0:
                kernels[a.key[:120]] = kernels.get(a.key[:120], 0.0) + us * 1e-3
        kernels = {k: round(v, 3) for k, v in sorted(kernels.items(), key=lambda kv: -kv[1])}
    else:
        levels = job(True)
    wall = time.perf_counter() - t0
    r = e.result()
    counts_ok = (r["generated"], r["distinct"], r["depth"]) == (o2["generated"], o2["distinct"], o2["depth"])
    digest_ok = tuple(e.digest()) == (o2["fp_xor"], o2["fp_sum"])
    e.close()
    kern = sum(lv["kernel_ms"] for lv in levels)
    clus = sum(lv["cluster_ms"] for lv in levels)
    reorder = sum(lv["reorder_bytes"] for lv in levels)
    print(json.dumps({"fixture": args.fixture, "W": cm.W, "distinct": r["distinct"], "generated": r["generated"],
                      "depth": r["depth"], "wall_s": round(wall, 4), "kernel_s": round(kern * 1e-3, 4),
                      "cluster_s": round(clus * 1e-3, 4), "reorder_gb": round(reorder * 1e-9, 2),
                      "reorder_gb_s": round(reorder / clus * 1e-6, 1) if clus else 0.0,
                      "other_s": round(wall - (kern + clus) * 1e-3, 4), "counts_match_oracle": counts_ok,
                      "digest_matches_oracle": digest_ok,
                      "switches": switches(),
                      **({"kernels": kernels} if kernels is not None else {}),
                      "gpu": gpu_info(os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0] or "0"),
                      "levels": levels}))


if __name__ == "__main__":
    main()
