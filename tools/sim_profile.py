"""Rate of `tlc -simulate` on the device: for each model (compiled fixtures) and both engines, one warm-up batch, then
timed batches of behaviours of at most --depth states.  Prints per run the walks per batch, states checked per second of
device time and the device time per step (a batch's device time over its steps), with the card's name and power limit
read in the same process.

    python tools/sim_profile.py [--models MCPaxos3_b4,MCraft_t4l3,MCssi_4x3] [--depth 100] [--batches 2]
"""
import argparse
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="MCPaxos3_b4,MCraft_t4l3,MCssi_4x3")
    ap.add_argument("--depth", type=int, default=100)
    ap.add_argument("--batches", type=int, default=2, help="timed batches per run (after one warm-up batch)")
    ap.add_argument("--engines", default="interp,sliced")
    a = ap.parse_args()
    from tla_rust_b200.compiled import load_compiled
    from tla_rust_b200.engine import Engine
    print(f"card: {card()}", flush=True)
    for name in a.models.split(","):
        cm, init, _exp, info = load_compiled(os.path.join(ROOT, "tests", "golden", name + ".tlagz"))
        for eng in a.engines.split(","):
            e = Engine(cm, deadlock=info["deadlock"], native="sliced" if eng == "sliced" else False, simulate=True)
            e.seed(init)
            # walks per batch (include/tlag.h): min(2^20, 4 GiB of history), a multiple of 32
            B = min(1 << 20, (4 << 30) // (a.depth * (4 * cm.W + 2))) // 32 * 32
            w = e.simulate(1, B, a.depth)                       # warm-up: one batch
            assert w["batch_walks"] == B
            r = e.simulate(2, B * a.batches, a.depth)
            # steps run: a batch that holds an error stops after its step (the rest of its steps are no-ops)
            steps = a.depth * (r["behaviours"] // B - 1) + (r["step"] + 1 if r["verdict"] else a.depth)
            out = dict(model=name, engine=eng, W=cm.W, depth=a.depth, batch_walks=B, behaviours=r["behaviours"],
                       verdict=r["verdict"], detail=r["detail"], error_step=r["step"] if r["verdict"] else None, checked=r["checked"], generated=r["generated"],
                       device_s=round(r["device_ms"] * 1e-3, 4),
                       checked_per_s=round(r["checked"] / (r["device_ms"] * 1e-3)) if r["device_ms"] else None,
                       ms_per_step=round(r["device_ms"] / steps, 4) if steps else None)
            print(json.dumps(out), flush=True)
            e.close()
    print(f"card: {card()}", flush=True)


if __name__ == "__main__":
    main()
