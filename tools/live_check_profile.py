"""Time `tlc`'s liveness check on the device: the label pass (tlag_label_graph), the obligation check and the lasso
(tlag_live_check), with the device memory in use once the graph is labelled, on the state graph of a search.

The default model is 7 counters mod 10 (10^7 states, 7 * 10^7 edges) under WF_c(Inc(i)) for every counter, with the
obligations []<>(c[i] = 0): they hold.  --drop-wf 1 drops the fairness of counter 1, so its obligation fails and the
lasso is built.  --spec / --cfg time a spec of your own instead.  Prints one JSON line with the card's name and power
limit, read in the same job.

    python tools/live_check_profile.py --repeat 3
    python tools/live_check_profile.py --drop-wf 1
"""
import argparse
import io
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

COUNTERS = """---- MODULE Counters ----
EXTENDS Naturals
VARIABLE c
Init == c = [i \\in 1..{k} |-> 0]
Inc(i) == c' = [c EXCEPT ![i] = (c[i] + 1) % {b}]
Next == \\E i \\in 1..{k} : Inc(i)
Spec == Init /\\ [][Next]_c /\\ \\A i \\in {fair} : WF_c(Inc(i))
Zero == \\A i \\in 1..{k} : []<>(c[i] = 0)
====
"""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--counters", type=int, default=7)
    ap.add_argument("--modulus", type=int, default=10)
    ap.add_argument("--drop-wf", type=int, default=0, help="counter whose WF condition is dropped (0: none)")
    ap.add_argument("--spec", help="a .tla of your own instead of the counters")
    ap.add_argument("--cfg")
    ap.add_argument("--engine", choices=["interp", "sliced"], default="interp")
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    import torch
    from tla_rust_b200.checker import compile_model, encode_states
    from tla_rust_b200.compile.lower import compile_labels
    from tla_rust_b200.engine import Engine, live_check
    from tla_rust_b200.front.spec import Model
    from tla_rust_b200.liveness import LabelPlan
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    if a.spec:
        path, cfg = a.spec, a.cfg
    else:
        d = tempfile.mkdtemp(prefix="live_check_profile_")
        fair = "{" + ", ".join(str(i) for i in range(1, a.counters + 1) if i != a.drop_wf) + "}"
        path = os.path.join(d, "Counters.tla")
        with open(path, "w") as f:
            f.write(COUNTERS.format(k=a.counters, b=a.modulus, fair=fair))
        cfg = os.path.join(d, "Counters.cfg")
        with open(cfg, "w") as f:
            f.write("SPECIFICATION Spec\nPROPERTY Zero\n")
    m = Model(path, cfg_path=cfg)
    m.ev.out = io.StringIO()
    cm = compile_model(m)
    plan = LabelPlan(m)
    img = compile_labels(m, cm, plan.state, plan.edge)
    e = Engine(cm, deadlock=False, native="sliced" if a.engine == "sliced" else False)
    e.seed(encode_states(cm, m.initial_states()))
    e.run()
    gi = e.build_graph()
    free0, total = torch.cuda.mem_get_info()
    label_ms, check_ms, lasso_ms, used = [], [], [], []
    verdicts = []
    for _ in range(a.repeat):
        label_ms.append(e.label_graph(img, *plan.en_map()))
        used.append(total - torch.cuda.mem_get_info()[0])
        view = e.graph_view()
        c, l, v = 0.0, 0.0, []
        for _ob, qy in plan.queries:
            r = live_check(view, **plan.args(qy, view.n_init))
            c += r["check_ms"]
            l += r["lasso_ms"]
            v.append(r["violated"])
        check_ms.append(c)
        lasso_ms.append(l)
        verdicts = v
    e.close()
    print(json.dumps({
        "gpu": q[0] if q else None, "model": os.path.basename(path), "n_states": gi["n_states"],
        "n_edges": gi["n_edges"], "obligations": len(plan.queries), "violated": sum(verdicts),
        "label_ms_median": statistics.median(label_ms), "check_ms_median": statistics.median(check_ms),
        "lasso_ms_median": statistics.median(lasso_ms), "repeat": a.repeat,
        "device_bytes_in_use_after_graph": total - free0,
        "device_bytes_in_use_after_labels": max(used) if used else None,
        "note": "check and lasso: sums over the obligations (CUDA events); memory: cudaMemGetInfo of the whole device "
                "(store, seen-set, graph, labels); the check's own buffers are freed when it returns and are not in it"}))


if __name__ == "__main__":
    main()
