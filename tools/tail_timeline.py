"""Timeline of the training step's tail: from the end of dw_grouped (the last weight-gradient kernel of step i) to the start of
resident_fwd (the first network kernel of step i + 1), in the configuration bench.py times (TCResNet8-1.0, N = 512, front-end
running ahead on the library's stream).

Kernel start / end times come from CUPTI's activity records (torch.profiler), one timebase for every kernel on both streams;
the kernels themselves are not instrumented, so what they compile to is what the step runs.  CUPTI adds a little per-launch
overhead: take the gaps as an upper bound and the step time from bench.py.

Reports per step: the gap dw_grouped end -> resident_fwd start, every kernel that runs inside it (start / end relative to
dw_grouped's end) and which of them ends last.  Environment knobs (TCR_FUSED_UPDATE, ...) pass through to the library.

    python tools/tail_timeline.py [--model TCResNet8 --width 1.0 --batch 512 --steps 20 --warmup 20] [--out FILE.json]
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import tcresnet_b200  # noqa: F401,E402
from tcresnet_b200.engine import Engine  # noqa: E402
from tcresnet_b200.plan import build_plan  # noqa: E402

SHORT = [("dw_grouped", "dw_grouped"), ("grad_finalize", "grad_finalize"), ("update_kernel", "update"),
         ("mfcc", "mfcc"), ("resident_fwd", "resident_fwd"), ("resident_bwd", "resident_bwd_data")]


def short_name(name):
    for key, s in SHORT:
        if key in name:
            return s
    return name.split("(")[0].split("<")[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="TCResNet8")
    ap.add_argument("--width", type=float, default=1.0)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None, help="write the per-step records as JSON")
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    n = a.batch
    eng = Engine(model=a.model, width_multiplier=a.width, max_batch=n, dropout_keep_prob=0.5, device=0)
    plan = build_plan(a.model, a.width)
    params, slots, moving = eng.new_variables(seed=0)
    gen = torch.Generator(device=dev).manual_seed(1234)
    wavs = [torch.rand(n, plan.clip, device=dev, generator=gen) * 2 - 1 for _ in range(2)]
    labels = torch.randint(0, 12, (2, n), device=dev, generator=torch.Generator(device=dev).manual_seed(4321))
    hots = [torch.nn.functional.one_hot(labels[i], 12).float().contiguous() for i in range(2)]
    losses = torch.zeros(2, device=dev)

    def step(i):
        eng.train_step(wavs[i % 2], hots[i % 2], params, slots, moving, 0.1, 0.9, 1e-3, dropout_seed=i, losses=losses,
                       input_resident=True)

    for i in range(a.warmup):
        step(i)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(a.steps):
            step(a.warmup + i)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    ks = sorted(((float(e["ts"]), float(e["ts"]) + float(e["dur"]), short_name(e["name"]))
                 for e in trace["traceEvents"] if e.get("cat") == "kernel"), key=lambda k: k[0])
    dws = [k for k in ks if k[2] == "dw_grouped"]
    fwds = [k for k in ks if k[2] == "resident_fwd"]
    steps = []
    for dw in dws:
        nxt = [f for f in fwds if f[0] >= dw[0]]
        if not nxt:
            continue
        rf = nxt[0]
        inside = [k for k in ks if k[1] > dw[1] and k[0] < rf[0] and k is not dw]
        rec = {"gap_us": rf[0] - dw[1], "dw_grouped_us": dw[1] - dw[0],
               "kernels": [{"name": k[2], "start_us": k[0] - dw[1], "end_us": k[1] - dw[1]} for k in inside]}
        rec["ends_last"] = max(inside, key=lambda k: k[1])[2] if inside else None
        steps.append(rec)
    if len(fwds) > 1:
        period = float(np.median(np.diff([f[0] for f in fwds])))
    else:
        period = float("nan")
    gaps = np.array([s["gap_us"] for s in steps])
    print(f"{a.model}-{a.width:g} N={n}: {len(steps)} steps, step period (resident_fwd to resident_fwd) median {period:.1f} us, "
          f"dw_grouped median {np.median([s['dw_grouped_us'] for s in steps]):.1f} us")
    print(f"gap dw_grouped end -> next resident_fwd start: median {np.median(gaps):.1f} us, min {gaps.min():.1f}, max {gaps.max():.1f}")
    last = {}
    for s in steps:
        last[s["ends_last"]] = last.get(s["ends_last"], 0) + 1
    print("ends last inside the gap:", last)
    names = sorted({k["name"] for s in steps for k in s["kernels"]})
    for nm in names:
        st = [k["start_us"] for s in steps for k in s["kernels"] if k["name"] == nm]
        en = [k["end_us"] for s in steps for k in s["kernels"] if k["name"] == nm]
        print(f"  {nm:18s} start {np.median(st):7.1f} us  end {np.median(en):7.1f} us  (medians, from dw_grouped's end; {len(st)} launches)")
    print("device:", torch.cuda.get_device_name(0))
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"model": a.model, "width": a.width, "batch": n, "period_us": period, "steps": steps,
                       "env": {k: v for k, v in os.environ.items() if k.startswith("TCR_")}}, f, indent=1)


if __name__ == "__main__":
    main()
