#!/usr/bin/env python
"""Training-step time with each optimizer of the fused update kernel: momentum, Adam and RMSProp.

One process, one GPU.  For TCResNet8-1.0 at N=512 and TCResNet14-1.5 at N=1024 it runs blocks of steps that alternate
mom / adam / rmsprop (10 warm-up steps, then 50 steps timed with CUDA events, 3 repeats), then a separate pass with the
library's launch profiler on (tcr_profile_enable) for the per-launch time of the `update` kernel.  The profiler brackets every
launch with events, so its numbers come from their own pass and the step times from passes without it.

Prints the device name, its power limit and max SM clock (read-only nvidia-smi query), one line per measurement, and a final
JSON line.  Usage: python tools/bench_optimizers.py [--warmup 10] [--steps 50] [--repeats 3] [--profile-steps 50]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import tcresnet_b200  # noqa: E402,F401
from tcresnet_b200.engine import Engine  # noqa: E402

SHAPES = [("TCResNet8", 1.0, 512), ("TCResNet14", 1.5, 1024)]
OPTIMIZERS = {
    "mom": None,
    "adam": dict(kind="adam", beta1=0.9, beta2=0.999, epsilon=1e-8),
    "rmsprop": dict(kind="rmsprop", decay=0.9, momentum=0.0, epsilon=1e-10),
}


def device_facts():
    """Name, power limit and max SM clock of GPU 0, queried read-only."""
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = (x.strip() for x in r.stdout.strip().splitlines()[0].split(","))
        out.update(name=name, power_limit_w=float(power), max_sm_mhz=float(clock))
    except Exception as e:                     # the numbers below still stand; say why the card facts are missing
        out["nvidia_smi_error"] = repr(e)
    return out


class Run:
    """One engine and its inputs; one state (params, slots, moving) per optimizer, so each kind trains its own replica."""

    def __init__(self, model, width, n):
        self.n = n
        self.eng = Engine(model=model, width_multiplier=width, max_batch=n, dropout_keep_prob=0.5)
        dev = self.eng.device
        gen = torch.Generator(device=dev).manual_seed(1234)
        self.wavs = [torch.rand(n, self.eng.cfg.clip_samples, device=dev, generator=gen) * 2 - 1 for _ in range(8)]
        labels = torch.randint(0, 12, (8, n), device=dev, generator=torch.Generator(device=dev).manual_seed(4321))
        self.hots = [torch.nn.functional.one_hot(labels[i], 12).float().contiguous() for i in range(8)]
        self.losses = torch.zeros(2, device=dev)
        self.state = {}
        for kind in OPTIMIZERS:
            params, _, moving = self.eng.new_variables(seed=0)
            slots, slots2 = self.eng.new_optimizer_state(kind)
            self.state[kind] = dict(params=params, slots=slots, slots2=slots2, moving=moving, t=0)
        self.num_trainable = self.eng.num_trainable

    def step(self, kind, i):
        s = self.state[kind]
        opt = OPTIMIZERS[kind]
        if opt is not None and opt["kind"] == "adam":
            s["t"] += 1
            opt = dict(opt, beta1_power=0.9 ** s["t"], beta2_power=0.999 ** s["t"])
        lr = 0.1 if kind == "mom" else 1e-3
        self.eng.train_step(self.wavs[i % 8], self.hots[i % 8], s["params"], s["slots"], s["moving"], lr, 0.9, 1e-3, dropout_seed=i,
                            losses=self.losses, input_resident=True, optimizer=opt, slots2=s["slots2"])

    def timed(self, kind, warmup, steps):
        for i in range(warmup):
            self.step(kind, i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            self.step(kind, warmup + i)
        e1.record()
        torch.cuda.synchronize()
        assert torch.isfinite(self.losses).all(), (kind, self.losses)
        return e0.elapsed_time(e1) / steps

    def update_launch_ms(self, kind, steps):
        for i in range(3):
            self.step(kind, i)
        torch.cuda.synchronize()
        self.eng.profile(True)                                # clears what earlier passes recorded
        for i in range(steps):
            self.step(kind, i)
        torch.cuda.synchronize()
        stats = self.eng.profile_read()
        self.eng.profile(False)
        total, launches = stats["update"]
        return total / launches


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--profile-steps", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_optimizers needs a CUDA device")
    facts = device_facts()
    print("device:", json.dumps(facts), flush=True)
    results = []
    for model, width, n in SHAPES:
        run = Run(model, width, n)
        ms = {k: [] for k in OPTIMIZERS}
        for rep in range(a.repeats):
            for kind in OPTIMIZERS:                           # alternate the kinds inside every repeat
                ms[kind].append(run.timed(kind, a.warmup, a.steps))
        upd = {kind: run.update_launch_ms(kind, a.profile_steps) for kind in OPTIMIZERS}
        for kind in OPTIMIZERS:
            bytes_per_param = {"mom": 20, "adam": 28, "rmsprop": 28}[kind]   # g, w, slot(s): loads + stores, fp32
            row = dict(model=f"{model}-{width}", batch=n, optimizer=kind, params=run.num_trainable,
                       ms_per_step_median=statistics.median(ms[kind]), ms_per_step_min=min(ms[kind]),
                       ms_per_step_max=max(ms[kind]), utt_per_s=n / (statistics.median(ms[kind]) * 1e-3),
                       update_launch_us=upd[kind] * 1e3, update_bytes=bytes_per_param * run.num_trainable)
            results.append(row)
            print(f"{row['model']:>16} N={n:<5} {kind:>8}: step {row['ms_per_step_median']:.4f} ms "
                  f"[{row['ms_per_step_min']:.4f}, {row['ms_per_step_max']:.4f}] over {a.repeats} x {a.steps} steps, "
                  f"{row['utt_per_s'] / 1e3:.0f} k utt/s; update launch {row['update_launch_us']:.1f} us (profiler pass), "
                  f"{row['update_bytes'] / 1e6:.2f} MB moved by the update", flush=True)
        run.eng.close()
    print(json.dumps(dict(device=facts, warmup=a.warmup, steps=a.steps, repeats=a.repeats, results=results)))


if __name__ == "__main__":
    main()
