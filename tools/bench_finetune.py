#!/usr/bin/env python
"""Training-step time of partial training (tcr_set_trainable) and the weight EMA (tcr_step_args::ema) against the full step.

One process, one GPU.  For TCResNet8-1.0 at N=512 and TCResNet14-1.5 at N=1024 it runs blocks of Adam steps that alternate the
variants full / full + EMA / block 2 only / BatchNorm only / head only (10 warm-up steps, then 50 steps timed with CUDA events,
3 repeats); each variant trains its own replica, and the trainable set is switched outside the timed windows.

Prints the device name, its power limit and max SM clock (read-only nvidia-smi query), one line per measurement, and a final
JSON line.  Usage: python tools/bench_finetune.py [--warmup 10] [--steps 50] [--repeats 3]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import tcresnet_b200  # noqa: E402,F401
from tcresnet_b200.common.model_loader import variables_to_train  # noqa: E402
from tcresnet_b200.engine import Engine  # noqa: E402
from bench_optimizers import device_facts  # noqa: E402

SHAPES = [("TCResNet8", 1.0, 512), ("TCResNet14", 1.5, 1024)]
VARIANTS = {"full": ("", False), "full+ema": ("", True), "block2": ("{m}/block2", False), "bn": (".*BatchNorm", False),
            "head": ("{m}/fc", False)}
ADAM = dict(kind="adam", beta1=0.9, beta2=0.999, epsilon=1e-8)


class Run:
    def __init__(self, model, width, n):
        self.n, self.model = n, model
        self.eng = Engine(model=model, width_multiplier=width, max_batch=n, dropout_keep_prob=0.5)
        dev = self.eng.device
        gen = torch.Generator(device=dev).manual_seed(1234)
        self.wavs = [torch.rand(n, self.eng.cfg.clip_samples, device=dev, generator=gen) * 2 - 1 for _ in range(8)]
        labels = torch.randint(0, 12, (8, n), device=dev, generator=torch.Generator(device=dev).manual_seed(4321))
        self.hots = [torch.nn.functional.one_hot(labels[i], 12).float().contiguous() for i in range(8)]
        self.losses = torch.zeros(2, device=dev)
        self.state = {}
        for v, (scope, ema) in VARIANTS.items():
            params, _, moving = self.eng.new_variables(seed=0)
            slots, slots2 = self.eng.new_optimizer_state("adam")
            trained = variables_to_train(scope.format(m=model), self.eng.trainable_names)
            self.state[v] = dict(params=params, slots=slots, slots2=slots2, moving=moving, t=0,
                                 ema=self.eng.new_ema(params) if ema else None,
                                 trained=None if len(trained) == len(self.eng.trainable_names) else trained)

    def step(self, v, i):
        s = self.state[v]
        s["t"] += 1
        opt = dict(ADAM, beta1_power=0.9 ** s["t"], beta2_power=0.999 ** s["t"])
        self.eng.train_step(self.wavs[i % 8], self.hots[i % 8], s["params"], s["slots"], s["moving"], 1e-3, 0.9, 1e-3, dropout_seed=i,
                            losses=self.losses, input_resident=True, optimizer=opt, slots2=s["slots2"], ema=s["ema"],
                            ema_decay=0.999)

    def timed(self, v, warmup, steps):
        self.eng.set_trainable(self.state[v]["trained"])
        for i in range(warmup):
            self.step(v, i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            self.step(v, warmup + i)
        e1.record()
        torch.cuda.synchronize()
        assert torch.isfinite(self.losses).all(), (v, self.losses)
        return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_finetune needs a CUDA device")
    facts = device_facts()
    print("device:", json.dumps(facts), flush=True)
    results = []
    for model, width, n in SHAPES:
        run = Run(model, width, n)
        ms = {v: [] for v in VARIANTS}
        for _ in range(a.repeats):
            for v in VARIANTS:                                # alternate the variants inside every repeat
                ms[v].append(run.timed(v, a.warmup, a.steps))
        full = statistics.median(ms["full"])
        for v in VARIANTS:
            med = statistics.median(ms[v])
            row = dict(model=f"{model}-{width}", batch=n, variant=v, ms_per_step_median=med, ms_per_step_min=min(ms[v]),
                       ms_per_step_max=max(ms[v]), vs_full=med / full)
            results.append(row)
            print(f"{row['model']:>16} N={n:<5} {v:>9}: step {med:.4f} ms [{min(ms[v]):.4f}, {max(ms[v]):.4f}] over "
                  f"{a.repeats} x {a.steps} steps, {row['vs_full']:.3f} x full", flush=True)
        run.eng.close()
    print(json.dumps(dict(device=facts, warmup=a.warmup, steps=a.steps, repeats=a.repeats, results=results)))


if __name__ == "__main__":
    main()
