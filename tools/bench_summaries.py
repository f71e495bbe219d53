#!/usr/bin/env python
"""The train_audio loop (SingleLabelAudioTrainer.train) with and without TensorBoard summaries, alternating in one process.

Same seeded on-disk split, recipe shape and paths as tools/bench_device_dataset.py (TCResNet8, 30 ms / 10 ms windows, batch 100,
host path and --device_dataset).  Both trainers run the reference's summary schedule (--step_save_summaries 10, --max_outputs 5
wav clips at 16 kHz); the one "without" has no writer, so the difference is the cost of the summaries alone.  Checkpoints and
evaluations are left out of the timed windows.  Each window is `--steps` steps of trainer.train(), closed by draining the
pipeline and a device synchronise; `--repeats` windows per variant, alternating; median, min and max.
Usage: python tools/bench_summaries.py [--clips 4400] [--steps 300] [--repeats 5]
"""
from __future__ import annotations

import argparse
import json
import os
import shlex
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import tcresnet_b200  # noqa: E402,F401
from tcresnet_b200 import train_audio  # noqa: E402
from tcresnet_b200.metrics.manager import Summaries  # noqa: E402
from bench_device_dataset import COMMON, make_split  # noqa: E402
from bench_optimizers import device_facts  # noqa: E402


def trainer(root, batch, device, run):
    args = train_audio.parse_arguments(shlex.split(
        f"--dataset_path {root} --dataset_split_name train {COMMON} --train_dir {root}/{run} --num_silent 100 "
        f"--augmentation_method anchored_slice_or_pad_with_shift --batch_size {batch} --boundaries 100000 "
        f"--max_step_from_restore 5 --lr_list 0.1 0.01 --absolute_schedule --no-boundaries_epoch --step_save_checkpoint 100000 "
        f"--step_evaluation 1000000000 --step_save_summaries 10 --max_outputs 5 --optimizer mom --momentum 0.9 "
        f"{'--device_dataset' if device else ''} TCResNet8Model --weight_decay 0.001 --width_multiplier 1.0"))
    t = train_audio.train(args)
    t.save_checkpoint = lambda step: None
    return t


def timed_train(t, steps, summaries):
    if summaries:
        t.metric_manager.summary = Summaries(t.args.train_dir, t.args.max_outputs)
    t.args.max_step_from_restore += steps
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    t.train()
    t.model.flush_feed()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--clips", type=int, default=4400)
    ap.add_argument("--batch", type=int, default=100)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_summaries needs a CUDA device")
    facts = device_facts()
    print("device:", json.dumps(facts), flush=True)
    results = []
    with tempfile.TemporaryDirectory() as root:
        make_split(root, "train", a.clips, 0)
        for path in ("host", "device"):
            runs = {on: trainer(root, a.batch, path == "device", f"run_{path}_{int(on)}") for on in (False, True)}
            for on, t in runs.items():
                if not on:
                    t.metric_manager.close_summaries()
                    t.metric_manager.summary = None
                timed_train(t, 20, on)                           # warm-up window
            ms = {on: [] for on in runs}
            for _ in range(a.repeats):
                for on, t in runs.items():                       # alternate the two variants inside every repeat
                    ms[on].append(timed_train(t, a.steps, on))
            for on, v in ms.items():
                med = statistics.median(v)
                row = dict(what="train_audio loop", batch=a.batch, path=path, summaries=on, ms_per_step_median=med,
                           ms_per_step_min=min(v), ms_per_step_max=max(v), steps=a.steps, repeats=a.repeats)
                results.append(row)
                print(f"train_audio N={a.batch} {path:>6} summaries={'on ' if on else 'off'}: {med:.3f} ms/step "
                      f"[{min(v):.3f}, {max(v):.3f}] over {a.repeats} x {a.steps} steps", flush=True)
            for t in runs.values():
                t.model.engine.close()
    print(json.dumps(dict(device=facts, clips=a.clips, results=results)))


if __name__ == "__main__":
    main()
