#!/usr/bin/env python
"""train_audio / evaluate_audio on a dataset read from disk: the host input path against --device_dataset.

One process, one GPU.  Writes a seeded Speech Commands-like split (wav files of 12,000 to 17,000 samples over 11 labels, silent
samples, six 60 s background recordings) into a temporary directory, then
  * times the train_audio loop (session.run of the train op, as the trainer runs it) at the recipe shape (TCResNet8, 30 ms / 10 ms
    windows: T = 98, batch 100) and at batch 512, host path and --device_dataset alternating in one process: `--warmup` steps, then
    per path a window of about `--seconds` of timed steps (at least `--min-steps`; the step count comes from one untimed
    calibration window, so the fast path is not timed over a few milliseconds), closed by a device synchronise, `--repeats`
    times; median, min and max;
  * times one evaluate_audio --valid_type once pass over the validation split both ways.
Prints the device name, its power limit and max SM clock (read-only nvidia-smi query), one line per measurement, and a final
JSON line.  Usage: python tools/bench_device_dataset.py [--clips 4400] [--warmup 5] [--seconds 2] [--min-steps 10] [--repeats 3]
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
import wave

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import tcresnet_b200  # noqa: E402,F401
from tcresnet_b200 import evaluate_audio, train_audio  # noqa: E402
from bench_optimizers import device_facts  # noqa: E402

LABELS = ["down", "go", "left", "no", "off", "on", "right", "stop", "unknown", "up", "yes"]
COMMON = ("--output_name output/softmax --num_classes 12 --preprocess_method mfcc --num_mfccs 40 --clip_duration_ms 1000 "
          "--window_size_ms 30 --window_stride_ms 10 ")


def _write(path, x):
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(16000)
        w.writeframes(np.ascontiguousarray(x, "<i2").tobytes())


def make_split(root, split, clips, seed):
    rng = np.random.RandomState(seed)
    for i in range(clips):
        d = os.path.join(root, split, LABELS[i % len(LABELS)])
        os.makedirs(d, exist_ok=True)
        _write(os.path.join(d, f"{i:06d}.wav"), rng.randint(-20000, 20000, rng.randint(12000, 17001)).astype(np.int16))
    noise = os.path.join(root, split, "_background_noise_")
    os.makedirs(noise, exist_ok=True)
    for j in range(6):
        _write(os.path.join(noise, f"noise{j}.wav"), rng.randint(-30000, 30000, 60 * 16000).astype(np.int16))


def trainer(root, batch, device, warmup):
    args = train_audio.parse_arguments(shlex.split(
        f"--dataset_path {root} --dataset_split_name train {COMMON} --train_dir {root}/run_{batch}_{int(device)} --num_silent 100 "
        f"--augmentation_method anchored_slice_or_pad_with_shift --batch_size {batch} --boundaries 100000 "
        f"--max_step_from_restore {warmup} --lr_list 0.1 0.01 --absolute_schedule --no-boundaries_epoch --step_save_checkpoint 100000 "
        f"--step_evaluation 100000 --step_save_summaries 100000 --step_save_first_n_summaries 0 --optimizer mom --momentum 0.9 "
        f"{'--device_dataset' if device else ''} TCResNet8Model --weight_decay 0.001 --width_multiplier 1.0"))
    return train_audio.train(args)


def timed_loop(t, steps):
    m = t.model
    fetch = {"step_op": t.train_op, "global_step": t.global_step, "total_loss": m.total_loss, "model_loss": m.model_loss}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        t.session.run(fetch)
    m.flush_feed()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def evaluate(root, device):
    args = evaluate_audio.parse_arguments(shlex.split(
        f"--dataset_path {root} --dataset_split_name valid {COMMON} --checkpoint_path {root}/run_100_1 --num_silent 100 "
        f"--augmentation_method anchored_slice_or_pad --background_frequency 0.0 --background_max_volume 0.0 --batch_size 100 "
        f"--no-shuffle --valid_type once --no-save_best_keeper {'--device_dataset' if device else ''} "
        f"TCResNet8Model --weight_decay 0.001 --width_multiplier 1.0"))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = evaluate_audio.main(args)[0]
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--clips", type=int, default=4400)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=2.0, help="timed work per window and path")
    ap.add_argument("--min-steps", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_device_dataset needs a CUDA device")
    facts = device_facts()
    print("device:", json.dumps(facts), flush=True)
    results = []
    with tempfile.TemporaryDirectory() as root:
        make_split(root, "train", a.clips, 0)
        make_split(root, "valid", a.clips // 4, 1)
        for batch in (100, 512):
            runs = {kind: trainer(root, batch, kind == "device", a.warmup) for kind in ("host", "device")}
            ms = {kind: [] for kind in runs}
            steps = {kind: max(a.min_steps, int(a.seconds * 1e3 / timed_loop(t, a.min_steps))) for kind, t in runs.items()}
            for _ in range(a.repeats):
                for kind, t in runs.items():                     # alternate the two paths inside every repeat
                    ms[kind].append(timed_loop(t, steps[kind]))
            for kind in runs:
                med = statistics.median(ms[kind])
                row = dict(what="train_audio loop", batch=batch, path=kind, ms_per_step_median=med, ms_per_step_min=min(ms[kind]),
                           ms_per_step_max=max(ms[kind]), steps=steps[kind], utt_per_s=batch / med * 1e3)
                results.append(row)
                print(f"train_audio N={batch:<4} {kind:>6}: {med:.3f} ms/step [{min(ms[kind]):.3f}, {max(ms[kind]):.3f}] over "
                      f"{a.repeats} x {steps[kind]} steps, {row['utt_per_s']:.0f} utt/s", flush=True)
            for t in runs.values():
                t.model.engine.close()
        evals = {}
        for kind in ("host", "device", "host", "device"):
            ms_eval, out = evaluate(root, kind == "device")
            evals.setdefault(kind, []).append(ms_eval)
            print(f"evaluate_audio once {kind:>6}: {ms_eval:.1f} ms (accuracy {out.get('accuracy')})", flush=True)
        for kind, v in evals.items():
            results.append(dict(what="evaluate_audio once", batch=100, path=kind, ms_median=statistics.median(v), ms_min=min(v),
                                ms_max=max(v), clips=a.clips // 4 + 100))
    print(json.dumps(dict(device=facts, clips=a.clips, warmup=a.warmup, seconds=a.seconds, repeats=a.repeats, results=results)))


if __name__ == "__main__":
    main()
