#!/usr/bin/env python
"""Honk's ResNets (Res8Model / Res8NarrowModel / Res15Model / Res15NarrowModel) in evaluation on one GPU, at the recipes' front-end
(40 MFCCs, 30 / 10 ms windows: 98 x 40), and TCResNet8-1.0 on the same clips.

Evaluation forward: utterances/s from int16 clips (front-end + network, the evaluate_audio.py path) at n = 512.  Per-kernel times:
the library's launch profiler (CUDA events around every launch) in a separate pass, ms per launch, each set against its FP32 FMA
floor: the layer's FLOPs (2 x multiply-adds, res_oracle's formula) at the data sheet's 67 TFLOP/s, and at the peak
tcr_measure_fp32_peak measures in the same run.  Every conv{k} has the same FLOPs, so the mean of the res_conv / res_conv_res
launches is set against one floor.  Yardstick: the same 45-channel 3x3 conv (dilation 1 and 16, n = 512, 98 x 40, NCHW fp32)
through torch.nn.functional.conv2d with TF32 off (cuDNN FP32).  Listener: ms per push of 64 streams x 10 windows (hop 1 frame,
100 ms chunks), eager and replayed from a CUDA graph.  Batch 1: ms per DeployedModel call replayed from its CUDA graph, wav in,
softmax copied out.  Warm-up, then `--repeats` rounds of `--iters` calls, each round timed with CUDA events; the result is the
median [min, max] over the rounds.  The card's name, power limit and maximum SM clock are read in the same run.

    python tools/bench_res_eval.py [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import shlex
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import tcresnet_b200  # noqa: E402,F401
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as TF  # noqa: E402
from bench_dscnn_eval import rounds  # noqa: E402
from bench_listener import card  # noqa: E402
from bench_res2d_eval import T, F, FRONTEND, FP32_TFLOPS, evaluation_tcresnet8, pcm_batch  # noqa: E402
from oracle import res_oracle as R  # noqa: E402
from tcresnet_b200.dscnn import RES_SIZES, DsCnn  # noqa: E402
from tcresnet_b200.engine import Engine  # noqa: E402


def handle(model, n):
    d = DsCnn(RES_SIZES[model], T, F, 12, n).set_frontend(**FRONTEND)
    return d, d.new_variables(seed=1), pcm_batch(n, d.device)


def evaluation(model, n, iters, repeats):
    d, params, pcm = handle(model, n)
    logits, probs = torch.empty(n, 12, device=d.device), torch.empty(n, 12, device=d.device)
    med, lo, hi = rounds(lambda: d.forward_input(pcm, params, logits=logits, probs=probs), iters, repeats)
    d.close()
    return dict(model=model, n=n, utt_per_s=n / med * 1e3, ms=[med, lo, hi], gflop_per_s=d.forward_flops * n / med * 1e-6)


def kernels(model, n, iters, eng, peak):
    d, params, pcm = handle(model, n)
    call = lambda: d.forward_input(pcm, params)  # noqa: E731
    for _ in range(5):
        call()
    torch.cuda.synchronize()
    eng.profile_read()                                               # drop earlier rows
    eng.profile(True)
    for _ in range(iters):
        call()
    torch.cuda.synchronize()
    eng.profile(False)
    rows = {k: (ms / max(c, 1), c // iters) for k, (ms, c) in eng.profile_read().items()}
    d.close()
    spec = R.build_spec(model, T, F)
    h, w = R.block_map(spec)
    fconv, conv = 2 * T * F * 9 * spec.c, 2 * h * w * 9 * spec.c * spec.c

    def entry(name, flops):
        ms = rows[name][0]
        f67, fpk = flops * n / (FP32_TFLOPS * 1e12) * 1e3, flops * n / (peak * 1e12) * 1e3
        return dict(ms_per_launch=ms, launches=rows[name][1], fp32_floor_ms_67=f67, fp32_floor_ms_measured_peak=fpk,
                    of_floor_67=f67 / ms, of_floor_measured_peak=fpk / ms)
    return dict(per_launch_ms={k: v[0] for k, v in rows.items()}, res_fconv=entry("res_fconv", fconv),
                res_conv=entry("res_conv", conv), res_conv_res=entry("res_conv_res", conv))


def yardstick(n, iters, repeats):
    """cuDNN FP32 (TF32 off): the 45 -> 45 3x3 conv at dilation 1 and 16 on [n, 45, 98, 40]."""
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        x = torch.randn(n, 45, T, F, device="cuda")
        wt = torch.randn(45, 45, 3, 3, device="cuda")
        out = {}
        for d in (1, 16):
            med, lo, hi = rounds(lambda: TF.conv2d(x, wt, dilation=d, padding=d), iters, repeats)
            f67 = 2 * T * F * 9 * 45 * 45 * n / (FP32_TFLOPS * 1e12) * 1e3
            out[f"dilation_{d}"] = dict(ms=[med, lo, hi], fp32_floor_ms_67=f67, of_floor_67=f67 / med)
        return out
    finally:
        torch.backends.cudnn.allow_tf32 = prev


def listener(model, streams, windows, iters, repeats):
    d = DsCnn(RES_SIZES[model], T, F, 12, streams * windows).set_frontend(**FRONTEND)
    params = d.new_variables(seed=1)
    chunk = windows * 160
    lis = d.listener(streams, 1, chunk, params)
    x = torch.rand(streams, chunk, device=d.device) * 2 - 1
    probs = torch.empty(streams, windows, 12, device=d.device)
    push = lambda: lis.push(x, probs=probs)  # noqa: E731
    eager = rounds(push, iters, repeats)
    s = torch.cuda.Stream(device=d.device)
    s.wait_stream(torch.cuda.current_stream(d.device))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        push()
    torch.cuda.current_stream(d.device).wait_stream(s)
    replay = rounds(graph.replay, iters, repeats)
    lis.close()
    d.close()
    return dict(model=model, streams=streams, windows=windows, eager_ms=list(eager), graph_ms=list(replay))


def batch1(model, iters, repeats):
    from tcresnet_b200 import evaluate_audio
    from tcresnet_b200.factory import audio_nets
    tail = " --width_multiplier 1.0" if model == "TCResNet8" else ""
    args = evaluate_audio.parse_arguments(shlex.split(
        "--dataset_path synthetic:8 --dataset_split_name valid --checkpoint_path x --batch_size 1 --augmentation_method "
        "anchored_slice_or_pad --output_name output/softmax --num_classes 12 --preprocess_method mfcc --num_mfccs 40 "
        f"--clip_duration_ms 1000 --window_size_ms 30 --window_stride_ms 10 {model}Model{tail}"))
    m = getattr(audio_nets, f"{model}Model")(args, None)
    _, dep = m.build_deployable_model(include_preprocess=True)
    x = np.random.default_rng(0).uniform(-1, 1, (1, 16000)).astype(np.float32)
    for _ in range(5):
        dep(x)
    assert dep._graph is not None
    ms = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        for _ in range(iters):
            dep(x)                                                   # ends in the D2H copy of the softmax: synchronised
        ms.append((time.perf_counter() - t0) / iters * 1e3)
    ms.sort()
    if isinstance(m.engine, DsCnn):
        m.engine.close()
    return dict(model=model, ms=[ms[len(ms) // 2], ms[0], ms[-1]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    models = list(RES_SIZES)
    res = dict(card=card(), geometry=[T, F])
    eng = Engine(max_batch=8)
    res["fp32_peak_tflops"] = peak = eng.fp32_peak_tflops()
    res["evaluation"] = [evaluation(m, 512, a.iters, a.repeats) for m in models] + [evaluation_tcresnet8(512, a.iters, a.repeats)]
    res["yardstick_cudnn_fp32_n512"] = yardstick(512, a.iters, a.repeats)
    res["listener"] = [listener(m, 64, 10, a.iters, a.repeats) for m in models]
    res["batch1"] = [batch1(m, a.iters, a.repeats) for m in models + ["TCResNet8"]]
    res["kernels_n512"] = {m: kernels(m, 512, a.iters, eng, peak) for m in models}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
