#!/usr/bin/env python
"""KWS baselines (KWSModel --architecture trad_fpool3 / one_fstride4) evaluation on one GPU, at the recipes' front-end (40 MFCCs,
40 / 20 ms windows: 49 x 40).

Evaluation forward: utterances/s of DsCnn.forward_input from int16 clips (front-end + network, the evaluate_audio.py path) at
n = 512 for both models.  Per-kernel times: the library's launch profiler (tcr_profile_enable, CUDA events around every launch) in
a separate pass, ms per launch.  trad_fpool3's two wgmma convs (kws_conv1_tc, kws_conv2_tc) are each set against two floors: the
3xTF32 MMA work at the data sheet's 495 TFLOP/s dense TF32, and the FLOPs at the FP32 FMA peak tcr_measure_fp32_peak measures in the
same run.  Listener: ms
per push of 64 streams x 10 windows (hop 1 frame = 20 ms, 200 ms chunks), eager and replayed from a CUDA graph.  Batch 1: ms per
DeployedModel call replayed from its CUDA graph, wav in, softmax copied out.  Warm-up, then `--repeats` rounds of `--iters` calls,
each round timed with CUDA events; the result is the median [min, max] over the rounds.  The card's name, power limit and maximum
SM clock are read in the same run.

    python tools/bench_kws_eval.py [--out result.json]
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
from bench_dscnn_eval import rounds  # noqa: E402
from bench_listener import card  # noqa: E402
from tcresnet_b200.dscnn import KWS_SIZES, DsCnn  # noqa: E402
from tcresnet_b200.engine import Engine  # noqa: E402

FRONTEND = dict(num_mfccs=40, window_size_ms=40, window_stride_ms=20)
TF32_DENSE_TFLOPS = 495.0                # H100 SXM data sheet, dense TF32
CONV1_FLOPS = 2 * 30 * 33 * 160 * 64     # trad_fpool3's 20 x 8 conv, 1 -> 64, per utterance at 49 x 40 (before the pool)
CONV2_FLOPS = 2 * 21 * 8 * 2560 * 64     # trad_fpool3's 10 x 4 conv, 64 -> 64


def handle(arch, n):
    d = DsCnn(KWS_SIZES[arch], 49, 40, 12, n).set_frontend(**FRONTEND)
    g = torch.Generator(device=d.device).manual_seed(0)
    pcm = torch.randint(-32768, 32768, (n, 16000), device=d.device, generator=g, dtype=torch.int32).to(torch.int16)
    return d, d.new_variables(seed=1), pcm


def evaluation(arch, n, iters, repeats):
    d, params, pcm = handle(arch, n)
    logits, probs = torch.empty(n, 12, device=d.device), torch.empty(n, 12, device=d.device)
    med, lo, hi = rounds(lambda: d.forward_input(pcm, params, logits=logits, probs=probs), iters, repeats)
    d.close()
    return dict(arch=arch, n=n, utt_per_s=n / med * 1e3, ms=[med, lo, hi], gflop_per_s=d.forward_flops * n / med * 1e-6)


def kernels(arch, n, iters, eng):
    d, params, pcm = handle(arch, n)
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
    rows = {k: ms / max(c, 1) for k, (ms, c) in eng.profile_read().items()}
    d.close()
    return rows


def listener(arch, streams, windows, iters, repeats):
    d = DsCnn(KWS_SIZES[arch], 49, 40, 12, streams * windows).set_frontend(**FRONTEND)
    params = d.new_variables(seed=1)
    chunk = windows * 320
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
    return dict(arch=arch, streams=streams, windows=windows, eager_ms=list(eager), graph_ms=list(replay))


def batch1(arch, iters, repeats):
    from tcresnet_b200 import evaluate_audio
    from tcresnet_b200.factory import audio_nets
    args = evaluate_audio.parse_arguments(shlex.split(
        "--dataset_path synthetic:8 --dataset_split_name valid --checkpoint_path x --batch_size 1 --augmentation_method "
        "anchored_slice_or_pad --output_name output/softmax --num_classes 12 --preprocess_method mfcc --num_mfccs 40 "
        f"--clip_duration_ms 1000 --window_size_ms 40 --window_stride_ms 20 KWSModel --architecture {arch}"))
    m = audio_nets.KWSModel(args, None)
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
    m.engine.close()
    return dict(arch=arch, ms=[ms[len(ms) // 2], ms[0], ms[-1]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    archs = list(KWS_SIZES)
    res = dict(card=card())
    res["evaluation"] = [evaluation(arch, 512, a.iters, a.repeats) for arch in archs]
    res["listener"] = [listener(arch, 64, 10, a.iters, a.repeats) for arch in archs]
    res["batch1"] = [batch1(arch, a.iters, a.repeats) for arch in archs]
    eng = Engine(max_batch=8)
    time.sleep(1.0)
    res["fp32_peak_tflops"] = peak = eng.fp32_peak_tflops()
    res["kernels_ms"] = {arch: kernels(arch, 512, a.iters, eng) for arch in archs}
    for key, name, flops in (("conv1_n512", "kws_conv1_tc", CONV1_FLOPS), ("conv2_n512", "kws_conv2_tc", CONV2_FLOPS)):
        ms = res["kernels_ms"]["trad_fpool3"].get(name)
        floors = dict(tf32_3x_ms=3 * flops * 512 / (TF32_DENSE_TFLOPS * 1e12) * 1e3, fp32_fma_ms=flops * 512 / (peak * 1e12) * 1e3)
        res[key] = dict(kernel=name, kernel_ms=ms, floors=floors, tflops=flops * 512 / (ms * 1e-3) / 1e12 if ms else None)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
