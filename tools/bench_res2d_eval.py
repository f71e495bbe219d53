#!/usr/bin/env python
"""The 2-D ablations of TC-ResNet8 (ResNet2D8Model / ResNet2D8PoolModel) in evaluation on one GPU, at the recipes' front-end
(40 MFCCs, 30 / 10 ms windows: 98 x 40), width 1.0, and TCResNet8-1.0 on the same clips for the paper's comparison.

Evaluation forward: utterances/s from int16 clips (front-end + network, the evaluate_audio.py path) at n = 512.  Per-kernel
times: the library's launch profiler (CUDA events around every launch) in a separate pass, ms per launch, each set against its
FP32 FMA floor: the layer's FLOPs (2 x multiply-adds, res2d_oracle.forward_flops's formula) at the data sheet's 67 TFLOP/s.
Listener: ms per push of 64 streams x 10 windows (hop 1 frame, 100 ms chunks), eager and replayed from a CUDA graph.  Batch 1:
ms per DeployedModel call replayed from its CUDA graph, wav in, softmax copied out.  Warm-up, then `--repeats` rounds of
`--iters` calls, each round timed with CUDA events; the result is the median [min, max] over the rounds.  The card's name, power
limit and maximum SM clock are read in the same run.

    python tools/bench_res2d_eval.py [--out result.json]
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
from oracle import res2d_oracle as R  # noqa: E402
from tcresnet_b200.dscnn import RES2D_SIZES, DsCnn  # noqa: E402
from tcresnet_b200.engine import Engine  # noqa: E402

FRONTEND = dict(num_mfccs=40, window_size_ms=30, window_stride_ms=10)
T, F = 98, 40
FP32_TFLOPS = 67.0                       # H100 SXM data sheet, FP32 (non-tensor)


def layer_flops(model):
    """FLOPs per utterance of each kernel at 98 x 40: res2d_conv0 and the three res2d_block launches."""
    spec = R.build_spec(model, T, F)
    geo = R.geometry(spec)
    out = [2 * T * F * 9 * spec.ch[0]]
    for i, b in enumerate(spec.blocks):
        ho, wo, n = geo[i + 1]
        cin = geo[i][2]
        out.append(2 * ho * wo * (9 * cin * n + 9 * n * n + (cin * n if b["down"] else 0)))
    return out


def pcm_batch(n, device):
    g = torch.Generator(device=device).manual_seed(0)
    return torch.randint(-32768, 32768, (n, 16000), device=device, generator=g, dtype=torch.int32).to(torch.int16)


def handle(model, n):
    d = DsCnn(RES2D_SIZES[model], T, F, 12, n).set_frontend(**FRONTEND)
    return d, d.new_variables(seed=1), pcm_batch(n, d.device)


def evaluation(model, n, iters, repeats):
    d, params, pcm = handle(model, n)
    logits, probs = torch.empty(n, 12, device=d.device), torch.empty(n, 12, device=d.device)
    med, lo, hi = rounds(lambda: d.forward_input(pcm, params, logits=logits, probs=probs), iters, repeats)
    d.close()
    return dict(model=model, n=n, utt_per_s=n / med * 1e3, ms=[med, lo, hi], gflop_per_s=d.forward_flops * n / med * 1e-6)


def evaluation_tcresnet8(n, iters, repeats):
    eng = Engine("TCResNet8", max_batch=n, **FRONTEND)
    assert (eng.info.frames, eng.info.features) == (T, F)
    params, _, moving = eng.new_variables(seed=1)
    pcm = pcm_batch(n, eng.device)
    med, lo, hi = rounds(lambda: eng.forward(pcm, params, moving), iters, repeats)
    flops = eng.info.forward_flops_per_utt
    del eng
    return dict(model="TCResNet8", n=n, utt_per_s=n / med * 1e3, ms=[med, lo, hi], gflop_per_s=flops * n / med * 1e-6)


def kernels(model, n, iters, eng):
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
    flops = layer_flops(model)
    conv0_ms = rows["res2d_conv0"][0]
    block_ms = rows["res2d_block"][0]                                # the mean of the three launches
    floor = lambda f: f * n / (FP32_TFLOPS * 1e12) * 1e3  # noqa: E731
    return dict(per_launch_ms={k: v[0] for k, v in rows.items()},
                res2d_conv0=dict(ms=conv0_ms, fp32_floor_ms=floor(flops[0])),
                res2d_block=dict(ms_mean_of_3=block_ms, fp32_floor_ms=[floor(f) for f in flops[1:]],
                                 fp32_floor_ms_sum=floor(sum(flops[1:])), ms_sum=3 * block_ms))


def listener(model, streams, windows, iters, repeats):
    d = DsCnn(RES2D_SIZES[model], T, F, 12, streams * windows).set_frontend(**FRONTEND)
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
    args = evaluate_audio.parse_arguments(shlex.split(
        "--dataset_path synthetic:8 --dataset_split_name valid --checkpoint_path x --batch_size 1 --augmentation_method "
        "anchored_slice_or_pad --output_name output/softmax --num_classes 12 --preprocess_method mfcc --num_mfccs 40 "
        f"--clip_duration_ms 1000 --window_size_ms 30 --window_stride_ms 10 {model}Model --width_multiplier 1.0"))
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
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    models = list(RES2D_SIZES)
    res = dict(card=card(), geometry=[T, F])
    res["evaluation"] = [evaluation(m, 512, a.iters, a.repeats) for m in models] + [evaluation_tcresnet8(512, a.iters, a.repeats)]
    res["listener"] = [listener(m, 64, 10, a.iters, a.repeats) for m in models]
    res["batch1"] = [batch1(m, a.iters, a.repeats) for m in models + ["TCResNet8"]]
    eng = Engine(max_batch=8)
    res["kernels_n512"] = {m: kernels(m, 512, a.iters, eng) for m in models}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
