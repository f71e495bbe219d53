#!/usr/bin/env python
"""Continuous-audio listener (tcr_listener_*) against the per-clip path, on one GPU.

Throughput: windows/s of Listener.push against Engine.forward on the same streams * K cut clips with the front-end included
(the way a caller scores a stream without the listener), TCResNet8-1.0 at T = 98 (30 / 10 ms front-end), 100 ms chunks.  The
two arms alternate in one process: warm-up, then `--repeats` rounds of `--iters` calls per arm, each timed with CUDA events;
the result is the median [min, max] over the rounds.  Latency: one stream, one push per call replayed from a CUDA graph, each
push timed with CUDA events.  The card's name, power limit and maximum SM clock are read in the same run.

    python tools/bench_listener.py [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import tcresnet_b200  # noqa: E402,F401
import torch  # noqa: E402
from tcresnet_b200.engine import Engine  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def throughput(streams, hop, iters, repeats):
    chunk = 1600
    K = chunk // (hop * 160)
    n = streams * K
    eng = Engine("TCResNet8", 1.0, window_size_ms=30, window_stride_ms=10, max_batch=n, dropout_keep_prob=1.0)
    params, _, moving = eng.new_variables(seed=1)
    lis = eng.listener(streams, hop, chunk, params, moving)
    g = torch.Generator(device=eng.device).manual_seed(0)
    x = torch.rand(streams, chunk, device=eng.device, generator=g) * 2 - 1
    clips = torch.rand(n, eng.cfg.clip_samples, device=eng.device, generator=g) * 2 - 1
    probs = torch.empty(streams, K, eng.num_classes, device=eng.device)
    arms = {"listener": lambda: lis.push(x, probs=probs),
            "per_clip": lambda: eng.forward(clips, params, moving)}
    for f in arms.values():
        timed(f, max(3, iters // 5))
    ms = {k: [] for k in arms}
    for _ in range(repeats):
        for k, f in arms.items():
            ms[k].append(timed(f, iters))
    lis.close()
    eng.close()
    out = dict(streams=streams, hop_frames=hop, windows_per_push=K, batch=n)
    for k, v in ms.items():
        rate = sorted(n / (t / 1e3) for t in v)
        out[k] = dict(windows_per_s=dict(median=rate[len(rate) // 2], min=rate[0], max=rate[-1]), ms_per_call=sorted(v))
    out["speedup_median"] = out["listener"]["windows_per_s"]["median"] / out["per_clip"]["windows_per_s"]["median"]
    return out


def latency(hop, pushes):
    """One stream, 100 ms chunks, the push replayed from a CUDA graph; every push timed with its own pair of events."""
    chunk = 1600
    eng = Engine("TCResNet8", 1.0, window_size_ms=30, window_stride_ms=10, max_batch=chunk // (hop * 160), dropout_keep_prob=1.0)
    params, _, moving = eng.new_variables(seed=1)
    lis = eng.listener(1, hop, chunk, params, moving)
    x = torch.rand(1, chunk, device=eng.device) * 2 - 1
    probs = torch.empty(1, lis.windows, eng.num_classes, device=eng.device)
    for _ in range(2):
        lis.push(x, probs=probs)
    s = torch.cuda.Stream(device=eng.device)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            lis.push(x, probs=probs)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(20):
        graph.replay()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(pushes)]
    for a, b in ev:
        a.record()
        graph.replay()
        b.record()
    torch.cuda.synchronize()
    t = sorted(a.elapsed_time(b) for a, b in ev)
    lis.close()
    eng.close()
    return dict(hop_frames=hop, windows_per_push=lis.windows, pushes=pushes,
                ms=dict(median=t[len(t) // 2], p10=t[len(t) // 10], p90=t[(9 * len(t)) // 10], min=t[0], max=t[-1]))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card(), throughput=[], latency=[])
    for S in (64, 512):
        for hop in (1, 2):
            r = throughput(S, hop, a.iters, a.repeats)
            print(json.dumps(r), flush=True)
            res["throughput"].append(r)
    for hop in (1, 2):
        r = latency(hop, 200)
        print(json.dumps(r), flush=True)
        res["latency"].append(r)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(dict(card=res["card"])))


if __name__ == "__main__":
    main()
