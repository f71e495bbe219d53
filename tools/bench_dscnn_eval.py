#!/usr/bin/env python
"""DS-CNN evaluation on one GPU: the reference's DSCNN{S,M,L}Model recipes' front-end (10 MFCCs, 40 / 20 ms windows: 49 x 10).

Evaluation forward: utterances/s of DsCnn.forward_input from int16 clips (front-end + network, the evaluate_audio.py path) at
n = 512, for S, M and L.  Listener: ms per push of 64 streams x 10 windows (hop 1 frame = 20 ms, 200 ms chunks), DS-CNN-S, eager
and replayed from a CUDA graph.  Warm-up, then `--repeats` rounds of `--iters` calls, each round timed with CUDA events; the result
is the median [min, max] over the rounds.  The card's name, power limit and maximum SM clock are read in the same run.

    python tools/bench_dscnn_eval.py [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import tcresnet_b200  # noqa: E402,F401
import torch  # noqa: E402
from bench_listener import card, timed  # noqa: E402
from tcresnet_b200.dscnn import DsCnn  # noqa: E402

FRONTEND = dict(num_mfccs=10, window_size_ms=40, window_stride_ms=20)


def rounds(fn, iters, repeats):
    timed(fn, max(3, iters // 5))
    ms = sorted(timed(fn, iters) for _ in range(repeats))
    return ms[len(ms) // 2], ms[0], ms[-1]


def evaluation(size, n, iters, repeats):
    d = DsCnn(size, 49, 10, 12, n).set_frontend(**FRONTEND)
    params = d.new_variables(seed=1)
    g = torch.Generator(device=d.device).manual_seed(0)
    pcm = torch.randint(-32768, 32768, (n, 16000), device=d.device, generator=g, dtype=torch.int32).to(torch.int16)
    logits, probs = torch.empty(n, 12, device=d.device), torch.empty(n, 12, device=d.device)
    med, lo, hi = rounds(lambda: d.forward_input(pcm, params, logits=logits, probs=probs), iters, repeats)
    d.close()
    return dict(size=size, n=n, utt_per_s=n / med * 1e3, ms=[med, lo, hi])


def listener(streams, windows, iters, repeats):
    d = DsCnn("S", 49, 10, 12, streams * windows).set_frontend(**FRONTEND)
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
    return dict(streams=streams, windows=windows, eager_ms=list(eager), graph_ms=list(replay),
                windows_per_s=streams * windows / replay[0] * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card(), evaluation=[evaluation(s, 512, a.iters, a.repeats) for s in ("S", "M", "L")],
               listener=listener(64, 10, a.iters, a.repeats))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
