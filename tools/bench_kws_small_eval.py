#!/usr/bin/env python
"""KWSModel's speech_commands nets (--architecture low_latency_conv / tiny_conv) evaluation on one GPU, at 49 x 40 (40 MFCCs,
40 / 20 ms windows), with tools/bench_kws_eval.py's measurements: the evaluation forward in utterances/s from int16 clips at
n = 512, ms per launch of each kernel from the library's launch profiler in a separate pass, a listener push of 64 streams x 10
windows (eager and graph-replayed), and the batch-1 deployable model.  Each compute kernel is set against its FP32 FMA floor (the
useful FLOPs at the FP32 peak tcr_measure_fp32_peak measures in the same run) and its HBM floor (bytes it must move at the data
sheet's 3.35 TB/s).  Median [min, max] over `--repeats` rounds.  The card's name, power limit and maximum SM clock are read in the
same run.

    python tools/bench_kws_small_eval.py [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import tcresnet_b200  # noqa: E402,F401
from bench_kws_eval import batch1, evaluation, kernels, listener  # noqa: E402
from bench_listener import card  # noqa: E402
from tcresnet_b200.engine import Engine  # noqa: E402

ARCHS = ["low_latency_conv", "tiny_conv"]
HBM_TBPS = 3.35                          # H100 SXM data sheet
N = 512
# per utterance at 49 x 40, 12 classes: (kernel, useful FLOPs, bytes it must move) -- low_latency_conv: W = 33 columns, K = 6,138;
# tiny_conv: 25 x 20 x 8 outputs, K = 4,000
FLOORS = {
    "low_latency_conv": [("kws_llconv", 2 * 33 * 392 * 186, (49 * 40 + 33 * 186) * 4),
                         ("kws_fcs", 2 * 6138 * 128, 6138 * 4)],
    "tiny_conv": [("kws_tinyconv", 2 * 25 * 20 * 80 * 8, (49 * 40 + 4000) * 4),
                  ("kws_fcs", 2 * 4000 * 12, 4000 * 4)],
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card())
    res["evaluation"] = [evaluation(arch, N, a.iters, a.repeats) for arch in ARCHS]
    res["listener"] = [listener(arch, 64, 10, a.iters, a.repeats) for arch in ARCHS]
    res["batch1"] = [batch1(arch, a.iters, a.repeats) for arch in ARCHS]
    eng = Engine(max_batch=8)
    time.sleep(1.0)
    res["fp32_peak_tflops"] = peak = eng.fp32_peak_tflops()
    res["kernels_ms"] = {arch: kernels(arch, N, a.iters, eng) for arch in ARCHS}
    res["floors"] = {}
    for arch in ARCHS:
        for name, flops, nbytes in FLOORS[arch]:
            ms = res["kernels_ms"][arch].get(name)
            fma = flops * N / (peak * 1e12) * 1e3
            hbm = nbytes * N / (HBM_TBPS * 1e12) * 1e3
            res["floors"][f"{arch}/{name}"] = dict(kernel_ms=ms, fp32_fma_ms=fma, hbm_ms=hbm,
                                                   tflops=flops * N / (ms * 1e-3) / 1e12 if ms else None,
                                                   fraction_of_fma_floor=fma / ms if ms else None,
                                                   fraction_of_binding_floor=max(fma, hbm) / ms if ms else None)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
