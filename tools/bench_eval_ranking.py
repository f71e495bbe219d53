#!/usr/bin/env python
"""The ranking metrics of one evaluation (per-class AP and mAP at macro / micro / weighted / samples) on one GPU, 12 classes, at
n = 4,890 (the Speech Commands test split), 10^5 and 10^6 utterances of softmax scores.

Device: collecting the n rows in batches of 500 (tcr_eval_collect) and, separately, the ranking pass (tcr_eval_rank) plus the one
D2H read of its 2 x 12 + 4 doubles.  Host: the D2H copy of the [n, 12] scores and labels plus sklearn.metrics.
average_precision_score at average=None and "micro" (the two rankings; macro and weighted follow from the per-class APs) and the
samples average vectorised in NumPy (sklearn's loops over the rows in Python and takes minutes at 10^6 rows), timed with a host
clock after a device synchronise.  Warm-up, then `--repeats` rounds; the result is the median [min, max] over the rounds.  The
device result is checked against sklearn's within 1e-12.  The card's name, power limit and maximum SM clock are read in the same run.

    python tools/bench_eval_ranking.py [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import tcresnet_b200  # noqa: E402,F401
import numpy as np  # noqa: E402
import torch  # noqa: E402
from sklearn.metrics import average_precision_score  # noqa: E402
from bench_dscnn_eval import rounds  # noqa: E402
from bench_listener import card  # noqa: E402
from tcresnet_b200.engine import Engine  # noqa: E402

CLASSES, BATCH = 12, 500


def sklearn_ranking(scores, labels):
    hot = np.eye(CLASSES)[labels]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        per_class = average_precision_score(hot, scores, average=None)
        micro = average_precision_score(hot, scores, average="micro")
    support = hot.sum(0)
    above = (scores >= scores[np.arange(len(labels)), labels][:, None]).sum(1)
    return np.concatenate([per_class, support, [per_class.mean(), micro, np.sum(per_class * support) / support.sum(),
                                                np.mean(1.0 / above)]])


def host_timed(fn, repeats):
    ms = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        ms.append((time.perf_counter() - t0) * 1e3)
    ms.sort()
    return ms[len(ms) // 2], ms[0], ms[-1]


def case(eng, n, iters, repeats):
    g = torch.Generator(device=eng.device).manual_seed(n)
    probs = torch.softmax(torch.randn(n, CLASSES, device=eng.device, generator=g) * 4, 1)
    probs[::5] = 1.0 / CLASSES                                          # tie groups
    labels = torch.randint(0, CLASSES, (n,), device=eng.device, generator=g)
    hot = torch.nn.functional.one_hot(labels, CLASSES).float()
    store = torch.empty(n, CLASSES, device=eng.device)
    store_labels = torch.empty(n, dtype=torch.int32, device=eng.device)
    ws = eng.eval_rank_workspace(n)

    def collect():
        for at in range(0, n, BATCH):
            m = min(BATCH, n - at)
            eng.eval_collect(probs[at:at + m], hot[at:at + m], store, store_labels, at)

    collect()
    got = eng.eval_rank(store, store_labels, n, ws).cpu().numpy()
    ref = sklearn_ranking(probs.cpu().numpy(), labels.cpu().numpy())
    err = float(np.abs(got - ref).max())
    assert err <= 1e-12, err
    c_ms = rounds(collect, iters, repeats)
    r_ms = host_timed(lambda: eng.eval_rank(store, store_labels, n, ws).cpu(), repeats)
    h_ms = host_timed(lambda: sklearn_ranking(probs.cpu().numpy(), store_labels.cpu().numpy()), max(3, repeats // 4))
    return dict(n=n, classes=CLASSES, workspace_mb=ws.numel() / 2 ** 20, max_abs_err_vs_sklearn=err,
                device_collect_ms=list(c_ms), device_rank_ms=list(r_ms), host_copy_and_sklearn_ms=list(h_ms),
                speedup_rank_vs_host=h_ms[0] / r_ms[0])


def main():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--sizes", type=int, nargs="*", default=[4890, 100_000, 1_000_000])
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--repeats", type=int, default=12)
    p.add_argument("--out", default=None)
    a = p.parse_args()
    eng = Engine(num_classes=CLASSES, max_batch=BATCH)
    res = dict(card=card(), cases=[case(eng, n, a.iters, a.repeats) for n in a.sizes])
    eng.close()
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
