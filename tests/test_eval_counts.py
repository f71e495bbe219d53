"""Evaluation counts on the device (tcr_eval_accumulate and tcr_dscnn_eval_accumulate: eval_accumulate_kernel, csrc/tcr_metrics.cu)
against the reference's rules, restated in oracle/metrics_oracle.py: prediction and label = np.argmax, top-k hit = the label is
among np.argsort(-scores, kind="stable")[:, :k].  Every class count 1-32 the handles accept at its edges (1, 2, 5, 12, 16, 17,
32), top-k 1, 5, C - 1, C and C + 1, batches of 1, 255, 256, 257 and 1,000 rows accumulated into one counts buffer, and the
score rows where an arg-max or a rank can go wrong: ties, constant and saturated rows, +-0, subnormals, +-inf, NaN at the first,
a middle, the last and the true class, all-NaN rows and all-zero one-hot rows.  The counts are integers, so they must match bit
for bit; metrics_from_counts must equal the --host_metrics path on the same scores.  On the GPU also tcr_eval_rank past 2^24
(score, class) pairs, where its scan carries a total across blocks of chunk totals, and evaluate_audio.py on checkpoints whose
softmax is NaN in every row, which is what a diverged run gives."""
import ctypes as C
import re
import time
import warnings

import numpy as np
import pytest

import tcresnet_b200  # noqa: F401
from oracle import metrics_oracle as MO
from tcresnet_b200 import _lib as L
from tcresnet_b200.metrics.manager import AudioMetricManager, metrics_from_counts, topn_accuracy
from tcr_harness import Engine, NumpyBackend

CLASSES = (1, 2, 5, 12, 16, 17, 32)
BATCHES = (1, 255, 256, 257, 1000)        # one row, both sides of the kernel's 256-row block, several blocks with a partial one
PATTERNS = ("softmax", "ties", "constant", "saturated", "signed_zero", "subnormal", "inf", "nan_first", "nan_middle", "nan_last",
            "nan_true", "all_nan", "zero_onehot")
HANDLES = ("tcresnet", "dscnn")


def topks(c):
    return sorted({1, 5, c - 1, c, c + 1} - {0})


def softmax(z):
    z = np.asarray(z, np.float32)
    e = np.exp(z - z.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)


def rows(pattern, c, seed):
    """sum(BATCHES) score rows of `pattern` and their one-hot rows (np.eye(c)[labels], all zero for zero_onehot)."""
    rng = np.random.default_rng(seed)
    n = sum(BATCHES)
    labels = rng.integers(0, c, n)
    s = softmax(3 * rng.standard_normal((n, c)))
    i = np.arange(n)
    if pattern in ("ties", "zero_onehot"):           # four levels: ties at the top, at the k-th place and at the true class
        s = (rng.integers(0, 4, (n, c)) / 4).astype(np.float32)
        s[i[1::2], labels[1::2]] = s[1::2].max(1)    # and in every other row the true class ties with the maximum
    elif pattern == "constant":
        s = np.repeat(rng.random((n, 1), np.float32), c, 1)
    elif pattern == "saturated":                     # fp32 softmax of wide logits: 1.0, exact 0.0 and a few values between
        s = softmax(60 * rng.standard_normal((n, c)))
    elif pattern == "signed_zero":                   # +0.0 and -0.0 are equal: first maximum, ties by class index
        s = rng.choice(np.array([0.0, -0.0, -0.25], np.float32), (n, c))
    elif pattern == "subnormal":                     # 0 to 5 ulps of the smallest subnormal, either sign: all zero if flushed
        bits = rng.integers(0, 6, (n, c)).astype(np.uint32) | (rng.random((n, c)) < 0.2).astype(np.uint32) << 31
        s = bits.view(np.float32)
    elif pattern == "inf":
        s[rng.random((n, c)) < 0.3] = np.inf
        s[rng.random((n, c)) < 0.2] = -np.inf
    elif pattern == "nan_first":
        s[:, 0] = np.nan
    elif pattern == "nan_middle":
        s[:, c // 2] = np.nan
    elif pattern == "nan_last":
        s[:, c - 1] = np.nan
    elif pattern == "nan_true":                      # and in every other row a second NaN, before or after the true class
        s[i, labels] = np.nan
        s[i[1::2], rng.integers(0, c, len(i[1::2]))] = np.nan
    elif pattern == "all_nan":
        s[:] = np.nan
    hot = np.eye(c, dtype=np.float32)[labels]
    if pattern == "zero_onehot":
        hot[:] = 0.0
    return s, hot


class Counter:
    """tcr_eval_accumulate through a TC-ResNet handle, or tcr_dscnn_eval_accumulate through a DS-CNN-S handle at 49 x 10, with
    `classes` classes; counts(...) accumulates the batches into one device buffer."""

    def __init__(self, backend, classes, handle):
        self.b, self.lib, self.classes, self.handle = backend, backend.lib, classes, handle
        if handle == "dscnn":
            cfg = L.TcrDscnnConfig(size=ord("S"), height=49, width=10, num_classes=classes, max_batch=4, device=0)
            self.h = C.c_void_p()
            L.check(self.lib, self.lib.tcr_dscnn_create(C.byref(cfg), C.byref(self.h)), "tcr_dscnn_create")
            self.fn = self.lib.tcr_dscnn_eval_accumulate
        else:
            self.eng = Engine(backend, max_batch=4, num_classes=classes)
            self.h, self.fn = self.eng.h, self.lib.tcr_eval_accumulate

    def close(self):
        if self.handle == "dscnn":
            self.lib.tcr_dscnn_destroy(self.h)
        else:
            self.eng.close()

    def call(self, scores, hot, n, topk, counts):
        b = self.b
        ptr = counts.data_ptr() if b.name == "cuda" else counts.ctypes.data
        return self.fn(self.h, b.ptr(scores), b.ptr(hot), n, topk, ptr, b.stream)

    def counts(self, scores, hot, topk, batches=BATCHES):
        b, c = self.b, self.classes
        counts = b.torch.zeros(c * c + 2, dtype=b.torch.int64, device=b.dev) if b.name == "cuda" else np.zeros(c * c + 2, np.int64)
        at = 0
        for m in batches:
            L.check(self.lib, self.call(b.upload(scores[at:at + m]), b.upload(hot[at:at + m]), m, topk, counts), "eval_accumulate")
            at += m
        assert at == len(scores)
        b.sync()
        return counts.cpu().numpy() if b.name == "cuda" else counts


def host_metrics(scores, hot, c):
    names = [f"c{k}" for k in range(c)]
    host = AudioMetricManager(False, True, [])
    with warnings.catch_warnings(), np.errstate(all="ignore"):       # NaN and inf scores make the host's mAP keys NaN
        warnings.simplefilter("ignore")
        host.evaluate_and_aggregate_metrics(1, {"labels_onehot": hot, "predictions_onehot": scores, "label_names": names}, {})
    return host.get_evaluation_result(1)


def check_counts(counter, pattern):
    c = counter.classes
    scores, hot = rows(pattern, c, seed=PATTERNS.index(pattern) * 100 + c)
    labels = hot.argmax(1)
    for k in topks(c):
        got = counter.counts(scores, hot, k)
        ref = MO.eval_counts(scores, hot, k)
        assert np.array_equal(got, ref), (pattern, c, k, got[c * c:], ref[c * c:],
                                          np.argwhere(got[:c * c].reshape(c, c) != ref[:c * c].reshape(c, c)))
        if k >= c:                                   # topk >= classes counts every row
            assert got[c * c] == len(scores)
        if pattern == "all_nan":                     # np.argmax: class 0; np.argsort puts NaN last, in class order
            assert got[c * c] == (labels < k).sum() and got[:c * c].reshape(c, c)[:, 1:].sum() == 0
    assert got[c * c + 1] == len(scores) and got[:c * c].sum() == len(scores)


def check_host(counter, pattern):
    c = counter.classes
    scores, hot = rows(pattern, c, seed=PATTERNS.index(pattern) * 100 + c)
    dev = metrics_from_counts(counter.counts(scores, hot, 5), [f"c{k}" for k in range(c)], use_class_metrics=True)
    host = host_metrics(scores, hot, c)
    assert set(dev) <= set(host)
    for key, v in dev.items():
        if key == "confusion_matrix":
            assert np.array_equal(v, host[key])
        else:
            assert abs(v - host[key]) <= 1e-12, (key, v, host[key])
    assert abs(dev["top5_accuracy"] - topn_accuracy(hot, scores, 5)) <= 1e-12


def check_refusals(counter):
    b, c = counter.b, counter.classes
    s = b.upload(np.zeros((2, c), np.float32))
    counts = b.torch.zeros(c * c + 2, dtype=b.torch.int64, device=b.dev) if b.name == "cuda" else np.zeros(c * c + 2, np.int64)
    for n, topk in ((2, 0), (2, -1), (0, 5), (-1, 5)):
        assert counter.call(s, s, n, topk, counts) == 1, (n, topk)          # TCR_ERR_INVALID
    b.sync()
    assert not (counts.cpu().numpy() if b.name == "cuda" else counts).any()


@pytest.fixture(scope="module")
def emu_counters():
    backend, made = NumpyBackend(), {}

    def get(handle, classes):
        if (handle, classes) not in made:
            made[handle, classes] = Counter(backend, classes, handle)
        return made[handle, classes]
    yield get
    for counter in made.values():
        counter.close()


@pytest.fixture(scope="module")
def cuda_counters():
    from tcr_harness import TorchBackend
    backend, made = TorchBackend(), {}

    def get(handle, classes):
        if (handle, classes) not in made:
            made[handle, classes] = Counter(backend, classes, handle)
        return made[handle, classes]
    yield get
    for counter in made.values():
        counter.close()


# ------------------------------------------------------------------------------------------------------------ the oracle
def test_oracle_follows_np_argmax_and_argsort():
    """The restated rules on hand-worked rows: the first NaN is the arg-max, NaN ranks after every number, +0 == -0, and equal
    scores keep the lower class first."""
    nan, inf = np.nan, np.inf
    s = np.array([[1, nan, 2, nan], [nan, 3, 3, 1], [0.0, -0.0, -1, -inf], [1, 1, 1, 1], [nan, nan, nan, nan]], np.float32)
    assert np.argmax(s, 1).tolist() == [1, 0, 0, 0, 0]
    order = np.argsort(-s, axis=1, kind="stable").tolist()
    assert order == [[2, 0, 1, 3], [1, 2, 3, 0], [0, 1, 2, 3], [0, 1, 2, 3], [0, 1, 2, 3]]
    assert MO.top_k_hits(s, np.array([3, 0, 1, 3, 2]), 2).tolist() == [False, False, True, False, False]
    assert MO.top_k_hits(s, np.array([1, 3, 2, 2, 3]), 3).tolist() == [True, True, True, True, False]
    assert MO.top_k_hits(s, np.zeros(5, int), 5).all()                     # k >= classes: every row


# ------------------------------------------------------------------------------------------------------------ emulator
@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("classes", CLASSES)
@pytest.mark.parametrize("handle", HANDLES)
def test_emulated_counts_follow_the_reference_rules(emu_counters, handle, classes, pattern):
    check_counts(emu_counters(handle, classes), pattern)


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("classes", CLASSES)
@pytest.mark.parametrize("handle", HANDLES)
def test_emulated_count_metrics_equal_host_metrics(emu_counters, handle, classes, pattern):
    check_host(emu_counters(handle, classes), pattern)


@pytest.mark.parametrize("handle", HANDLES)
def test_emulated_refusals(emu_counters, handle):
    check_refusals(emu_counters(handle, 12))


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("classes", CLASSES)
@pytest.mark.parametrize("handle", HANDLES)
def test_cuda_counts_follow_the_reference_rules(cuda_counters, handle, classes, pattern):
    check_counts(cuda_counters(handle, classes), pattern)


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("classes", CLASSES)
@pytest.mark.parametrize("handle", HANDLES)
def test_cuda_count_metrics_equal_host_metrics(cuda_counters, handle, classes, pattern):
    check_host(cuda_counters(handle, classes), pattern)


@pytest.mark.gpu
@pytest.mark.parametrize("handle", HANDLES)
def test_cuda_refusals(cuda_counters, handle):
    check_refusals(cuda_counters(handle, 12))


@pytest.mark.gpu
def test_cuda_rank_past_2_to_the_24_pairs():
    """tcr_eval_rank over 1,400,000 x 12 = 16.8e6 (score, class) pairs: the exclusive scans then span more than 4,096 chunk totals,
    so scan_top_kernel carries a running total into a second block.  Against sklearn within 1e-12 (the samples average from
    ranking_vector), collected in uneven batches, and bit-identical to a single-batch collect."""
    from tcr_harness import TorchBackend
    from test_eval_ranking import Ranker, case, sklearn_vector
    n, classes = 1_400_000, 12
    assert n * classes > 2 ** 24 and (n * classes + 4095) // 4096 > 4096
    cycle, splits = (1, 255, 65_537, 4_890, 131_071, 7), []
    while sum(splits) < n:
        splits.append(min(cycle[len(splits) % len(cycle)], n - sum(splits)))
    scores, labels = case(np.random.default_rng(4), n, classes, "ties")
    r = Ranker(TorchBackend(), classes)
    try:
        t0 = time.perf_counter()
        got = r.run(scores, labels, splits)
        t1 = time.perf_counter()
        err = np.abs(got - sklearn_vector(scores, labels, classes, samples=False)).max()
        print(f"\n{n} x {classes} pairs in {len(splits)} batches: collected and ranked in {t1 - t0:.2f} s, "
              f"max error against sklearn {err:.3g}")
        assert err <= 1e-12
        assert np.array_equal(got, r.run(scores, labels))
    finally:
        r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("model,flags", [("TCResNet8Model", "--weight_decay 0.001 --width_multiplier 1.0"), ("DSCNNSModel", "")])
def test_evaluate_audio_on_a_diverged_checkpoint(tmp_path, monkeypatch, model, flags):
    """evaluate_audio.py on a checkpoint whose fc weights are NaN, so every softmax row is NaN (the fc and not an earlier layer:
    a NaN before a ReLU can vanish, since the kernels' fmaxf returns the other operand).  Every prediction is class 0 and the
    true class ranks at its own index, so top-5 is the share of labels below 5, on the device path as on --host_metrics."""
    from test_device_dataset import make_split
    from test_eval_ranking import _args
    from tcresnet_b200 import evaluate_audio
    from tcresnet_b200.common import checkpoint as ckpt
    from tcresnet_b200.factory import audio_nets
    make_split(tmp_path, "valid", per_label=3, seed=1)
    init = getattr(audio_nets, model)(_args(tmp_path, model, flags), None)
    init.build_inference(None, is_training=False)
    variables = init.get_variables()
    fc = [k for k in variables if re.search(r"/fc1?/weights$", k)]
    assert len(fc) == 1, sorted(variables)
    variables[fc[0]] = np.full_like(variables[fc[0]], np.nan)
    ckpt.save(tmp_path / "run", model, 1000, variables, fmt="tf")
    init.engine.close()
    seen = {}
    original = AudioMetricManager.evaluate_and_aggregate_metrics

    def spy(self, step, non_tensor_data, eval_dict):
        if non_tensor_data.get("predictions_onehot") is not None:
            seen["scores"], seen["hot"] = non_tensor_data["predictions_onehot"], non_tensor_data["labels_onehot"]
        return original(self, step, non_tensor_data, eval_dict)

    monkeypatch.setattr(AudioMetricManager, "evaluate_and_aggregate_metrics", spy)
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore")
        dev, host = (evaluate_audio.main(_args(tmp_path, model, flags, extra))[0] for extra in ("", "--host_metrics"))
    assert seen["scores"].size and np.isnan(seen["scores"]).all()
    labels = seen["hot"].argmax(1)
    assert dev["accuracy"] == host["accuracy"] and dev["top5_accuracy"] == host["top5_accuracy"]
    assert np.array_equal(dev["confusion_matrix"], host["confusion_matrix"])
    assert abs(dev["top5_accuracy"] - np.mean(labels < 5)) <= 1e-12 and dev["top5_accuracy"] < 1.0
    assert abs(dev["accuracy"] - np.mean(labels == 0)) <= 1e-12
