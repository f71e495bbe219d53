"""Ranking metrics on the device (tcr_eval_collect / tcr_eval_rank and the tcr_dscnn_ twins): per-class AP and mAP at macro, micro,
weighted and samples against sklearn.metrics.average_precision_score, the reference's own library (metrics/ops/non_tensor_ops.py
:15-61, :296-343); on the CPU emulator and on the GPU, then through evaluate_audio.py on both evaluation paths."""
import ctypes as C
import shlex
import warnings

import numpy as np
import pytest
from sklearn.metrics import average_precision_score

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L
from tcresnet_b200.metrics.manager import AudioMetricManager, ranking_metrics, ranking_vector
from tcr_harness import Engine, NumpyBackend

AVERAGES = ("macro", "micro", "weighted", "samples")


def sklearn_vector(scores, labels, classes, samples=True):
    """tcr_eval_rank's layout from sklearn: per-class AP, positives, then the four averages.  samples=False takes the samples
    average from ranking_vector instead (sklearn loops over the rows in Python: minutes at 10^6 rows)."""
    hot = np.eye(classes)[labels]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                  # a class without positives warns and gets AP 0
        per_class = np.atleast_1d(average_precision_score(hot, scores, average=None))
        avg = [average_precision_score(hot, scores, average=a) if samples or a != "samples" else ranking_vector(hot, scores)[-1]
               for a in AVERAGES]
    return np.concatenate([per_class, hot.sum(0), avg])


def case(rng, n, classes, kind="plain"):
    scores = rng.random((n, classes)).astype(np.float32)
    scores /= scores.sum(1, keepdims=True)
    labels = rng.integers(0, classes, n)
    if kind == "ties":                                   # exact ties: constant rows and saturated softmax columns
        scores[::3] = np.float32(0.25)
        scores[:, 0] = (scores[:, 0] > 0.5 / classes).astype(np.float32)
        if classes > 2:
            scores[:, 2] = np.where(np.arange(n) % 2, 1.0, 0.0).astype(np.float32)
    if kind == "absent" and classes > 1:
        labels[labels == classes - 1] = 0
    return scores, labels


class Ranker:
    """Collect + rank through one handle: the TC-ResNet handle (tcr_eval_*) or the DS-CNN handle (tcr_dscnn_eval_*)."""

    def __init__(self, backend, classes, dscnn=False):
        self.b, self.lib, self.classes, self.dscnn = backend, backend.lib, classes, dscnn
        if dscnn:
            cfg = L.TcrDscnnConfig(size=ord("S"), height=49, width=10, num_classes=classes, max_batch=4, device=0)
            self.h = C.c_void_p()
            L.check(self.lib, self.lib.tcr_dscnn_create(C.byref(cfg), C.byref(self.h)), "tcr_dscnn_create")
        else:
            self.eng = Engine(backend, max_batch=4, num_classes=classes)
            self.h = self.eng.h
        pre = "tcr_dscnn_" if dscnn else "tcr_"
        self.collect_fn, self.rank_fn = getattr(self.lib, pre + "eval_collect"), getattr(self.lib, pre + "eval_rank")

    def close(self):
        if self.dscnn:
            self.lib.tcr_dscnn_destroy(self.h)
        else:
            self.eng.close()

    def _buf(self, a):
        if self.b.name == "cuda":
            return self.b.torch.from_numpy(np.ascontiguousarray(a)).to(self.b.dev)
        return np.ascontiguousarray(a).copy()

    def _ptr(self, t):
        return t.data_ptr() if self.b.name == "cuda" else t.ctypes.data

    def _get(self, t):
        return t.cpu().numpy() if self.b.name == "cuda" else t

    def workspace_bytes(self, n):
        nb = C.c_int64()
        st = self.rank_fn(self.h, None, None, n, None, C.byref(nb), None, self.b.stream)
        return st, nb.value

    def run(self, scores, labels, splits=None, capacity=None):
        """Collects the rows in batches of `splits` sizes, ranks the first n: the fp64 result [2C + 4]."""
        n, c = scores.shape
        capacity = capacity or n
        hot = np.eye(c, dtype=np.float32)[labels]
        store, store_labels = self._buf(np.full((capacity, c), np.nan, np.float32)), self._buf(np.full(capacity, -1, np.int32))
        at = 0
        for m in splits or [n]:
            s, h = self.b.upload(scores[at:at + m]), self.b.upload(hot[at:at + m])
            L.check(self.lib, self.collect_fn(self.h, self.b.ptr(s), self.b.ptr(h), m, at, capacity, self._ptr(store),
                                              self._ptr(store_labels), self.b.stream), "eval_collect")
            at += m
        assert at == n
        st, nb = self.workspace_bytes(n)
        L.check(self.lib, st, "eval_rank query")
        ws = self._buf(np.zeros(nb, np.uint8))
        out = self._buf(np.full(2 * c + 4, -1.0))
        nbc = C.c_int64(nb)
        L.check(self.lib, self.rank_fn(self.h, self._ptr(store), self._ptr(store_labels), n, self._ptr(ws), C.byref(nbc),
                                       self._ptr(out), self.b.stream), "eval_rank")
        self.b.sync()
        assert np.array_equal(self._get(store_labels)[:n], labels)
        return self._get(out).copy()


def check_against_sklearn(r, n, classes, kind, seed=0, splits=None):
    rng = np.random.default_rng(seed)
    scores, labels = case(rng, n, classes, kind)
    got = r.run(scores, labels, splits)
    ref = sklearn_vector(scores, labels, classes, samples=n <= 10_000)
    assert np.abs(got - ref).max() <= 1e-12, (n, classes, kind, got, ref)
    assert np.abs(ranking_vector(np.eye(classes)[labels], scores) - ref).max() <= 1e-12
    return scores, labels, got


def check_nan(r, classes):
    """A NaN score makes its class's AP, and the macro, micro and weighted averages and samples (its row) NaN; the rest stays."""
    rng = np.random.default_rng(7)
    scores, labels = case(rng, 39, classes)
    scores[5, 1 % classes] = np.nan
    got = r.run(scores, labels)
    c = classes
    assert np.isnan(got[1 % c]) and np.isnan(got[2 * c:]).all()
    others = [k for k in range(c) if k != 1 % c]
    assert np.isfinite(got[others]).all() and np.array_equal(got[c:2 * c], np.eye(c)[labels].sum(0))
    assert np.array_equal(np.isnan(got), np.isnan(ranking_vector(np.eye(c)[labels], scores)))


def check_splits(r):
    """The result depends only on the stored rows: bit-identical for any collect batches, and for a store larger than n."""
    rng = np.random.default_rng(3)
    scores, labels = case(rng, 300, 12, "ties")
    whole = r.run(scores, labels)
    assert np.array_equal(whole, r.run(scores, labels, [1, 38, 261]))
    assert np.array_equal(whole, r.run(scores, labels, [150] * 2, capacity=400))
    assert np.array_equal(whole, r.run(scores, labels, [7] * 42 + [6]))


def check_refusals(r, classes):
    n_max = (2 ** 31 - 1) // classes
    assert r.workspace_bytes(n_max)[0] == 0                      # the largest n is accepted (the query allocates nothing)
    for n in (0, -1, n_max + 1):
        st, _ = r.workspace_bytes(n)
        assert st == 1, n                                         # TCR_ERR_INVALID
    scores = r.b.upload(np.zeros((2, classes), np.float32))
    store = r._buf(np.zeros((4, classes), np.float32))
    labels = r._buf(np.zeros(4, np.int32))
    for at, m, cap in ((3, 2, 4), (-1, 2, 4), (0, 0, 4), (0, 2, n_max + 1)):
        st = r.collect_fn(r.h, r.b.ptr(scores), r.b.ptr(scores), m, at, cap, r._ptr(store), r._ptr(labels), r.b.stream)
        assert st == 1, (at, m, cap)
    nb = C.c_int64(16)                                            # a workspace smaller than the query's
    assert r.rank_fn(r.h, r._ptr(store), r._ptr(labels), 4, r._ptr(store), C.byref(nb), r._ptr(store), r.b.stream) == 1


# ------------------------------------------------------------------------------------------------------------ emulator
@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


@pytest.mark.parametrize("classes", [1, 2, 12, 32])
@pytest.mark.parametrize("n", [1, 3, 39, 5000])
@pytest.mark.parametrize("kind", ["plain", "ties", "absent"])
def test_emulated_rank_matches_sklearn(emu, classes, n, kind):
    if n == 5000 and kind != "ties" and classes != 32:
        pytest.skip("n = 5000 runs the heaviest cases only: ties at every class count, every kind at 32 classes")
    r = Ranker(emu, classes)
    try:
        check_against_sklearn(r, n, classes, kind, seed=n + classes)
    finally:
        r.close()


def test_emulated_dscnn_handle_ranks_like_the_tcresnet_handle(emu):
    r, d = Ranker(emu, 12), Ranker(emu, 12, dscnn=True)
    try:
        rng = np.random.default_rng(11)
        scores, labels = case(rng, 39, 12, "ties")
        assert np.array_equal(r.run(scores, labels), d.run(scores, labels, [3] * 13))
        check_against_sklearn(d, 39, 12, "absent", seed=2)
    finally:
        r.close()
        d.close()


@pytest.mark.parametrize("classes", [2, 12])
def test_emulated_nan_score(emu, classes):
    r = Ranker(emu, classes)
    try:
        check_nan(r, classes)
    finally:
        r.close()


def test_emulated_collect_splits_are_bit_identical(emu):
    r = Ranker(emu, 12)
    try:
        check_splits(r)
    finally:
        r.close()


@pytest.mark.parametrize("classes", [1, 12, 32])
def test_emulated_refusals(emu, classes):
    for dscnn in (False, True):
        r = Ranker(emu, classes, dscnn)
        try:
            check_refusals(r, classes)
        finally:
            r.close()


# ------------------------------------------------------------------------------------------------------------ host side
def test_ranking_metrics_keys_and_the_host_path():
    rng = np.random.default_rng(5)
    scores, labels = case(rng, 500, 12, "ties")
    hot = np.eye(12, dtype=np.float32)[labels]
    names = [f"c{i}" for i in range(12)]
    ref = sklearn_vector(scores, labels, 12)
    keys = ranking_metrics(ref, names, use_class_metrics=True)
    assert [k for k in keys if k.startswith("mAP/")] == [f"mAP/{a}" for a in AVERAGES]
    assert all(keys[f"ap/c{k}"] == ref[k] for k in range(12))
    assert set(ranking_metrics(ref, names)) == {f"mAP/{a}" for a in AVERAGES}
    host = AudioMetricManager(False, True, ["mAP/samples", "ap/c3"])
    host.evaluate_and_aggregate_metrics(1, {"labels_onehot": hot, "predictions_onehot": scores, "label_names": names}, {})
    got = host.get_evaluation_result(1)
    assert "mAP" in got and "mAP/samples" not in got and "ap/c3" not in got
    for k in ("mAP/macro", "mAP/micro", "mAP/weighted", "ap/c0", "ap/c11"):
        assert abs(got[k] - keys[k]) <= 1e-12, k
    lines = []
    host.log_metrics(1, log=lines.append)
    assert "mAP/macro" in lines[0] and "mAP/micro" in lines[0] and "ap/c0" not in lines[0] and "precision/" not in lines[0]
    assert host.get_best_keep_metric_with_modes() == {"accuracy": "max"}


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


@pytest.mark.gpu
@pytest.mark.parametrize("classes", [1, 2, 12, 32])
@pytest.mark.parametrize("n", [1, 3, 39, 5000])
@pytest.mark.parametrize("kind", ["plain", "ties", "absent"])
def test_cuda_rank_matches_sklearn(cuda, classes, n, kind):
    r = Ranker(cuda, classes, dscnn=kind == "absent")
    try:
        check_against_sklearn(r, n, classes, kind, seed=n + classes)
    finally:
        r.close()


@pytest.mark.gpu
def test_cuda_rank_a_million_rows(cuda):
    """n = 10^6 x 12 classes: against sklearn (the samples average against ranking_vector, which the smaller cases pin to sklearn),
    and bit-identical when collected in 4,890-row batches."""
    r = Ranker(cuda, 12)
    try:
        scores, labels, whole = check_against_sklearn(r, 1_000_000, 12, "ties", seed=1)
        splits = [4890] * (1_000_000 // 4890) + [1_000_000 % 4890]
        assert np.array_equal(whole, r.run(scores, labels, splits))
    finally:
        r.close()


@pytest.mark.gpu
def test_cuda_nan_splits_and_refusals(cuda):
    for classes in (2, 12):
        r = Ranker(cuda, classes)
        try:
            check_nan(r, classes)
            check_refusals(r, classes)
        finally:
            r.close()
    r = Ranker(cuda, 12)
    try:
        check_splits(r)
    finally:
        r.close()


def _args(tmp_path, model, flags, extra="", checkpoint="run"):
    from tcresnet_b200 import evaluate_audio
    return evaluate_audio.parse_arguments(shlex.split(
        f"--dataset_path {tmp_path} --dataset_split_name valid --output_name output/softmax --num_classes 12 --num_silent 5 "
        f"--checkpoint_path {tmp_path}/{checkpoint} --augmentation_method anchored_slice_or_pad --preprocess_method mfcc "
        f"--num_mfccs 40 --clip_duration_ms 1000 --window_size_ms 40 --window_stride_ms 20 --background_frequency 0.0 "
        f"--background_max_volume 0.0 --batch_size 4 --no-shuffle --valid_type once --no-save_best_keeper --maximum_num_labels_for_metric 100 "
        f"{extra} {model} {flags}"))


@pytest.mark.gpu
@pytest.mark.parametrize("model,flags", [("TCResNet8Model", "--weight_decay 0.001 --width_multiplier 1.0"), ("DSCNNSModel", "")])
def test_evaluate_audio_device_and_host_rankings_agree_with_sklearn(tmp_path, monkeypatch, model, flags):
    """evaluate_audio.py on a small split with seeded weights: the device path's mAP/* and ap/* equal the --host_metrics path's and
    sklearn's on the softmax the host path received; --device_dataset (TC-ResNet) gives the device path's results bit for bit; the
    count metrics are those of the host path."""
    from test_device_dataset import make_split
    from tcresnet_b200 import evaluate_audio
    from tcresnet_b200.common import checkpoint as ckpt
    from tcresnet_b200.factory import audio_nets
    make_split(tmp_path, "valid", per_label=3, seed=1)
    init = getattr(audio_nets, model)(_args(tmp_path, model, flags), None)
    init.build_inference(None, is_training=False)
    ckpt.save(tmp_path / "run", model, 1000, init.get_variables(), fmt="tf")
    init.engine.close()
    seen = {}
    original = AudioMetricManager.evaluate_and_aggregate_metrics

    def spy(self, step, non_tensor_data, eval_dict):
        if non_tensor_data.get("predictions_onehot") is not None:
            seen["scores"], seen["hot"] = non_tensor_data["predictions_onehot"], non_tensor_data["labels_onehot"]
        return original(self, step, non_tensor_data, eval_dict)

    monkeypatch.setattr(AudioMetricManager, "evaluate_and_aggregate_metrics", spy)
    extras = ("", "--host_metrics", "--device_dataset") if model == "TCResNet8Model" else ("", "--host_metrics")
    runs = {extra: evaluate_audio.main(_args(tmp_path, model, flags, extra))[0] for extra in extras}
    dev, host = runs[""], runs["--host_metrics"]
    ref = sklearn_vector(seen["scores"].astype(np.float32), seen["hot"].argmax(1), 12)
    names = [k for k in dev if k.startswith("mAP/") or k.startswith("ap/")]
    assert len(names) == 4 + 12
    for k in names:
        assert abs(dev[k] - host[k]) <= 1e-12, k
    for a, v in zip(AVERAGES, ref[24:]):
        assert abs(dev[f"mAP/{a}"] - v) <= 1e-12, a
    assert np.abs(np.array([dev[k] for k in names if k.startswith("ap/")]) - ref[:12]).max() <= 1e-12
    assert dev["accuracy"] == host["accuracy"] and np.array_equal(dev["confusion_matrix"], host["confusion_matrix"])
    assert "mAP" in host and "mAP" not in dev
    if "--device_dataset" in runs:
        dd = runs["--device_dataset"]
        assert set(dd) == set(dev) and all(np.array_equal(np.asarray(dd[k]), np.asarray(dev[k])) for k in dev)
