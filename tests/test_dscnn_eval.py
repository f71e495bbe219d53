"""DS-CNN evaluation from audio (tcr_dscnn_set_frontend, tcr_dscnn_mfcc_forward, tcr_dscnn_forward_input,
tcr_dscnn_eval_accumulate) and the DSCNN{S,M,L}Model surface: the front-end features against a TC-ResNet handle's tcr_mfcc_forward
bit for bit, the forward from wav against the forward on those features bit for bit and against the fp64 oracle (tcr_oracle's
front-end -> dscnn_oracle).  The FMA kernels on the CPU emulator; every kernel path, S / M / L and evaluate_audio.py end to end on
the GPU."""
import ctypes as C
import shlex

import numpy as np
import pytest

from oracle import dscnn_oracle as D
from oracle import tcr_oracle as O
from tcr_harness import Engine, NumpyBackend, launched

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L

# front-end flags (tcr_config fields) of the cases: the recipes' 10 MFCCs at 40 / 20 ms (the frame-pair window / stride), the
# 40-coefficient shape of TC-ResNet's baseline, 30 / 10 ms windows, and log-mel
FRONTENDS = {
    "49x10": dict(num_mfccs=10),
    "49x40": dict(),
    "98x40": dict(window_size_samples=480, window_stride_samples=160),
    "49x40-logmel": dict(feature_kind=L.TCR_FEATURE_LOG_MEL, num_mel_bins=40),
}


class Ds:
    """A DS-CNN handle with a front-end, through the C ABI, over a tests/tcr_harness backend, with seeded oracle variables whose
    BatchNorm statistics are non-trivial (dscnn_oracle.init_variables)."""

    def __init__(self, b, size, frontend, max_batch, seed=0, classes=12):
        self.b, self.lib = b, b.lib
        c = L.TcrConfig()
        L.check(self.lib, self.lib.tcr_config_default(C.byref(c)), "tcr_config_default")
        for k, v in frontend.items():
            setattr(c, k, v)
        c.num_classes = classes
        self.cfg = c
        T = 1 + (c.clip_samples - c.window_size_samples) // c.window_stride_samples
        F = c.num_mfccs if c.feature_kind == L.TCR_FEATURE_MFCC else c.num_mel_bins
        self.T, self.F, self.classes, self.size = T, F, classes, size
        self.info = type("Info", (), dict(frames=T, features=F))
        self.h = C.c_void_p()
        L.check(self.lib, self.lib.tcr_dscnn_create(C.byref(L.TcrDscnnConfig(ord(size), T, F, classes, max_batch, 0)), C.byref(self.h)),
                "tcr_dscnn_create")
        L.check(self.lib, self.lib.tcr_dscnn_set_frontend(self.h, C.byref(c)), "tcr_dscnn_set_frontend")
        self.spec = D.build_spec(size, T, F, classes)
        self.p64 = D.init_variables(self.spec, seed)
        self.flat = D.flatten(self.spec, self.p64)
        self.params = b.upload(self.flat)

    def close(self):
        if self.h:
            self.lib.tcr_dscnn_destroy(self.h)
            self.h = C.c_void_p()

    def mfcc(self, wav):
        b = self.b
        n = wav.shape[0]
        x, feat = b.upload(wav), b.empty(n, self.T, self.F)
        kind = L.TCR_INPUT_WAV_PCM16 if wav.dtype == np.int16 else L.TCR_INPUT_WAV_F32
        L.check(self.lib, self.lib.tcr_dscnn_mfcc_forward(self.h, b.ptr(x), kind, b.ptr(feat), n, b.stream), "tcr_dscnn_mfcc_forward")
        b.sync()
        return b.download(feat)

    def forward_input(self, x, kind):
        b = self.b
        n = x.shape[0]
        d = b.upload(x)
        logits, probs = b.empty(n, self.classes), b.empty(n, self.classes)
        L.check(self.lib, self.lib.tcr_dscnn_forward_input(self.h, b.ptr(d), kind, b.ptr(self.params), n, b.ptr(logits), b.ptr(probs),
                                                           b.stream), "tcr_dscnn_forward_input")
        b.sync()
        return b.download(logits), b.download(probs)

    def wav_forward(self, wav):
        return self.forward_input(wav, L.TCR_INPUT_WAV_PCM16 if wav.dtype == np.int16 else L.TCR_INPUT_WAV_F32)

    def oracle_logits(self, wav):
        """fp64: tcr_oracle's front-end (datasets/preprocessors.py) -> dscnn_oracle's forward."""
        c = self.cfg
        x = wav.astype(np.float64) / 32768.0 if wav.dtype == np.int16 else wav.astype(np.float64)
        kw = dict(num_mel_bins=c.num_mel_bins, sample_rate=c.sample_rate, lower_edge_hertz=c.lower_edge_hertz,
                  upper_edge_hertz=c.upper_edge_hertz)
        if c.feature_kind == L.TCR_FEATURE_MFCC:
            feat = O.mfcc(x, c.window_size_samples, c.window_stride_samples, num_mfccs=c.num_mfccs, **kw)
        else:
            feat = O.log_mel_spectrogram(x, c.window_size_samples, c.window_stride_samples, magnitude_squared=False, **kw)
        return D.forward(self.spec, self.p64, feat)


def clips(n, samples=16000, seed=0, pcm=False):
    rng = np.random.default_rng(seed)
    if pcm:
        return rng.integers(-32768, 32768, (n, samples)).astype(np.int16)
    x = rng.uniform(-1.0, 1.0, (n, samples)).astype(np.float32)
    x[::2, : samples // 3] *= np.float32(0.01)            # quiet and loud stretches
    return x


def check_parity(ds, wav, rows=None):
    """forward_input(wav) == forward(features) bit for bit on every row; against the fp64 oracle (on `rows`) within 1e-4 of
    max |logit|, and the same arg-max wherever the oracle's top-2 margin exceeds that error.  Returns the relative error."""
    logits, probs = ds.wav_forward(wav)
    feat = ds.mfcc(wav)
    f_logits, f_probs = ds.forward_input(feat, L.TCR_INPUT_FEATURES)
    assert np.array_equal(logits, f_logits) and np.array_equal(probs, f_probs)
    rows = np.arange(wav.shape[0]) if rows is None else rows
    ref = ds.oracle_logits(wav[rows])
    err = np.abs(logits[rows] - ref).max()
    rel = float(err / np.abs(ref).max())
    assert rel <= 1e-4, rel
    top2 = np.sort(ref, axis=1)[:, -2:]
    clear = (top2[:, 1] - top2[:, 0]) > 2 * err
    assert np.array_equal(logits[rows][clear].argmax(1), ref[clear].argmax(1))
    return rel


@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


@pytest.mark.parametrize("case", list(FRONTENDS))
def test_frontend_features_equal_the_tcresnet_front_end(emu, case):
    """The DS-CNN handle's front-end is the TC-ResNet handle's: same tables, same kernel choice, bit-identical features.  A TC-ResNet
    handle needs a multiple of 4 coefficients, so the 10-MFCC case is compared against the first 10 of 12: every coefficient is
    its own DCT row dot product, the same sums whatever the count."""
    fe = FRONTENDS[case]
    ds = Ds(emu, "S", fe, 3)
    tc_fe = dict(fe, num_mfccs=12) if fe.get("num_mfccs") == 10 else fe
    eng = Engine(emu, max_batch=3, **tc_fe)
    try:
        for pcm in (False, True):
            wav = clips(3, seed=1, pcm=pcm)
            got = ds.mfcc(wav)
            ref = eng.mfcc(wav)[..., :ds.F]
            assert got.shape == (3, ds.T, ds.F) and np.array_equal(got, ref)
    finally:
        eng.close()
        ds.close()


@pytest.mark.parametrize("case", list(FRONTENDS))
def test_emulated_wav_forward_matches_features_and_oracle(emu, case):
    ds = Ds(emu, "S", FRONTENDS[case], 2, seed=3)
    try:
        assert check_parity(ds, clips(2, seed=2)) < 1e-5
        assert check_parity(ds, clips(2, seed=4, pcm=True)) < 1e-5
    finally:
        ds.close()


def test_emulated_eval_counts(emu):
    """tcr_dscnn_eval_accumulate is tcr_eval_accumulate's kernel: the same counts as the host's arg-max / rank rules."""
    ds = Ds(emu, "S", FRONTENDS["49x10"], 4)
    try:
        rng = np.random.default_rng(0)
        scores = rng.normal(size=(37, 12)).astype(np.float32)
        scores[3] = scores[3, 0]                                       # a tie: the first maximum wins
        hot = np.eye(12, dtype=np.float32)[rng.integers(0, 12, 37)]
        counts = np.zeros(12 * 12 + 2, np.int64)
        d_s, d_h = emu.upload(scores), emu.upload(hot)
        for _ in range(2):                                             # accumulated
            L.check(emu.lib, emu.lib.tcr_dscnn_eval_accumulate(ds.h, emu.ptr(d_s), emu.ptr(d_h), 37, 5, counts.ctypes.data, None), "acc")
        y, p = hot.argmax(1), scores.argmax(1)
        cm = np.zeros((12, 12), np.int64)
        np.add.at(cm, (y, p), 2)
        rank = np.array([(scores[i] > scores[i, y[i]]).sum() + (scores[i, :y[i]] == scores[i, y[i]]).sum() for i in range(37)])
        assert np.array_equal(counts[:144].reshape(12, 12), cm)
        assert counts[144] == 2 * (rank < 5).sum() and counts[145] == 74
    finally:
        ds.close()


def _err(lib):
    return lib.tcr_last_error().decode()


def test_refusals(emu):
    lib = emu.lib
    h = C.c_void_p()
    L.check(lib, lib.tcr_dscnn_create(C.byref(L.TcrDscnnConfig(ord("S"), 49, 10, 12, 4, 0)), C.byref(h)), "create")
    try:
        c = L.TcrConfig()
        lib.tcr_config_default(C.byref(c))                             # 49 x 40 MFCCs
        assert lib.tcr_dscnn_set_frontend(h, C.byref(c)) == 1
        assert "(T, F) = (49, 40)" in _err(lib) and "(height, width) = (49, 10)" in _err(lib)
        c.num_mfccs, c.window_size_samples, c.window_stride_samples = 10, 480, 160
        assert lib.tcr_dscnn_set_frontend(h, C.byref(c)) == 1 and "(T, F) = (98, 10)" in _err(lib)
        c.window_size_samples = 642
        assert lib.tcr_dscnn_set_frontend(h, C.byref(c)) == 3 and "multiples of 4" in _err(lib)   # tcr_create's refusals
        wav = np.zeros((1, 16000), np.float32)
        out = np.zeros(12, np.float32)
        assert lib.tcr_dscnn_forward_input(h, wav.ctypes.data, L.TCR_INPUT_WAV_F32, out.ctypes.data, 1, None, None, None) == 1
        assert "no front-end" in _err(lib)
        cfg = L.TcrListenerConfig(1, 1, 320)
        lis = C.c_void_p()
        assert lib.tcr_dscnn_listener_create(h, C.byref(cfg), C.byref(lis)) == 1 and "no front-end" in _err(lib)
        c.window_size_samples, c.window_stride_samples = 640, 320
        assert lib.tcr_dscnn_set_frontend(h, C.byref(c)) == 0
        assert lib.tcr_dscnn_forward_input(h, wav.ctypes.data, 7, out.ctypes.data, 1, None, None, None) == 1
        assert "unknown input kind 7" in _err(lib)
        assert lib.tcr_dscnn_forward_input(h, wav.ctypes.data, 0, out.ctypes.data, 5, None, None, None) == 1   # n > max_batch
        assert lib.tcr_dscnn_set_frontend(None, C.byref(c)) == 1
    finally:
        lib.tcr_dscnn_destroy(h)


def test_training_a_dscnn_recipe_still_raises():
    """train_audio.py on the reference's DS-CNN-S training line builds the model and stops there: training is out of scope."""
    from tcresnet_b200 import train_audio
    from tcresnet_b200.factory import audio_nets
    from tcresnet_b200.runtime import Node
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    line = [x for x in open(os.path.join(root, "tests", "golden", "reference_recipes.txt"))
            if x.startswith("python train_audio.py") and x.rstrip().endswith("DSCNNSModel")][0]
    args = train_audio.parse_arguments(shlex.split(line)[2:])
    assert args.model == "DSCNNSModel" and args.weight_decay == 0.0
    model = audio_nets.DSCNNSModel(args, None)
    with pytest.raises(NotImplementedError, match="training DS-CNN is out of scope.*evaluation"):
        model.build(Node("wav", [None, 16000, 1]), Node("labels", [None, 12]), is_training=True)


# ---------------------------------------------------------------------------------------------------------------- GPU
MODES = {"fma": "0", "lockstep": "1", "default": None}


@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("size", ["S", "M", "L"])
@pytest.mark.parametrize("case", ["49x10", "49x40"])
def test_cuda_wav_forward_matches_features_and_oracle(cuda, monkeypatch, case, size, mode):
    """n = 1, 3, 39 and 512 from fp32 and int16 clips, in each TCR_DSCNN_TC mode (conv_1 on dscnn_conv, dscnn_conv_tc or
    dscnn_conv_ws for S; M and L always run dscnn_conv).  The oracle is checked on 40 rows of each batch."""
    if MODES[mode] is None:
        monkeypatch.delenv("TCR_DSCNN_TC", raising=False)
    else:
        monkeypatch.setenv("TCR_DSCNN_TC", MODES[mode])
    ds = Ds(cuda, size, FRONTENDS[case], 512, seed=5)
    try:
        for n, pcm in ((1, False), (3, True), (39, False), (512, True)):
            wav = clips(n, seed=n, pcm=pcm)
            rows = np.unique(np.r_[np.arange(min(n, 32)), np.arange(max(0, n - 8), n)])
            assert check_parity(ds, wav, rows) < 1e-5
        if size == "S":
            conv = {"fma": "dscnn_conv", "lockstep": "dscnn_conv_tc", "default": "dscnn_conv_ws"}[mode]
            got = launched(cuda.lib, lambda: ds.wav_forward(clips(3)))
            assert got[conv] == 1, got
    finally:
        ds.close()


def _recipe_args(extra, model="DSCNNSModel"):
    return ("--output_name output/softmax --num_classes 12 --preprocess_method mfcc --num_mfccs 10 --clip_duration_ms 1000 "
            f"--window_size_ms 40 --window_stride_ms 20 {extra} {model}")


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["DSCNNSModel", "DSCNNLModel"])
def test_deployed_model_replay_matches_the_eager_call(cuda, model):
    """build_deployable_model: batch 1, two eager calls then CUDA-graph replay; every call equals forward_input on the clip."""
    import torch
    from tcresnet_b200 import evaluate_audio
    from tcresnet_b200.factory import audio_nets
    args = evaluate_audio.parse_arguments(shlex.split(_recipe_args("--dataset_path synthetic:8 --dataset_split_name valid "
                                                                   "--checkpoint_path x --batch_size 1 --augmentation_method anchored_slice_or_pad", model)))
    m = getattr(audio_nets, model)(args, None)
    _, dep = m.build_deployable_model(include_preprocess=True)
    for i in range(5):
        x = clips(1, seed=10 + i)
        got = dep(x)
        ref = m.engine.forward_input(torch.from_numpy(x).cuda(), m.params)[1].cpu().numpy()
        assert np.array_equal(got, ref), i
    assert dep._graph is not None
    m.engine.close()


@pytest.mark.gpu
def test_evaluate_audio_on_a_dscnn_checkpoint_counts_the_oracles_predictions(tmp_path):
    """The reference's DS-CNN-S evaluation recipe (--batch_size 3, --valid_type once) on a small on-disk split and a TF-V2 bundle of
    seeded weights with non-trivial moving statistics under the reference's variable names: the confusion matrix and accuracy
    equal the counts of the fp64 oracle's arg-max on the same clips."""
    from test_device_dataset import make_split
    from tcresnet_b200 import evaluate_audio
    from tcresnet_b200.common import checkpoint as ckpt
    from tcresnet_b200.datasets.audio_data_wrapper import SingleLabelAudioDataWrapper
    from tcresnet_b200.runtime import Session
    make_split(tmp_path, "valid", per_label=3, seed=2)
    spec = D.build_spec("S", 49, 10, 12)
    values = D.init_variables(spec, 11)
    path = ckpt.save(tmp_path / "run", "DSCNNSModel", 1000, {k: v.astype(np.float32) for k, v in values.items()}, fmt="tf")
    args = evaluate_audio.parse_arguments(shlex.split(_recipe_args(
        f"--dataset_path {tmp_path} --dataset_split_name valid --checkpoint_path {path} --num_silent 6 "
        "--augmentation_method anchored_slice_or_pad --background_frequency 0.0 --background_max_volume 0.0 --batch_size 3 "
        "--no-shuffle --valid_type once --no-save_best_keeper")))
    results = evaluate_audio.main(args)
    assert len(results) == 1
    got = results[0]
    # the same clips, in the same order, from the same wrapper; the oracle's predictions
    args2 = evaluate_audio.parse_arguments(shlex.split(_recipe_args(
        f"--dataset_path {tmp_path} --dataset_split_name valid --checkpoint_path {path} --num_silent 6 "
        "--augmentation_method anchored_slice_or_pad --background_frequency 0.0 --background_max_volume 0.0 --batch_size 3 "
        "--no-shuffle --valid_type once --no-save_best_keeper")))
    session = Session()
    ds = SingleLabelAudioDataWrapper(args2, session, "valid", False)
    ds.get_input_and_output_op()
    ds.setup_iterator(session, ds.placeholders, ds.data)
    cm = np.zeros((12, 12))
    w64 = {k: np.asarray(v, np.float64) for k, v in ckpt.load(path).items() if k in spec.var_shapes}
    for _ in range(ds.num_samples // 3):
        wav, hot = ds.next_batch()
        feat = O.mfcc(wav[..., 0].astype(np.float64), 640, 320, num_mfccs=10)
        ref = D.forward(spec, w64, feat)
        top2 = np.sort(ref, axis=1)[:, -2:]
        assert (top2[:, 1] - top2[:, 0]).min() > 1e-4 * np.abs(ref).max()      # no near-tie: the arg-max is well defined
        np.add.at(cm, (hot.argmax(1), ref.argmax(1)), 1)
    assert np.array_equal(np.asarray(got["confusion_matrix"]), cm)
    assert got["accuracy"] == np.trace(cm) / cm.sum()
    assert np.isfinite(got["total_loss"])
