"""The front-end and the training step away from the two recipe geometries, against the fp64 oracle.

tcr_create accepts FFT lengths 128..2048, up to 128 mel bins, any multiple of 4 coefficients up to the mel count, any mel edges,
MFCC or log-mel features, 1..32 classes and any clip length; the frame count T follows from clip, window and stride.  Each
table below runs twice: on the emulator at n <= 8 (kernel logic on a CPU box) and with -m gpu on the sm_90a build at
production batches, where the resident planner sizes its shared-memory layout for ceil(max_batch / #SMs) utterances per CTA.
"""
import argparse

import numpy as np
import pytest

from oracle import tcr_oracle as O
from parity_cases import check_eval, check_step, perturbed_variables, reference_features, run_case, spectral_lines
from tcr_harness import Engine, NumpyBackend, launched, rel_err

BASE = dict(sample_rate=16000, clip=16000, window=640, stride=320, mel=64, mfcc=40, lower=80.0, upper=7600.0, feature_kind=0)


def geometry(**kw):
    return dict(BASE, **kw)


def engine_cfg(g):
    return dict(sample_rate=g["sample_rate"], clip_samples=g["clip"], window_size_samples=g["window"],
                window_stride_samples=g["stride"], num_mel_bins=g["mel"], num_mfccs=g["mfcc"], lower_edge_hertz=g["lower"],
                upper_edge_hertz=g["upper"], feature_kind=g["feature_kind"])


def ref_args(g):
    return g["window"], g["stride"], g["sample_rate"], g["mel"], g["mfcc"], g["lower"], g["upper"], g["feature_kind"]


@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


# ------------------------------------------------------------------------------------------------------------------------
# Front-end
# ------------------------------------------------------------------------------------------------------------------------

FRONT_END = {
    "fft512-400-160": geometry(window=400, stride=160),                                  # 25/10 ms: FFT 512, T=98
    "fft2048-T23": geometry(window=1600, stride=640),                                    # mfcc_kernel<1024>: separate spectrum
    "fft256-40-20": geometry(window=256, stride=128, mel=40, mfcc=20, lower=20.0, upper=8000.0),
    "fft128-32-12": geometry(window=128, stride=64, mel=32, mfcc=12),
    "fft128-64-12-empty-bands": geometry(window=128, stride=64, mel=64, mfcc=12),        # bands 2,3,6,9,12,15 cover no bin
    "dct-80-32": geometry(mel=80, mfcc=32),                                              # general DCT loop
    "dct-41-40-odd": geometry(mel=41, mfcc=40),                                          # odd mel count: middle DCT row
    "dct-128-64": geometry(mel=128, mfcc=64, lower=20.0),                                # one full pass of 64 coefficients
    "dct-80-80": geometry(mel=80, mfcc=80),                                              # second pass: coefficients 64..79
    "dct-128-128": geometry(mel=128, mfcc=128, lower=20.0),                              # widest table, two full passes
    "dct-81-68-odd": geometry(mel=81, mfcc=68),                                          # second pass with the middle row
    "8k-above-nyquist": geometry(sample_rate=8000, clip=8000, window=240, stride=80, mel=40, mfcc=20),   # bands 32..39 empty
    "T148-24000": geometry(clip=24000, window=480, stride=160),                          # long clip, frame chunking
    "logmel-32": geometry(feature_kind=1, mel=32),                                       # num_mfccs 40 > 32 bins: unused
    "logmel-96": geometry(feature_kind=1, mel=96),
}
TOL_MFCC, TOL_LOG_MEL = 2e-6, 2e-5


def check_front_end(backend, g, n_clips, n_lines):
    """eng.mfcc against the fp64 oracle on U(-1, 1) clips with silence and a full-scale square wave among them, plus full-scale
    spectral lines over a -60 dB floor (16 kHz, one-second clips only); int16 input bit-identical to the decoded samples."""
    if (g["sample_rate"], g["clip"]) != (16000, 16000):                 # the lines are one-second 16 kHz clips: more noise instead
        n_clips, n_lines = n_clips + n_lines, 0
    wav, _ = O.synthetic_batch(n_clips, num_samples=g["clip"], adversarial=True)
    tones = spectral_lines()[:n_lines].astype(np.float32) if n_lines else np.zeros((0, g["clip"]), np.float32)
    batch = np.concatenate([wav, tones])
    eng = Engine(backend, max_batch=len(batch), **engine_cfg(g))
    try:
        got = eng.mfcc(batch)
        ref = reference_features(batch, *ref_args(g))
        f = g["mfcc"] if g["feature_kind"] == 0 else g["mel"]
        assert got.shape == ref.shape == (len(batch), O.num_frames(g["clip"], g["window"], g["stride"]), f)
        assert eng.info.fft_length == O.next_pow2(g["window"])
        tol = TOL_MFCC if g["feature_kind"] == 0 else TOL_LOG_MEL
        report = {"clips": rel_err(got[:n_clips], ref[:n_clips])}
        assert report["clips"] <= tol, report
        if n_lines:
            # Under a full-scale line the quiet bands hold the fp32 FFT's round-off of the line, not the -60 dB floor, so the
            # kernel can be no closer than an fp32 restatement of the same front-end (NumPy's float32 FFT); like the training
            # step's floor (parity_cases.check_step), four times that distance bounds it.  Measured on an H100: up to 2.4x.
            floor = rel_err(reference_features(tones, *ref_args(g), dtype=np.float32), ref[n_clips:])
            report["lines"], report["lines_f32_oracle_floor"] = rel_err(got[n_clips:], ref[n_clips:]), floor
            assert report["lines"] <= max(tol, 4 * floor), report
        pcm = np.clip(np.round(batch * 32768.0), -32768, 32767).astype(np.int16)
        assert np.array_equal(eng.mfcc(pcm), eng.mfcc(pcm.astype(np.float32) / 32768.0))
        return report
    finally:
        eng.close()


@pytest.mark.parametrize("name", list(FRONT_END))
def test_emulated_front_end_geometry(emu, name):
    check_front_end(emu, FRONT_END[name], 4, 4)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FRONT_END))
def test_front_end_geometry(cuda, name):
    print(name, check_front_end(cuda, FRONT_END[name], 30, 7))


@pytest.mark.parametrize("name", list(FRONT_END) + ["baseline-mfcc", "baseline-logmel"])
def test_only_the_recipe_shape_takes_the_frame_pair_kernel(emu, monkeypatch, name):
    """mfcc_pair_supported: every shape of the table runs the one-frame-per-warp kernel whether or not the frame-pair kernel is
    enabled (bit-identical features); the 640/320, 64-bin shape does take it (the features differ in the last bits)."""
    g = FRONT_END.get(name) or geometry(feature_kind=int(name.endswith("logmel")))
    wav, _ = O.synthetic_batch(4, num_samples=g["clip"], adversarial=True)
    out = {}
    for pair in ("1", "0"):
        monkeypatch.setenv("TCR_MFCC_PAIR", pair)
        eng = Engine(emu, max_batch=4, **engine_cfg(g))
        out[pair] = eng.mfcc(wav)
        eng.close()
    assert np.array_equal(out["1"], out["0"]) == (name in FRONT_END)


# ------------------------------------------------------------------------------------------------------------------------
# Training step and evaluation forward
# ------------------------------------------------------------------------------------------------------------------------

def _t(frames):
    """640/320 windows: the clip length that gives `frames` frames."""
    return dict(clip=640 + 320 * (frames - 1))


# The log-mel features carry the fp32 FFT's round-off in their quiet bands (up to ~1e-5 of the largest feature, inside the
# front-end's 2e-5 bound) and the gradient amplifies it past 1e-4 at small T (1.3e-4 for TCResNet14 at T=7, n=5): those cases
# are floored by an fp32 restatement of the oracle that computes its features in fp32 too (parity_cases.run_case).
F20, F64, F128, LM96 = dict(mfcc=20), dict(mfcc=64), dict(mel=128, mfcc=128), dict(feature_kind=1, mel=96)
C2, C13, C32 = dict(num_classes=2), dict(num_classes=13, ls=0.1), dict(num_classes=32)
T148 = dict(clip=24000, window=480, stride=160)
# every T with both models, the feature counts and class counts in rotation; T <= 3 with the fp32-oracle floor (below)
TRAIN = {
    "r8-T1-F20-c2": dict(model="TCResNet8", **_t(1), **F20, **C2),
    "r14-T1-F64-c13": dict(model="TCResNet14", **_t(1), **F64, **C13, keep=0.5),
    "r8-T3-logmel96-c32": dict(model="TCResNet8", **_t(3), **LM96, **C32, keep=0.5),
    "r14-T3-F20-c2": dict(model="TCResNet14", **_t(3), **F20, **C2),
    "r8-T7-F64-c13": dict(model="TCResNet8", **_t(7), **F64, **C13),
    "r14-T7-logmel96-c32": dict(model="TCResNet14", **_t(7), **LM96, **C32, keep=0.5),
    "r8-T14-F20-c32": dict(model="TCResNet8", **_t(14), **F20, **C32, keep=0.5),
    "r14-T14-F64-c2": dict(model="TCResNet14", **_t(14), **F64, **C2),
    "r8-T24-logmel96-c13": dict(model="TCResNet8", **_t(24), **LM96, **C13),
    "r14-T24-F20-c13": dict(model="TCResNet14", **_t(24), **F20, **C13, keep=0.5),
    "r8-T148-F64-c32": dict(model="TCResNet8", **T148, **F64, **C32, keep=0.5),
    "r14-T148-logmel96-c2": dict(model="TCResNet14", **T148, **LM96, **C2),
    "r8x1.5-T148-F20-c13": dict(model="TCResNet8", wm=1.5, **T148, **F20, **C13, keep=0.5),
    "r8-T7-F128-c13": dict(model="TCResNet8", **_t(7), **F128, **C13, keep=0.5),          # the widest front-end into conv0
}


def frames_of(kw):
    return O.num_frames(kw.get("clip", 16000), kw.get("window", 640), kw.get("stride", 320))


def train_case(backend, name, n, **extra):
    kw = dict(TRAIN[name], **extra)
    # BatchNorm over n * T <= 3n rows: the fp32 restatement of the oracle is itself ~4e-4 from fp64 at T = 2..3, n = 3
    log_mel = kw.get("feature_kind", 0) == 1
    return run_case(backend, n=n, check_f32_floor=frames_of(kw) <= 3 or log_mel, f32_front_end=log_mel, **kw)


def emulator_batch(kw):
    """n <= 8 on the emulator.  T <= 3 takes all 8: BatchNorm over 5 rows of TCResNet14 at T=1 makes gradients of ~500 whose
    fp32 round-off alone exceeds 1e-4 (the fp32 oracle is 1.8e-4 from fp64 there); T=148 takes 3 to keep the oracle quick."""
    t = frames_of(kw)
    return 8 if t <= 3 else 3 if t >= 148 else 5


@pytest.mark.parametrize("name", list(TRAIN))
def test_emulated_training_step_geometry(emu, name):
    train_case(emu, name, emulator_batch(TRAIN[name]), steps=2)


def resident_mode(backend, name, n):
    """The mode a handle of max_batch n picks for the case (launch profiler): 3 resident forward and backward-data kernels,
    1 resident forward kernel only, 0 per-layer kernels."""
    kw = TRAIN[name] if isinstance(name, str) else name
    g = geometry(**{k: v for k, v in kw.items() if k in BASE})
    spec = O.build_spec(kw["model"], kw.get("wm", 1.0), frames_of(kw), f_in=g["mfcc"] if g["feature_kind"] == 0 else g["mel"],
                        num_classes=kw.get("num_classes", 12))
    pv, mv = O.init_variables(spec, 0)
    pf, mf = O.flatten_vars(spec, pv), O.flatten_moving(spec, mv)
    wav, onehot = O.synthetic_batch(n, num_samples=g["clip"], num_classes=spec.num_classes)
    eng = Engine(backend, model=int(kw["model"][len("TCResNet"):]), width_multiplier=kw.get("wm", 1.0), max_batch=n,
                 num_classes=spec.num_classes, dropout_keep_prob=0.5, **engine_cfg(g))
    try:
        names = launched(backend.lib, lambda: eng.train_step(wav, onehot, pf, np.zeros_like(pf), mf))
    finally:
        eng.close()
    return 3 if "resident_bwd_data" in names else 1 if "resident_fwd" in names else 0


# (case, max_batch) -> the mode the resident planner falls back to on an H100 (132 SMs): at T=148 the activation tiles of even
# one utterance per CTA leave no room in 227 KB of shared memory for the wider nets, and two or more do not fit for TCResNet8
# either.  Every other shape runs mode 3.
FALLBACK = {
    ("r8-T148-F64-c32", 133): 0, ("r8-T148-F64-c32", 512): 0,
    ("r14-T148-logmel96-c2", 8): 0, ("r14-T148-logmel96-c2", 133): 0, ("r14-T148-logmel96-c2", 512): 0,
    ("r8x1.5-T148-F20-c13", 8): 0, ("r8x1.5-T148-F20-c13", 133): 0, ("r8x1.5-T148-F20-c13", 512): 0,
    ("r14x1.5", 1024): 0,
}

GPU_RUNS = {"n8": (8, None), "n133": (133, None), "n512": (512, None), "n133-res0": (133, "0"), "n133-res1": (133, "1")}


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(GPU_RUNS))
@pytest.mark.parametrize("name", list(TRAIN))
def test_training_step_geometry(cuda, monkeypatch, name, run):
    """n = 133: one CTA owns two utterances; n = 512: four.  TCR_RESIDENT = 0 / 1 pin the per-layer / resident-forward paths."""
    n, env = GPU_RUNS[run]
    if env is None:
        monkeypatch.delenv("TCR_RESIDENT", raising=False)
    else:
        monkeypatch.setenv("TCR_RESIDENT", env)
    report = train_case(cuda, name, n, force_masks=n > 8)
    default = FALLBACK.get((name, n), 3)
    mode = resident_mode(cuda, name, n)
    print(name, run, "mode", mode, {k: float("%.2e" % v) for k, v in report.items()})
    assert mode == (default if env is None else min(int(env), default))


# ------------------------------------------------------------------------------------------------------------------------
# One handle, shrinking batches
# ------------------------------------------------------------------------------------------------------------------------

def shrinking_batches(backend, model, wm, max_batch, sizes, eval_n, keep=0.5):
    """Steps of decreasing n on one handle sized for max_batch, then an evaluation forward, each against the oracle started
    from the handle's own previous state: per-CTA records, weight-gradient chunks or BatchNorm partials that a larger step left
    behind must not reach a smaller one."""
    spec = O.build_spec(model, wm, 49)
    eng = Engine(backend, model=int(model[len("TCResNet"):]), width_multiplier=wm, max_batch=max_batch, dropout_keep_prob=keep)
    try:
        params, moving = perturbed_variables(spec)
        rng = np.random.RandomState(7)
        slots = {k: 0.01 * rng.randn(*v.shape) for k, v in params.items()}
        state = O.flatten_vars(spec, params), O.flatten_moving(spec, moving), O.flatten_vars(spec, slots)
        report = {}
        for i, n in enumerate(sizes):
            wav, onehot = O.synthetic_batch(n, seed_wav=100 + i, seed_label=200 + i, adversarial=True)
            mask = (rng.rand(n, spec.c_last) < keep).astype(np.float32)
            state = check_step(eng, spec, wav, O.mfcc(wav, 640, 320), onehot, state, 0.1, 0.9, 1e-3, keep, mask, 0.0, report,
                               f"_n{n}", seed=i, force_masks=n > 8)
        wav, onehot = O.synthetic_batch(eval_n, seed_wav=99, adversarial=True)
        check_eval(eng, spec, wav, O.mfcc(wav, 640, 320), onehot, O.unflatten_vars(spec, state[0]),
                   O.unflatten_moving(spec, state[1]), 1e-3, 0.0, report, tag=f"eval_n{eval_n}")
        return report
    finally:
        eng.close()


def test_emulated_shrinking_batches_on_one_handle(emu, monkeypatch):
    """The emulator runs 3 CTAs and sizes the resident head for 8 utterances per CTA: a 24-utterance handle is the largest that
    runs the resident kernels (mode 3) there."""
    monkeypatch.delenv("TCR_RESIDENT", raising=False)
    shrinking_batches(emu, "TCResNet8", 1.0, 24, [24, 1, 5, 23], 3)


@pytest.mark.gpu
def test_shrinking_batches_on_one_handle(cuda, monkeypatch):
    monkeypatch.delenv("TCR_RESIDENT", raising=False)
    print(shrinking_batches(cuda, "TCResNet8", 1.0, 512, [512, 1, 37, 133, 511], 3))
    print(shrinking_batches(cuda, "TCResNet14", 1.5, 1024, [1024, 100], 3))
    assert resident_mode(cuda, dict(model="TCResNet8"), 512) == 3
    assert resident_mode(cuda, dict(model="TCResNet14", wm=1.5), 1024) == FALLBACK.get(("r14x1.5", 1024), 3)


# ------------------------------------------------------------------------------------------------------------------------
# Refusals
# ------------------------------------------------------------------------------------------------------------------------

# (flag overrides of the reference's CLI, the same as tcr_config fields, status, message)
REFUSALS = {
    "num_mfccs-10": (dict(num_mfccs=10), dict(num_mfccs=10), 3, "feature count 10 is not a multiple of 4"),
    "fft-64": (dict(window_size_ms=4.0, window_stride_ms=2.0), dict(window_size_samples=64, window_stride_samples=32), 3,
               "fft length 64 outside"),
    "fft-4096": (dict(window_size_ms=160.0), dict(window_size_samples=2560), 3, "fft length 4096 outside"),
    "num_classes-33": (dict(num_classes=33), dict(num_classes=33), 3, r"num_classes must be in \[1,32\]"),
    "num_mel_bins-129": (dict(num_mel_bins=129), dict(num_mel_bins=129), 1, "bad num_mel_bins"),
    "clip-shorter-than-window": (dict(clip_duration_ms=30), dict(clip_samples=480), 1, "bad window/stride/clip"),
}


@pytest.mark.parametrize("name", list(REFUSALS))
def test_emulated_refusals(emu, name):
    from tcresnet_b200._lib import TcrError
    _, cfg, status, msg = REFUSALS[name]
    with pytest.raises(TcrError, match=rf"status {status}\): {msg}"):
        Engine(emu, **cfg)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(REFUSALS))
def test_refusals_through_the_model_class(cuda, name):
    """The same refusals from the CLI flags, through the reference-named model class (as width_multiplier 0.75 is)."""
    from tcresnet_b200._lib import TcrError
    from tcresnet_b200.factory import audio_nets
    from tcresnet_b200.runtime import Node
    flags, cfg, status, msg = REFUSALS[name]
    with pytest.raises(TcrError, match=rf"status {status}\): {msg}"):
        Engine(cuda, **cfg)
    args = dict(width_multiplier=1.0, num_classes=12, sample_rate=16000, clip_duration_ms=1000, window_size_ms=40.0,
                window_stride_ms=20.0, num_mel_bins=64, num_mfccs=40, lower_edge_hertz=80.0, upper_edge_hertz=7600.0,
                preprocess_method="mfcc", batch_size=8, dropout_keep_prob=0.5, output_name="output/softmax", weight_decay=1e-3)
    args.update(flags)
    model = audio_nets.TCResNet8Model(argparse.Namespace(**args), None)
    with pytest.raises(TcrError, match=rf"status {status}\): {msg}"):
        model.build(Node("wavs", [None, args["clip_duration_ms"] * 16, 1]), Node("labels", [None, args["num_classes"]]), True)


def check_pcm16_refused_fp32_computed(backend, n):
    """12 kHz with a 25 ms window: 300 samples, a multiple of 4 but not of 8, so int16 rows cannot be staged whole; PCM16 input is
    an error from the front-end and from a training step, and fp32 input on the same handle still matches the oracle."""
    from tcresnet_b200._lib import TcrError
    g = geometry(sample_rate=12000, clip=12000, window=300, stride=120)
    eng = Engine(backend, max_batch=n, dropout_keep_prob=1.0, **engine_cfg(g))
    try:
        wav, onehot = O.synthetic_batch(n, num_samples=12000, adversarial=True)
        pcm = np.clip(np.round(wav * 32768.0), -32768, 32767).astype(np.int16)
        spec = O.build_spec("TCResNet8", 1.0, eng.info.frames)
        params, moving = perturbed_variables(spec)
        pf, mf = O.flatten_vars(spec, params), O.flatten_moving(spec, moving)
        with pytest.raises(TcrError, match=r"status 3\): int16 input needs"):
            eng.mfcc(pcm)
        with pytest.raises(TcrError, match=r"status 3\): int16 input needs"):
            eng.train_step(pcm, onehot, pf, np.zeros_like(pf), mf)
        feat = reference_features(wav, *ref_args(g))
        assert eng.info.frames == 98 and eng.info.fft_length == 512
        assert rel_err(eng.mfcc(wav), feat) <= TOL_MFCC
        check_step(eng, spec, wav, feat, onehot, (pf, mf, np.zeros_like(pf)), 0.1, 0.9, 1e-3, 1.0, None, 0.0, {}, 0,
                   force_masks=n > 8)
    finally:
        eng.close()


def test_emulated_pcm16_needs_rows_of_8_samples(emu):
    check_pcm16_refused_fp32_computed(emu, 5)


@pytest.mark.gpu
def test_pcm16_needs_rows_of_8_samples(cuda):
    check_pcm16_refused_fp32_computed(cuda, 133)
