"""The widths and clip lengths tcr_create accepts, against the fp64 oracle, and what it refuses.

tcr_create refuses every configuration the per-layer kernels cannot run (net_check_envelope): a layer wider than the 128
channels their one-pass BatchNorm statistics cover (2 x C columns over 256 threads), a head tile over its 110 KB
two-CTAs-per-SM budget, or a forward, backward-data or weight-gradient tile that does not fit in the 232,448 B one CTA may opt in
to on an H100 (the emulator draws the same boundary).  So a handle it accepts can always evaluate and always train with
TCR_RESIDENT=0.  The head's tile holds 4 utterances x 3 planes of T_last x C floats.

As in test_geometry, each table runs on the emulator at small n and with -m gpu on the sm_90a build at production batches.
"""
import argparse
import re

import pytest

from parity_cases import run_case
from tcr_harness import Engine, NumpyBackend
from test_geometry import GPU_RUNS, resident_mode


@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


def _t(frames):
    """640/320 windows: the clip length that gives `frames` frames."""
    return 640 + 320 * (frames - 1)


# ------------------------------------------------------------------------------------------------------------------------
# Widths
# ------------------------------------------------------------------------------------------------------------------------

# The widths away from the recipes' 1.0 / 1.5 that tcr_create accepts, at T = 49 and 98: x0.5 has 8/12/16/24 channels (rows
# padded to chan_stride); x2.5 has 40/60/80/120 (weight-gradient tiles of 20 and 12 output channels) and is the widest: x3.0
# ends in 144 channels (REFUSALS).
WIDTHS = {f"r{m}x{wm}-T{t}": dict(model=f"TCResNet{m}", wm=wm, clip=_t(t)) for m in (8, 14) for t in (49, 98) for wm in (0.5, 2.5)}

# The emulator runs the update kernels one fiber per parameter (~10 us each, ~4 s per step at x2.5): it runs one case per
# width-dependent path, two steps at n = 2 (x2.5) or 3; the GPU runs all of them.
EMULATED = {"r8x0.5-T49": 2, "r14x0.5-T98": 2, "r8x2.5-T98": 2}


def width_case(backend, name, n, steps=2):
    """The oracle takes the CUDA path's ReLU decisions at every batch (parity_cases.cuda_relu_masks): at x2.5 one activation
    within round-off of zero flips even at n = 8 (TCResNet14, T = 98: gradients 2.1e-3 from fp64 unforced, 6.4e-6 forced)."""
    kw = WIDTHS[name]
    return run_case(backend, model=kw["model"], wm=kw["wm"], clip=kw["clip"], n=n, keep=0.5, steps=steps, force_masks=True)


@pytest.mark.parametrize("name", list(EMULATED))
def test_emulated_width(emu, name):
    width_case(emu, name, 2 if WIDTHS[name]["wm"] > 2 else 3, steps=EMULATED[name])


def test_width_table_is_the_envelope(emu):
    """x2.5 is accepted at T = 98 and x3.0 (the next multiple of 0.5 with channel counts that are multiples of 4) is refused at T = 49."""
    from tcresnet_b200._lib import TcrError
    for m in (8, 14):
        Engine(emu, model=m, width_multiplier=2.5, clip_samples=_t(98), max_batch=8).close()
        with pytest.raises(TcrError, match=rf"status 3\): workspace allocation failed: TCResNet{m} has a 144-channel layer"):
            Engine(emu, model=m, width_multiplier=3.0, max_batch=8)


def expected_mode(name, n):
    """On an H100 the resident kernels stage the largest filter bank whole: at x2.5 (9 x 80 x 80 floats = 230 KB) it does not
    fit in 227 KB and every step takes the per-layer kernels; x0.5 runs both resident kernels at every batch."""
    return 3 if WIDTHS[name]["wm"] < 2 else 0


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(GPU_RUNS))
@pytest.mark.parametrize("name", list(WIDTHS))
def test_width(cuda, monkeypatch, name, run):
    n, env = GPU_RUNS[run]
    if env is None:
        monkeypatch.delenv("TCR_RESIDENT", raising=False)
    else:
        monkeypatch.setenv("TCR_RESIDENT", env)
    report = width_case(cuda, name, n)
    mode = resident_mode(cuda, WIDTHS[name], n)
    print(name, run, "mode", mode, {k: float("%.2e" % v) for k, v in report.items()})
    default = expected_mode(name, n)
    assert mode == (default if env is None else min(int(env), default))


# ------------------------------------------------------------------------------------------------------------------------
# Clip length
# ------------------------------------------------------------------------------------------------------------------------

# 30 / 10 ms windows (480 / 160 samples): the most frames tcr_create accepts.  T_last = ceil(T / 8) and the head tile grows as
# 48 x T_last x C bytes: one frame more gives T_last 44 x 48 channels or 29 x 72, over the head's 112,640 B.
LONGEST = {("TCResNet8", 1.0): 344, ("TCResNet8", 1.5): 224, ("TCResNet14", 1.0): 344, ("TCResNet14", 1.5): 224}
# the complete message one frame past LONGEST: tcr_create's own, then net_check_envelope's
PAST_LONGEST = {
    1.0: "tcr_create failed (status 3): workspace allocation failed: head tile of {} (T_last 44, 48 channels) needs 112896 B of "
         "shared memory, limit 112640 B: shorten the clip or the width",
    1.5: "tcr_create failed (status 3): workspace allocation failed: head tile of {} (T_last 29, 72 channels) needs 115200 B of "
         "shared memory, limit 112640 B: shorten the clip or the width",
}


def clip_of(frames):
    return 480 + 160 * (frames - 1)


def check_longest_clip(backend, model, wm, n, monkeypatch, parity=True):
    """At the longest clip: features, evaluation forward and a step, in the default mode and with TCR_RESIDENT=0; one frame
    longer, the complete refusal."""
    from tcresnet_b200._lib import TcrError
    frames = LONGEST[(model, wm)]
    m = int(model[len("TCResNet"):])
    with pytest.raises(TcrError) as e:
        Engine(backend, model=m, width_multiplier=wm, window_size_samples=480, window_stride_samples=160,
               clip_samples=clip_of(frames + 1), max_batch=n)
    assert str(e.value) == PAST_LONGEST[wm].format(model)            # intact: not formatted into itself
    reports = {}
    for env in (None, "0") if parity else ():
        if env is None:
            monkeypatch.delenv("TCR_RESIDENT", raising=False)
        else:
            monkeypatch.setenv("TCR_RESIDENT", env)
        reports[env or "default"] = run_case(backend, model=model, wm=wm, window=480, stride=160, clip=clip_of(frames), n=n,
                                             keep=0.5, steps=1, force_masks=True)
    return reports


@pytest.mark.parametrize("model,wm", list(LONGEST))
def test_emulated_longest_clip(emu, monkeypatch, model, wm):
    """Every boundary is asserted; the parity runs (6-10 s each here) cover the narrowest and the widest net."""
    check_longest_clip(emu, model, wm, 2, monkeypatch, parity=(model, wm) in {("TCResNet8", 1.0), ("TCResNet14", 1.5)})


@pytest.mark.gpu
@pytest.mark.parametrize("model,wm", list(LONGEST))
def test_longest_clip(cuda, monkeypatch, model, wm):
    print(model, wm, check_longest_clip(cuda, model, wm, 133, monkeypatch))


# ------------------------------------------------------------------------------------------------------------------------
# Refusals
# ------------------------------------------------------------------------------------------------------------------------

# (flag overrides of the reference's CLI, the same as tcr_config fields, model, message after "status 3): ")
_CREATE = "workspace allocation failed: "
_WIDE = " channels: lower the width"
REFUSALS = {
    "r8x3.0": (dict(width_multiplier=3.0), dict(width_multiplier=3.0), 8,
               _CREATE + "TCResNet8 has a 144-channel layer, the per-layer kernels' BatchNorm statistics take at most 128" + _WIDE),
    "r8x5.5": (dict(width_multiplier=5.5), dict(width_multiplier=5.5), 8,
               _CREATE + "TCResNet8 has a 264-channel layer, the per-layer kernels' BatchNorm statistics take at most 128" + _WIDE),
    "r14x3.0-T98": (dict(width_multiplier=3.0, clip_duration_ms=1980), dict(width_multiplier=3.0, clip_samples=_t(98)), 14,
                    _CREATE + "TCResNet14 has a 144-channel layer, the per-layer kernels' BatchNorm statistics take at most 128" + _WIDE),
    "r8-T345": (dict(window_size_ms=30.0, window_stride_ms=10.0, clip_duration_ms=clip_of(345) // 16),
                dict(window_size_samples=480, window_stride_samples=160, clip_samples=clip_of(345)), 8,
                _CREATE + "head tile of TCResNet8 (T_last 44, 48 channels) needs 112896 B of shared memory, limit 112640 B"),
}


@pytest.mark.parametrize("name", list(REFUSALS))
def test_emulated_refusals(emu, name):
    from tcresnet_b200._lib import TcrError
    _, cfg, m, msg = REFUSALS[name]
    with pytest.raises(TcrError) as e:
        Engine(emu, model=m, **cfg)
    assert str(e.value).startswith("tcr_create failed (status 3): " + msg), str(e.value)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(REFUSALS))
def test_refusals_through_the_model_class(cuda, name):
    """The same refusals from the CLI flags, through the reference-named model classes, when the model is built."""
    from tcresnet_b200._lib import TcrError
    from tcresnet_b200.factory import audio_nets
    from tcresnet_b200.runtime import Node
    flags, cfg, m, msg = REFUSALS[name]
    with pytest.raises(TcrError) as e:
        Engine(cuda, model=m, **cfg)
    assert str(e.value).startswith("tcr_create failed (status 3): " + msg), str(e.value)
    args = dict(width_multiplier=1.0, num_classes=12, sample_rate=16000, clip_duration_ms=1000, window_size_ms=40.0,
                window_stride_ms=20.0, num_mel_bins=64, num_mfccs=40, lower_edge_hertz=80.0, upper_edge_hertz=7600.0,
                preprocess_method="mfcc", batch_size=8, dropout_keep_prob=0.5, output_name="output/softmax", weight_decay=1e-3)
    args.update(flags)
    model = getattr(audio_nets, f"TCResNet{m}Model")(argparse.Namespace(**args), None)
    with pytest.raises(TcrError, match=re.escape("status 3): " + msg)):
        model.build(Node("wavs", [None, args["clip_duration_ms"] * 16, 1]), Node("labels", [None, args["num_classes"]]), True)
