"""Kernel LOGIC parity on a CPU box: the product kernel sources compiled against the test-only fiber
emulator (tests/emu) and driven through the same C ABI, compared with the fp64 oracle.  Sizes are tiny; the real
parity tests are the -m gpu ones (tests/test_gpu_parity.py) that run the sm_90a build."""
import numpy as np
import pytest

from parity_cases import run_case
from tcr_harness import Engine, NumpyBackend, rel_err
from oracle import tcr_oracle as O


@pytest.fixture(scope="module")
def backend():
    return NumpyBackend()


@pytest.mark.parametrize("kw", [
    dict(model="TCResNet8", wm=1.0, window=640, stride=320, n=5, keep=1.0),
    dict(model="TCResNet14", wm=1.5, window=640, stride=320, n=3, keep=0.5),
    dict(model="TCResNet8", wm=1.0, window=480, stride=160, n=3, keep=0.5, ls=0.1),
    dict(model="TCResNet14", wm=1.0, window=480, stride=160, n=2, use_wav=False),
    dict(model="TCResNet8", wm=1.5, window=640, stride=320, n=1, steps=2),
    dict(model="TCResNet8", wm=1.0, window=640, stride=320, n=37, keep=0.5, max_batch=512),   # plan sized for 512, ragged clusters
    dict(model="TCResNet14", wm=2.0, window=640, stride=320, n=6),                           # 96-channel layers: filters via L1
], ids=["r8-T49", "r14x1.5-T49-dropout", "r8-T98-smoothing", "r14-T98-features", "r8x1.5-n1-2steps", "r8-n37-of-512", "r14x2-n6"])
def test_emulated_kernels_match_oracle(backend, kw):
    report = run_case(backend, **kw)
    assert report["features"] < 1e-6


@pytest.mark.parametrize("mode", ["0", "1", "3"])
def test_emulated_resident_kernels(backend, monkeypatch, mode):
    """TCR_RESIDENT = 0: per-layer kernels; 1: resident forward kernel; 3 (the default): resident forward and backward-data kernels
    (tcr_resident.cu; the emulator runs 3 co-resident CTAs, so ownership is ragged: 7 utterances = 3 + 2 + 2)."""
    monkeypatch.setenv("TCR_RESIDENT", mode)
    run_case(backend, model="TCResNet8", wm=1.0, window=640, stride=320, n=7, keep=0.5, steps=2)
    run_case(backend, model="TCResNet14", wm=1.0, window=480, stride=160, n=2, use_wav=False)      # identity-shortcut blocks


def test_mask_forced_gradient_comparison(backend):
    """The oracle run with the CUDA path's own ReLU decisions (rebuilt from the workspace tensors): same bounds, no fp32 floor."""
    report = run_case(backend, model="TCResNet8", wm=1.0, window=640, stride=320, n=6, keep=0.5, force_masks=True)
    assert report["grads0"] < 1e-4


def test_unsupported_width_status(backend):
    """Channel counts that are not multiples of 4 (width 0.75 -> 18) are refused with TCR_ERR_UNSUPPORTED, never computed wrongly."""
    from tcresnet_b200._lib import TcrError
    with pytest.raises(TcrError, match=r"status 3.*multiple of 4"):
        Engine(backend, width_multiplier=0.75)


def test_log_mel_front_end(backend):
    eng = Engine(backend, feature_kind=1, max_batch=4)
    wav, _ = O.synthetic_batch(2, adversarial=True)
    got = eng.mfcc(wav)
    ref = O.log_mel_spectrogram(wav, 640, 320, magnitude_squared=False)
    assert got.shape == (2, 49, 64)
    assert rel_err(got, ref) < 2e-5      # log of tiny magnitudes (square wave): fp32 FFT round-off
    eng.close()


def test_pcm16_input_is_bit_identical_to_decoded_samples(backend):
    """TCR_INPUT_WAV_PCM16: int16 samples scaled by 1/32768 in the framing stage == decode_wav then the fp32 path."""
    eng = Engine(backend, max_batch=4)
    rng = np.random.default_rng(5)
    pcm = rng.integers(-32768, 32768, size=(3, 16000), dtype=np.int16)
    pcm[0, :700] = [-32768, 32767] * 350
    got = eng.mfcc(pcm)
    ref = eng.mfcc(pcm.astype(np.float32) / 32768.0)
    assert np.array_equal(got, ref)
    assert rel_err(got, O.mfcc(pcm.astype(np.float64) / 32768.0, 640, 320)) < 2e-5   # full-scale Nyquist square wave in clip 0
    spec = O.build_spec("TCResNet8", 1.0, 49)
    pv, mv = O.init_variables(spec, 3)
    params, moving = O.flatten_vars(spec, pv).astype(np.float32), O.flatten_moving(spec, mv).astype(np.float32)
    slots = np.zeros_like(params)
    onehot = np.eye(12, dtype=np.float32)[[1, 5, 7]]
    a = eng.train_step(pcm, onehot, params, slots, moving, seed=4)
    b = eng.train_step(pcm.astype(np.float32) / 32768.0, onehot, params, slots, moving, seed=4)
    assert np.array_equal(a["params"], b["params"]) and np.array_equal(a["losses"], b["losses"])
    eng.close()


def test_host_buffer_step_and_its_loss_pipeline(backend):
    """tcr_train_step_host: same update as the device-buffer step; losses come back `lag` submissions late, in order."""
    import ctypes as C
    from tcresnet_b200 import _lib as L
    eng = Engine(backend, max_batch=4)
    spec = O.build_spec("TCResNet8", 1.0, 49)
    pv, mv = O.init_variables(spec, 3)
    params0, moving0 = O.flatten_vars(spec, pv).astype(np.float32), O.flatten_moving(spec, mv).astype(np.float32)
    wav, onehot = O.synthetic_batch(3, seed_wav=9)
    ref = eng.train_step(wav, onehot, params0, np.zeros_like(params0), moving0, seed=4)

    def host_step(params, slots, moving, lag, seed):
        a = L.TcrStepArgs()
        a.input, a.input_is_features, a.onehot, a.n = wav.ctypes.data, 0, onehot.ctypes.data, 3
        a.params, a.slots, a.moving = params.ctypes.data, slots.ctypes.data, moving.ctypes.data
        a.learning_rate, a.momentum, a.weight_decay, a.dropout_seed, a.apply_update = 0.1, 0.9, 1e-3, seed, 1
        out, step = (C.c_float * 2)(), C.c_int64(-7)
        L.check(eng.lib, eng.lib.tcr_train_step_host(eng.h, C.byref(a), lag, None, out, C.byref(step)), "tcr_train_step_host")
        return step.value, (out[0], out[1])

    p, sl, mvv = params0.copy(), np.zeros_like(params0), moving0.copy()
    step, losses = host_step(p, sl, mvv, 0, 4)
    assert step == 0 and np.array_equal(p, ref["params"]) and np.allclose(losses, ref["losses"], rtol=0, atol=0)
    got = [host_step(p, sl, mvv, 2, 5 + i)[0] for i in range(4)]
    assert got == [-1, -1, 1, 2]                     # step 0 was collected above; lag 2 keeps two in flight
    out, stepv, rest = (C.c_float * 2)(), C.c_int64(0), []
    while True:
        L.check(eng.lib, eng.lib.tcr_host_flush(eng.h, out, C.byref(stepv)), "tcr_host_flush")
        if stepv.value < 0:
            break
        rest.append(stepv.value)
    assert rest == [3, 4]
    eng.close()


def test_unsupported_width_is_an_error(backend):
    with pytest.raises(Exception, match="multiple of 4"):
        Engine(backend, width_multiplier=1.3)


def test_batch_larger_than_workspace_is_an_error(backend):
    eng = Engine(backend, max_batch=2)
    wav, _ = O.synthetic_batch(3)
    with pytest.raises(Exception, match="max_batch"):
        eng.mfcc(wav)
    eng.close()


@pytest.mark.parametrize("pair", ["1", "4", "0"], ids=["pairs-10-per-item", "pairs-4-per-item", "one-frame-per-warp"])
def test_both_front_end_kernels_match_the_oracle(backend, monkeypatch, pair):
    """TCR_MFCC_PAIR: the frame-pair kernel (tcr_mfcc_pair.cu, default for the 640 / 320 / 1024 shape; 49 frames = an odd count, so
    the last work item of an utterance ends on half a pair) and the one-frame-per-warp kernel (tcr_mfcc.cu), MFCC and log-mel,
    fp32 and int16 input, silence and a full-scale square wave among the clips."""
    monkeypatch.setenv("TCR_MFCC_PAIR", pair)
    wav, _ = O.synthetic_batch(5, adversarial=True)
    for kind, ref in ((0, O.mfcc(wav, 640, 320)), (1, O.log_mel_spectrogram(wav, 640, 320, magnitude_squared=False))):
        eng = Engine(backend, feature_kind=kind, max_batch=8)
        got = eng.mfcc(wav)
        assert got.shape == ref.shape
        assert rel_err(got, ref) < (1e-6 if kind == 0 else 2e-5)
        pcm = np.clip(np.round(wav * 32768.0), -32768, 32767).astype(np.int16)
        assert np.array_equal(eng.mfcc(pcm), eng.mfcc(pcm.astype(np.float32) / 32768.0))
        eng.close()


def test_single_spectral_lines_through_the_run_based_mel_stage(backend, monkeypatch):
    """The frame-pair kernel forms the falling half of a band as a difference (sum P - sum u P over a run of bins), worst on a
    band that one spectral line dominates (bin 147 = 2296.875 Hz has the smallest 1 - u).  Strong lines over a -60 dB floor:
    the error is the fp32 FFT's round-off floor under the line in BOTH kernels; the run-based stage must not add to it."""
    from parity_cases import spectral_lines
    tones = spectral_lines()
    err = {}
    for pair in ("1", "0"):
        monkeypatch.setenv("TCR_MFCC_PAIR", pair)
        for kind, ref in ((0, O.mfcc(tones, 640, 320)), (1, O.log_mel_spectrogram(tones, 640, 320, magnitude_squared=False))):
            eng = Engine(backend, feature_kind=kind, max_batch=8)
            err[pair, kind] = rel_err(eng.mfcc(tones), ref)
            eng.close()
    assert err["1", 0] < 2e-5 and err["1", 0] < 1.5 * err["0", 0] + 1e-7
    assert err["1", 1] < 1e-3 and err["1", 1] < 1.5 * err["0", 1] + 1e-7
