"""Device input stage (tcr_augment_pcm16) vs the NumPy restatement of datasets/augmentation_factory.py: bit-exact for the same
random draws.  Kernel logic on the CPU emulator here, the sm_90a build under -m gpu."""
import numpy as np
import pytest

from oracle import augment_oracle as A
from oracle import tcr_oracle as O
from tcr_harness import Engine, NumpyBackend

L = 16000


def _case(seed, n, stride, with_bg=True):
    rng = np.random.RandomState(seed)
    pcm = rng.randint(-32768, 32768, size=(n, stride)).astype(np.int16)
    bg_lengths = [L, 23000, 61234] if with_bg else []
    background = (rng.uniform(-1, 1, size=int(sum(bg_lengths))).astype(np.float32)) if with_bg else None
    clips = A.random_clips(rng, n, L, stride, bg_lengths)
    return pcm, clips, background


def _edge_clips(clips):
    clips = clips.copy()
    clips[0]["shift"], clips[0]["silent"], clips[0]["length"] = 1599, 0, 16000       # largest forward shift
    clips[1]["shift"], clips[1]["silent"] = -1600, 0                                  # largest backward shift
    clips[2]["silent"] = 1                                                            # synthesised silence (+ background)
    clips[3]["length"], clips[3]["shift"], clips[3]["silent"] = 9000, 0, 0            # short recording: zero-padded
    clips[4]["bg_volume"] = np.float32(1.0)                                           # forces the clip to [-1, 1] to act
    return clips


def _check(backend, seed, n, stride, with_bg=True):
    eng = Engine(backend, max_batch=n)
    pcm, clips, background = _case(seed, n, stride, with_bg)
    if n >= 5:
        clips = _edge_clips(clips)
    got = eng.augment(pcm, clips, background)
    ref = A.augment(pcm, clips, background, L)
    assert got.dtype == np.float32 and got.shape == (n, L)
    assert np.array_equal(got, ref), np.abs(got - ref).max()
    assert got.min() >= -1.0 and got.max() <= 1.0
    eng.close()
    return got


def test_emulated_input_stage_is_bit_exact():
    b = NumpyBackend()
    _check(b, 1, 6, 16000)
    _check(b, 2, 5, 20000)                     # recordings longer than the clip are cropped
    _check(b, 3, 2, 16000, with_bg=False)      # evaluation split: no background bank


def _step_inputs(seed, n, stride):
    pcm, clips, background = _case(seed, n, stride)
    spec = O.build_spec("TCResNet8", 1.0, 49)
    pv, mv = O.init_variables(spec, 3)
    params, moving = O.flatten_vars(spec, pv).astype(np.float32), O.flatten_moving(spec, mv).astype(np.float32)
    onehot = np.eye(12, dtype=np.float32)[np.random.RandomState(seed).randint(0, 12, n)]
    return pcm, clips, background, params, moving, onehot


def _check_step_with_input_stage(backend, n, stride):
    """A step that starts from int16 clips + draws == the input stage followed by a step on its fp32 output, bit for bit."""
    eng = Engine(backend, max_batch=n)
    pcm, clips, background, params, moving, onehot = _step_inputs(21, n, stride)
    wav = eng.augment(pcm, clips, background)
    a = eng.train_step(pcm, onehot, params, np.zeros_like(params), moving, seed=4, clips_np=clips, background_np=background)
    b = eng.train_step(wav, onehot, params, np.zeros_like(params), moving, seed=4)
    assert np.array_equal(a["params"], b["params"]) and np.array_equal(a["losses"], b["losses"])
    assert np.isfinite(a["params"]).all()
    eng.close()


def test_emulated_step_with_the_input_stage_in_front():
    _check_step_with_input_stage(NumpyBackend(), 3, 16500)


def test_emulated_host_buffer_step_with_the_input_stage():
    """tcr_train_step_host with int16 rows + draws in host memory == the device-buffer step with the same stage in front."""
    import ctypes as C
    from tcresnet_b200 import _lib as Lb
    b = NumpyBackend()
    eng = Engine(b, max_batch=3)
    pcm, clips, background, params, moving, onehot = _step_inputs(33, 3, 16200)
    ref = eng.train_step(pcm, onehot, params, np.zeros_like(params), moving, seed=6, clips_np=clips, background_np=background)
    p, sl, mv = params.copy(), np.zeros_like(params), moving.copy()
    rec = np.frombuffer(np.ascontiguousarray(clips).tobytes(), np.uint8).copy()
    a = Lb.TcrStepArgs()
    a.input, a.input_is_features, a.onehot, a.n = pcm.ctypes.data, Lb.TCR_INPUT_WAV_PCM16, onehot.ctypes.data, 3
    a.clips, a.background, a.pcm_stride = rec.ctypes.data, background.ctypes.data, pcm.shape[1]
    a.params, a.slots, a.moving = p.ctypes.data, sl.ctypes.data, mv.ctypes.data
    a.learning_rate, a.momentum, a.weight_decay, a.dropout_seed, a.apply_update = 0.1, 0.9, 1e-3, 6, 1
    out, step = (C.c_float * 2)(), C.c_int64(-7)
    Lb.check(eng.lib, eng.lib.tcr_train_step_host(eng.h, C.byref(a), 0, None, out, C.byref(step)), "tcr_train_step_host")
    assert step.value == 0 and np.array_equal(p, ref["params"]) and (out[0], out[1]) == tuple(ref["losses"])
    eng.close()


def test_oracle_matches_the_host_restatement_of_the_input_pipeline():
    """The oracle and the host-side module that mirrors the reference's API agree sample for sample."""
    import tcresnet_b200  # noqa: F401
    from tcresnet_b200.datasets import augmentation_factory as H
    rng = np.random.RandomState(5)
    x = rng.uniform(-1, 1, L).astype(np.float32)
    pcm = np.round(x * 32767).astype(np.int16)[None]
    shifted = H.shift_audio(pcm[0].astype(np.float32) / np.float32(32768.0), np.random.RandomState(11))
    amount = int(np.random.RandomState(11).randint(-1600, 1600))
    clips = np.zeros(1, A.CLIP_DTYPE)
    clips[0]["length"], clips[0]["shift"], clips[0]["bg_offset"] = L, amount, -1
    assert np.array_equal(A.augment(pcm, clips, None, L)[0], shifted)


def test_host_side_draws_use_the_abi_record_layout():
    import tcresnet_b200  # noqa: F401
    from tcresnet_b200.datasets import device_input_stage as D
    assert D.CLIP_DTYPE == A.CLIP_DTYPE and D.CLIP_DTYPE.itemsize == 24
    clips = D.draw_clips(np.random.RandomState(3), [16000, 12000, 20000], [False, True, False], L, [L, 40000])
    assert (np.abs(clips["shift"]) <= 1600).all() and (clips["bg_offset"] >= 0).all() and (clips["bg_volume"] <= 0.1).all()
    assert ((clips["bg_offset"] < L + 40000 - L + 1)).all()
    ev = D.draw_clips(np.random.RandomState(3), [16000], [False], L, [], shift=False, is_training=False)
    assert ev[0]["shift"] == 0 and ev[0]["bg_offset"] == -1


@pytest.mark.gpu
def test_cuda_input_stage_is_bit_exact_and_feeds_the_front_end():
    from tcr_harness import TorchBackend
    b = TorchBackend()
    wav = _check(b, 7, 64, 16000)
    _check(b, 8, 33, 17000)
    _check(b, 9, 3, 16000, with_bg=False)
    eng = Engine(b, max_batch=64)
    feat = eng.mfcc(wav)
    assert np.abs(feat - O.mfcc(wav.astype(np.float64), 640, 320)).max() / np.abs(feat).max() < 2e-5
    eng.close()
    _check_step_with_input_stage(b, 48, 16000)


@pytest.mark.gpu
def test_host_feed_with_the_device_input_stage():
    """tcr_train_step_host fed int16 clips + draws from pinned host memory == device-buffer steps on the augmented fp32 wav."""
    import torch
    import tcresnet_b200  # noqa: F401
    from tcresnet_b200.datasets import device_input_stage as D
    from tcresnet_b200.engine import Engine as PublicEngine, HostFeed
    eng = PublicEngine(max_batch=32)
    rng = np.random.RandomState(2)
    bg = [rng.uniform(-1, 1, 40000).astype(np.float32), rng.uniform(-1, 1, 70000).astype(np.float32)]
    stage = D.DeviceInputStage(eng, bg)
    pcm = [torch.from_numpy(rng.randint(-30000, 30000, (32, 16000)).astype(np.int16)).pin_memory() for _ in range(3)]
    clips = [D.draw_clips(rng, [16000] * 32, rng.uniform(size=32) < 0.1, 16000, stage.bg_lengths) for _ in range(3)]
    h_clips = [torch.from_numpy(np.frombuffer(c.tobytes(), np.uint8).copy()).pin_memory() for c in clips]
    hot = [torch.nn.functional.one_hot(torch.from_numpy(rng.randint(0, 12, 32)), 12).float().pin_memory() for _ in range(3)]
    results = {}
    for kind in ("device", "host"):
        params, slots, moving = eng.new_variables(seed=1)
        if kind == "device":
            for i in range(5):
                wav = stage(pcm[i % 3].cuda(), clips[i % 3])
                eng.train_step(wav, hot[i % 3].cuda(), params, slots, moving, 0.05, 0.9, 1e-3, dropout_seed=i)
        else:
            feed = HostFeed(eng, lag=2)
            for i in range(5):
                feed.submit(pcm[i % 3], hot[i % 3], params, slots, moving, 0.05, 0.9, 1e-3, dropout_seed=i, h_clips=h_clips[i % 3],
                            background=stage.background)
            assert len(feed.flush()) == 2
        torch.cuda.synchronize()
        results[kind] = params.cpu().numpy()
    assert np.array_equal(results["host"], results["device"])
    eng.close()
