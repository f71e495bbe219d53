"""The continuous-audio listener (tcr_listener_*) away from the two recipe front-ends: every front-end geometry tcr_create accepts
(test_geometry.FRONT_END), the network's width, clip-length and class range, conv0 with its filters read through L1/L2, stream
state across resets and across two listeners on one handle, and the fp64 oracle once per new front-end kind.  Every push is
checked bit for bit against tcr_forward on the clips cut from the zero-prefixed streams, and the carried history against
tcr_mfcc_forward (listener_cases.check_push).  The emulator runs each front-end geometry at two streams; -m gpu runs them at
31 streams of 17 windows, so CTAs of the windowed conv0 hold windows of two streams."""
import shlex

import numpy as np
import pytest

from listener_cases import Listener, Offline, check_push, pushes_needed, random_chunk, variables
from oracle import tcr_oracle as O
from parity_cases import TOL_LOGITS, check_argmax, perturbed_variables, reference_features
from tcr_harness import Engine, NumpyBackend, rel_err
from test_geometry import BASE, FRONT_END, engine_cfg, ref_args


@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


def hop_of(hop, T):
    """hop_frames from a case: an int (at most T), "T", "T-1" (one carried frame, T - 1 when T > 1) or "T/3"."""
    if hop == "T":
        return T
    if hop == "T-1":
        return max(1, T - 1)
    if hop == "T/3":
        return max(1, -(-T // 3))
    return min(hop, T)


def conv0_tile(T, F, cout, n, sms):
    """(utterances per CTA, filters staged in shared memory) of conv0 at batch n: a restatement of the forward planner
    (tcr_net_fwd.cu: pick_fwd_tile over fwd_smem_bytes and tile_cost) for the 3-tap, stride-1, SAME conv on raw features."""
    cs = F if (F >> 2) & 1 else F + 4                                   # chan_stride

    def smem(U, KS, wsm):
        f = U * (T + 2) * cs + KS * U * T * cout + 2 * 256 + 8 * F + 2 * cout + 4 + (3 * F * cout if wsm else 0)
        return 4 * f

    best, pick = 1e30, None
    for p in range(4):
        wsm, occ = p < 2, 1 if p & 1 else 2
        budget = 110 * 1024 if occ == 2 else 200 * 1024
        if wsm and 3 * F * cout * 4 + 16 * 1024 > budget:
            continue
        for U in range(min(16, max(1, -(-n // (sms * occ)))), 0, -1):
            if smem(U, 1, wsm) > budget:
                continue
            waves = -(-(-(-n // U)) // (sms * occ))
            c = waves * (U * (1.7 if occ == 2 else 1.8) * (1.0 if wsm else 1.1) + 4.0)
            if c < best - 1e-9:
                best, pick = c, (U, wsm)
            break
    return pick or (1, False)


def conv0_of(eng):
    """(F, conv0 output channels) of a handle, from its parameter table (conv0's filter bank is [3, 1, F, cout])."""
    w = next(d for d in eng.param_table() if d["name"].endswith("/conv0/weights"))
    return w["shape"][2], w["shape"][3]


def run_listener(backend, cfg, S, K, hop, resets=(), model=8, wm=1.0, num_classes=12, seed=0, extra_pushes=0):
    """S streams, K windows per push, every push until the zero prefix has left the window plus two (plus extra_pushes);
    resets: (push index, stream or -1) applied before that push.  int16 pushes alternate with fp32 ones where the window, stride
    and chunk lengths allow them.  Returns the engine's frame count and hop."""
    eng = Engine(backend, model=model, width_multiplier=wm, max_batch=S * K, num_classes=num_classes, dropout_keep_prob=1.0, **cfg)
    T = eng.info.frames
    hop = hop_of(hop, T)
    s, w = eng.cfg.window_stride_samples, eng.cfg.window_size_samples
    lis = Listener(eng, S, hop, K * hop * s)
    try:
        p_h, m_h = variables(eng, 11 + seed)
        p, m = backend.upload(p_h), backend.upload(m_h)
        off = Offline(eng, S, hop)
        rng = np.random.default_rng(seed + hop)
        pcm_ok = w % 8 == 0 and s % 8 == 0 and lis.chunk % 8 == 0
        for i in range(pushes_needed(T, K, hop) + extra_pushes):
            for at, stream in resets:
                if at == i:
                    lis.reset(stream)
                    for r in (range(S) if stream < 0 else (stream,)):
                        off.reset(r)
            check_push(eng, lis, off, random_chunk(rng, S, lis.chunk, pcm=pcm_ok and i % 2 == 1), p_h, p, m_h, m)
        return T, hop
    finally:
        lis.close()
        eng.close()


# ------------------------------------------------------------------------------------------------------------------------
# Every front-end geometry
# ------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(FRONT_END))
def test_emulated_listener_front_end_geometry(emu, name):
    """Two streams, two windows per push a third of a clip apart; the last stream is reset halfway."""
    run_listener(emu, engine_cfg(FRONT_END[name]), 2, 2, "T/3", resets=((2, 1),))


# (S, K, hop, resets): (a) 527 windows, so the planner puts U >= 2 windows in a CTA and, K being odd, a CTA holds the last window
# of one stream and the first of the next; (b) pushes longer than a clip with one carried frame (K * hop = 2T - 2 > T), a reset
# of every stream and then of the last one.
GPU_RUNS = {"a-S31-K17-hop2": (31, 17, 2, ((3, 15),)), "b-S3-K2-hopT-1": (3, 2, "T-1", ((1, -1), (2, 2)))}
CASES = [(f"{name}-{run}", FRONT_END[name], run, {}) for name in FRONT_END for run in GPU_RUNS]
CASES += [(f"pair-{env}-{run}", BASE, run, {"TCR_MFCC_PAIR": env}) for env in ("0", "6") for run in GPU_RUNS]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_listener_front_end_geometry(cuda, monkeypatch, case):
    import torch
    _, g, run, env = case
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    S, K, hop, resets = GPU_RUNS[run]
    T, hop = run_listener(cuda, engine_cfg(g), S, K, hop, resets=resets)
    eng = Engine(cuda, max_batch=S * K, dropout_keep_prob=1.0, **engine_cfg(g))
    F, cout = conv0_of(eng)
    eng.close()
    U, wsm = conv0_tile(T, F, cout, S * K, torch.cuda.get_device_properties(0).multi_processor_count)
    print(case[0], "T", T, "hop", hop, "conv0 U", U, "staged filters", wsm)
    if run.startswith("a"):
        assert U >= 2 and wsm
    else:
        assert K * hop > T


@pytest.mark.gpu
def test_listener_one_frame_per_push(cuda):
    """K = hop = 1: each push is one stride of samples and one new frame per stream (FFT 2048, T = 23)."""
    run_listener(cuda, engine_cfg(FRONT_END["fft2048-T23"]), 5, 1, 1, resets=((7, 4),))


# ------------------------------------------------------------------------------------------------------------------------
# Network shapes
# ------------------------------------------------------------------------------------------------------------------------

def _clip(frames, window=480, stride=160):
    return window + stride * (frames - 1)


T1 = dict(engine_cfg(BASE), clip_samples=640)                                          # clip = window: T = 1, nothing carried
T344 = dict(engine_cfg(BASE), clip_samples=_clip(344), window_size_samples=480, window_stride_samples=160)   # longest at width 1.0
F128 = engine_cfg(FRONT_END["dct-128-128"])                                              # 128 features into conv0
LOGMEL = engine_cfg(FRONT_END["logmel-96"])
# 128 features at T = 300: conv0's staged-filter tile needs more than 200 KB, so the planner reads its filters through L1/L2
# (conv_fwd_kernel<3, false, true>) at every batch size
NOSTAGE = dict(F128, clip_samples=_clip(300), window_size_samples=480, window_stride_samples=160)
# (model, width, config, classes, S, K, hop)
NETS = {
    "r8-T1": (8, 1.0, T1, 12, 7, 3, 1),
    "r14-T1-c2": (14, 1.0, T1, 2, 31, 17, 1),
    "r8-T344": (8, 1.0, T344, 12, 4, 5, "T-1"),
    "r8-T344-hop7": (8, 1.0, T344, 12, 3, 4, 7),
    "r14x0.5-F128": (14, 0.5, F128, 12, 31, 17, 2),
    "r8x2.5-F128": (8, 2.5, F128, 12, 31, 17, 3),
    "r8-c2": (8, 1.0, engine_cfg(BASE), 2, 31, 17, 2),
    "r14-c32": (14, 1.0, engine_cfg(BASE), 32, 31, 17, 2),
    "r8-logmel": (8, 1.0, LOGMEL, 12, 31, 17, 2),
    "r14-logmel": (14, 1.0, LOGMEL, 12, 31, 17, "T-1"),
    "r8-conv0-unstaged": (8, 1.0, NOSTAGE, 12, 31, 17, "T-1"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(NETS))
def test_listener_network_shape(cuda, name):
    model, wm, cfg, nc, S, K, hop = NETS[name]
    T, hop = run_listener(cuda, cfg, S, K, hop, model=model, wm=wm, num_classes=nc, resets=((2, S - 1),))
    print(name, "T", T, "hop", hop)


def test_emulated_conv0_without_staged_filters(emu):
    """The one accepted shape family whose conv0 runs conv_fwd_kernel<3, false, true>: the planner restatement says so here and
    says the opposite for every front-end geometry, and the listener is exact there too."""
    eng = Engine(emu, max_batch=4, **NOSTAGE)
    T, (F, cout) = eng.info.frames, conv0_of(eng)
    eng.close()
    assert (T, F, cout) == (300, 128, 16)
    for n in (1, 4, 527, 65537):
        assert not conv0_tile(T, F, cout, n, 132)[1]
    for g in FRONT_END.values():
        e = Engine(emu, max_batch=1, **engine_cfg(g))
        assert conv0_tile(e.info.frames, *conv0_of(e), 527, 132)[1]
        e.close()
    run_listener(emu, NOSTAGE, 2, 2, "T-1", resets=((1, 0),))


# ------------------------------------------------------------------------------------------------------------------------
# The fp64 oracle, once per new front-end kind
# ------------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", ["logmel-96", "fft2048-T23", "8k-above-nyquist"])
def test_listener_front_end_against_the_fp64_oracle(cuda, name):
    g = FRONT_END[name]
    S, K = 4, 4
    eng = Engine(cuda, max_batch=S * K, dropout_keep_prob=1.0, **engine_cfg(g))
    T, F = eng.info.frames, eng.info.features
    hop = max(1, T // 5)
    spec = O.build_spec("TCResNet8", 1.0, T, F)
    params, moving = perturbed_variables(spec, 0)
    p_h, m_h = O.flatten_vars(spec, params), O.flatten_moving(spec, moving)
    lis = Listener(eng, S, hop, K * hop * eng.cfg.window_stride_samples)
    try:
        p, m = cuda.upload(p_h), cuda.upload(m_h)
        off = Offline(eng, S, hop)
        rng = np.random.default_rng(2)
        for _ in range(pushes_needed(T, K, hop)):
            x = random_chunk(rng, S, lis.chunk, pcm=False)
            logits, probs = lis.push(x, p, m)
            clips = off.push(x).reshape(S * K, -1)
        ref, _ = O.forward(spec, params, moving, reference_features(clips.astype(np.float64), *ref_args(g)), False)
        got = logits.reshape(S * K, -1)
        err = rel_err(got, ref)
        print(name, "logits vs fp64", err)
        assert err <= TOL_LOGITS, err
        check_argmax(got, ref, err * np.abs(ref).max())
        np.testing.assert_allclose(probs.reshape(S * K, -1), O.softmax(ref), rtol=0, atol=2e-5)
    finally:
        lis.close()
        eng.close()


# ------------------------------------------------------------------------------------------------------------------------
# Two listeners on one handle
# ------------------------------------------------------------------------------------------------------------------------

def two_listeners(backend, forward_n, step_n, steps_at):
    """Listeners of 3 streams at hop 2 and 5 streams at hop 7 on one handle, pushed alternately; between pushes the handle runs
    tcr_forward at another batch size, and at push `steps_at` a training step changes the variables.  Each listener continues
    from its own history exactly."""
    eng = Engine(backend, max_batch=max(forward_n, step_n, 15), dropout_keep_prob=1.0)
    s, T = eng.cfg.window_stride_samples, eng.info.frames
    a, b = Listener(eng, 3, 2, 5 * 2 * s), Listener(eng, 5, 7, 2 * 7 * s)
    try:
        p_h, m_h = variables(eng, 5)
        off_a, off_b = Offline(eng, 3, 2), Offline(eng, 5, 7)
        rng = np.random.default_rng(9)
        for i in range(max(pushes_needed(T, 5, 2), pushes_needed(T, 2, 7)) + 1):
            if i in steps_at:
                wav, onehot = O.synthetic_batch(step_n, seed_wav=50 + i)
                r = eng.train_step(wav.astype(np.float32), onehot.astype(np.float32), p_h, np.zeros_like(p_h), m_h, lr=0.05)
                assert not np.array_equal(r["params"], p_h)
                p_h, m_h = r["params"], r["moving"]
            p, m = backend.upload(p_h), backend.upload(m_h)
            check_push(eng, a, off_a, random_chunk(rng, 3, a.chunk, pcm=i % 2 == 0), p_h, p, m_h, m)
            wav, _ = O.synthetic_batch(forward_n, seed_wav=70 + i)
            assert np.isfinite(eng.forward(wav.astype(np.float32), p_h, m_h)["logits"]).all()
            check_push(eng, b, off_b, random_chunk(rng, 5, b.chunk, pcm=i % 2 == 1), p_h, p, m_h, m)
    finally:
        a.close()
        b.close()
        eng.close()


def test_emulated_two_listeners_on_one_handle(emu):
    two_listeners(emu, 3, 4, (2,))


@pytest.mark.gpu
def test_two_listeners_on_one_handle(cuda):
    two_listeners(cuda, 37, 64, (2, 4))


# ------------------------------------------------------------------------------------------------------------------------
# The Python entry points at a log-mel, 30 / 10 ms geometry
# ------------------------------------------------------------------------------------------------------------------------

LOGMEL_FLAGS = ("--output_name output/softmax --num_classes 12 --preprocess_method log_mel_spectrogram --num_mel_bins 40 "
                "--clip_duration_ms 1000 --window_size_ms 30 --window_stride_ms 10 ")


@pytest.mark.gpu
def test_streaming_model_graph_replay_equals_eager_log_mel(cuda):
    import torch
    from tcresnet_b200 import listen_audio
    from tcresnet_b200.factory import audio_nets
    args = listen_audio.parse_arguments(shlex.split(LOGMEL_FLAGS + "TCResNet8Model --width_multiplier 1.0 unused.wav"))
    model = audio_nets.TCResNet8Model(args, None)
    graph = model.build_streaming_model(streams=3, hop_ms=30, chunk_ms=120)
    eager = audio_nets.StreamingModel(model, graph.engine, 3, 3, 1920, use_graph=False)
    assert graph.engine.info.frames == 98 and graph.engine.info.features == 40
    rng = np.random.default_rng(5)
    for i in range(6):
        x = random_chunk(rng, 3, 1920, pcm=i % 2 == 1)
        a, b = graph(x), eager(x)
        assert a.shape == (3, 4, 12) and np.array_equal(a, b), i
    assert set(graph._graphs) == {torch.float32, torch.int16}
    graph.listener.close()
    eager.listener.close()


@pytest.mark.gpu
def test_listen_audio_end_to_end_log_mel(tmp_path):
    """listen_audio.py at log-mel features with 30 / 10 ms windows: train a few steps on `synthetic:` data, score two wav files
    at a 30 ms hop and 150 ms chunks, and check every window against tcr_forward on the clip it covers (n = S * K per push)."""
    import torch
    from tcresnet_b200 import listen_audio, train_audio
    from tcresnet_b200.common import checkpoint as ckpt
    from tcresnet_b200.common import model_loader as ML
    from tcresnet_b200.factory import audio_nets
    from test_listener import _write_wav
    t = train_audio.train(train_audio.parse_arguments(shlex.split(
        "--dataset_path synthetic:96 " + LOGMEL_FLAGS + "--dataset_split_name train --augmentation_method "
        "anchored_slice_or_pad_with_shift --batch_size 32 --boundaries 100 --lr_list 0.01 0.005 --absolute_schedule "
        f"--no-boundaries_epoch --step_save_checkpoint 100 --step_evaluation 100 --train_dir {tmp_path / 'train'} "
        "--max_step_from_restore 4 TCResNet8Model --width_multiplier 1.0")))
    t.model.engine.close()
    rng = np.random.default_rng(6)
    a = rng.integers(-20000, 20000, 30001).astype(np.int16)
    b = (6000 * np.sin(2 * np.pi * 700 * np.arange(17003) / 16000.0)).astype(np.int16)
    _write_wav(tmp_path / "a.wav", a)
    _write_wav(tmp_path / "b.wav", b)
    out = tmp_path / "out"
    args = listen_audio.parse_arguments(shlex.split(
        LOGMEL_FLAGS + f"--hop_ms 30 --chunk_ms 150 --checkpoint_path {tmp_path / 'train'} --output_dir {out} TCResNet8Model "
        f"--width_multiplier 1.0 {tmp_path / 'a.wav'} {tmp_path / 'b.wav'}"))
    got = listen_audio.listen(args)
    hop, K, S, T, stride, window = 480, 5, 2, 98, 160, 480
    windows = [-(-30001 // hop), -(-17003 // hop)]
    for name, n, g in zip(("a", "b"), windows, got):
        arr = np.load(out / f"{name}.npy")
        assert arr.shape == (n, 12) and np.array_equal(arr, g)
        rows = (out / f"{name}.csv").read_text().strip().splitlines()
        assert rows[0] == "end_s,class,probability" and len(rows) == n + 1
        assert rows[1].split(",")[0] == "0.030" and int(rows[1].split(",")[1]) == int(arr[0].argmax())
    model = audio_nets.TCResNet8Model(args, None)
    model.build_inference(None, is_training=False)
    values, restore = ML.evaluation_restore(args, ckpt.load(ckpt.resolve_checkpoint_path(str(tmp_path / "train"))),
                                            lambda: model.engine.trainable_names)
    model.set_variables(values, strict=True, restore=restore)
    eng = model._new_engine(S * K)
    assert eng.info.frames == T and eng.info.features == 40
    pre = (T - hop // stride) * stride + (window - stride)
    pushes = -(-max(windows) // K)
    seqs = [np.concatenate([np.zeros(pre, np.float32), x.astype(np.float32) / 32768.0, np.zeros(pushes * K * hop, np.float32)])
            for x in (a, b)]
    for p in range(pushes):
        clips = np.stack([s[k * hop:k * hop + 16000] for s in seqs for k in range(p * K, (p + 1) * K)])
        ref = eng.forward(torch.from_numpy(clips).to(eng.device), model.params, model.moving)["probs"].cpu().numpy().reshape(S, K, 12)
        for i in range(S):
            lo, hi = p * K, min((p + 1) * K, windows[i])
            if lo < hi:
                assert np.array_equal(got[i][lo:hi], ref[i, :hi - lo]), (i, p)
    eng.close()
    model.engine.close()
