"""The continuous-audio listener on the GPU (include/tcr_b200.h, tcr_listener_*): every push equals tcr_forward on the clips cut
from the zero-prefixed streams at the same batch size, bit for bit, and the carried features equal tcr_mfcc_forward's, across
models, both front-end kernels, hops and stream counts; then the fp64 oracle once, the CUDA-graph StreamingModel and
listen_audio.py end to end."""
import os
import shlex
import wave

import numpy as np
import pytest

from listener_cases import Listener, Offline, check_push, pushes_needed, random_chunk, variables
from oracle import tcr_oracle as O
from parity_cases import TOL_LOGITS, check_argmax, perturbed_variables, reference_features
from tcr_harness import Engine, rel_err

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


PAIR = dict(window_size_samples=640, window_stride_samples=320)       # 40 / 20 ms, T = 49: the frame-pair front-end
ONE = dict(window_size_samples=480, window_stride_samples=160)        # 30 / 10 ms, T = 98: the one-frame-per-warp kernel
# (name, model, width, front-end, hop ("T": the clip length), streams, windows per push, environment)
CASES = []
for model, wm in ((8, 1.0), (14, 1.5), (8, 2.5)):
    for hop, S, K in ((1, 37, 5), (2, 3, 4), (3, 1, 3), ("T", 3, 2)):
        CASES.append((f"r{model}-{wm}-pair-hop{hop}-S{S}", model, wm, PAIR, hop, S, K, {}))
for hop, S, K in ((1, 37, 10), (2, 3, 5), (3, 37, 2), ("T", 1, 2)):
    CASES.append((f"r8-1.0-onekernel-T98-hop{hop}-S{S}", 8, 1.0, ONE, hop, S, K, {}))
for hop, S, K in ((1, 3, 5), (3, 37, 3)):
    CASES.append((f"r8-1.0-pair-off-hop{hop}-S{S}", 8, 1.0, PAIR, hop, S, K, {"TCR_MFCC_PAIR": "0"}))


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_listener_matches_the_cut_clips(cuda, monkeypatch, case):
    """Pushes alternate fp32 and int16 until the zero prefix has left the window, then two more; with several streams, one of
    them is reset halfway and the others carry on."""
    _, model, wm, fe, hop, S, K, env = case
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    eng = Engine(cuda, model=model, width_multiplier=wm, max_batch=S * K, dropout_keep_prob=1.0, **fe)
    T = eng.info.frames
    hop = T if hop == "T" else hop
    lis = Listener(eng, S, hop, K * hop * eng.cfg.window_stride_samples)
    try:
        p_h, m_h = variables(eng, 11)
        p, m = cuda.upload(p_h), cuda.upload(m_h)
        off = Offline(eng, S, hop)
        rng = np.random.default_rng(model + hop)
        n = pushes_needed(T, K, hop)
        for i in range(n):
            if S > 1 and i == n // 2:
                lis.reset(S // 2)
                off.reset(S // 2)
            check_push(eng, lis, off, random_chunk(rng, S, lis.chunk, pcm=i % 2 == 1), p_h, p, m_h, m)
    finally:
        lis.close()
        eng.close()


def test_training_step_between_pushes(cuda):
    """A training step on the handle between two pushes: the next push scores with the new variables and the stream continues
    from the history the step did not touch."""
    S, hop, K = 3, 2, 5
    eng = Engine(cuda, max_batch=64, dropout_keep_prob=1.0)
    lis = Listener(eng, S, hop, K * hop * eng.cfg.window_stride_samples)
    try:
        p_h, m_h = variables(eng, 5)
        off = Offline(eng, S, hop)
        rng = np.random.default_rng(1)
        for i in range(8):
            if i in (3, 6):
                wav, onehot = O.synthetic_batch(64)
                r = eng.train_step(wav.astype(np.float32), onehot.astype(np.float32), p_h, np.zeros_like(p_h), m_h, lr=0.05)
                assert not np.array_equal(r["params"], p_h)
                p_h, m_h = r["params"], r["moving"]
            p, m = cuda.upload(p_h), cuda.upload(m_h)
            check_push(eng, lis, off, random_chunk(rng, S, lis.chunk, pcm=False), p_h, p, m_h, m)
    finally:
        lis.close()
        eng.close()


def test_listener_against_the_fp64_oracle(cuda):
    S, hop, K = 4, 3, 4
    eng = Engine(cuda, max_batch=S * K, dropout_keep_prob=1.0)
    T, F = eng.info.frames, eng.info.features
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
        ref, _ = O.forward(spec, params, moving, reference_features(clips.astype(np.float64), 640, 320), False)
        got = logits.reshape(S * K, -1)
        err = rel_err(got, ref)
        assert err <= TOL_LOGITS, err
        check_argmax(got, ref, err * np.abs(ref).max())
        np.testing.assert_allclose(probs.reshape(S * K, -1), O.softmax(ref), rtol=0, atol=2e-5)
    finally:
        lis.close()
        eng.close()


def _model_args(extra=""):
    from tcresnet_b200 import listen_audio
    return listen_audio.parse_arguments(shlex.split(
        "--output_name output/softmax --num_classes 12 --preprocess_method mfcc --num_mfccs 40 --clip_duration_ms 1000 "
        f"--window_size_ms 40 --window_stride_ms 20 {extra} TCResNet8Model --width_multiplier 1.0 unused.wav"))


def test_streaming_model_graph_replay_equals_eager(cuda):
    import torch
    from tcresnet_b200.factory import audio_nets
    model = audio_nets.TCResNet8Model(_model_args(), None)
    graph = model.build_streaming_model(streams=3, hop_ms=20, chunk_ms=100)
    eager = audio_nets.StreamingModel(model, graph.engine, 3, 1, 1600, use_graph=False)
    rng = np.random.default_rng(3)
    for i in range(6):
        x = random_chunk(rng, 3, 1600, pcm=i % 2 == 1)
        a, b = graph(x), eager(x)
        assert a.shape == (3, 5, 12) and np.array_equal(a, b), i
    assert set(graph._graphs) == {torch.float32, torch.int16}
    graph.listener.close()
    eager.listener.close()


def _write_wav(path, samples):
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(16000)
        w.writeframes(np.ascontiguousarray(samples, "<i2").tobytes())


def test_listen_audio_end_to_end(tmp_path):
    """Train a few steps on `synthetic:` data, score two generated wav files with listen_audio.py, and check every window against
    tcr_forward on the clip it covers (same batch grouping as the listener's pushes)."""
    import torch
    from tcresnet_b200 import listen_audio, train_audio
    from tcresnet_b200.common import checkpoint as ckpt
    from tcresnet_b200.common import model_loader as ML
    from tcresnet_b200.factory import audio_nets
    common = ("--dataset_path synthetic:96 --output_name output/softmax --num_classes 12 --preprocess_method mfcc "
              "--num_mfccs 40 --clip_duration_ms 1000 --window_size_ms 40 --window_stride_ms 20 ")
    t = train_audio.train(train_audio.parse_arguments(shlex.split(
        common + f"--dataset_split_name train --augmentation_method anchored_slice_or_pad_with_shift --batch_size 32 --boundaries 100 "
        f"--lr_list 0.01 0.005 --absolute_schedule --no-boundaries_epoch --step_save_checkpoint 100 --step_evaluation 100 "
        f"--train_dir {tmp_path / 'train'} --max_step_from_restore 4 TCResNet8Model --width_multiplier 1.0")))
    t.model.engine.close()
    rng = np.random.default_rng(4)
    t_ax = np.arange(37000) / 16000.0
    a = (8000 * np.sin(2 * np.pi * 440 * t_ax) * (t_ax > 0.7) + rng.normal(0, 300, t_ax.size)).astype(np.int16)
    b = rng.integers(-20000, 20000, 23101).astype(np.int16)
    _write_wav(tmp_path / "a.wav", a)
    _write_wav(tmp_path / "b.wav", b)
    out = tmp_path / "out"
    args = listen_audio.parse_arguments(shlex.split(
        "--output_name output/softmax --num_classes 12 --preprocess_method mfcc --num_mfccs 40 --clip_duration_ms 1000 "
        f"--window_size_ms 40 --window_stride_ms 20 --hop_ms 40 --chunk_ms 200 --checkpoint_path {tmp_path / 'train'} "
        f"--output_dir {out} TCResNet8Model --width_multiplier 1.0 {tmp_path / 'a.wav'} {tmp_path / 'b.wav'}"))
    got = listen_audio.listen(args)
    hop, K, S = 640, 5, 2
    windows = [-(-37000 // hop), -(-23101 // hop)]
    for name, n, g in zip(("a", "b"), windows, got):
        arr = np.load(out / f"{name}.npy")
        assert arr.shape == (n, 12) and np.array_equal(arr, g)
        rows = (out / f"{name}.csv").read_text().strip().splitlines()
        assert rows[0] == "end_s,class,probability" and len(rows) == n + 1
        assert rows[1].split(",")[0] == "0.040" and int(rows[1].split(",")[1]) == int(arr[0].argmax())
    # per-window tcr_forward with the restored variables, n = S * K per push like the listener
    model = audio_nets.TCResNet8Model(args, None)
    model.build_inference(None, is_training=False)
    values, restore = ML.evaluation_restore(args, ckpt.load(ckpt.resolve_checkpoint_path(str(tmp_path / "train"))),
                                            lambda: model.engine.trainable_names)
    model.set_variables(values, strict=True, restore=restore)
    eng = model._new_engine(S * K)
    pre = (49 - hop // 320) * 320 + (640 - 320)               # (T - hop_frames) * stride + (window - stride) zeros
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
