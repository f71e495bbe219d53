"""The listener on a DS-CNN handle (tcr_dscnn_listener_create): every push against tcr_dscnn_forward_input on the clips cut from the
zero-prefixed streams at the same n, bit for bit, and the carried history against tcr_dscnn_mfcc_forward.  conv_1 reads each
window in place from the history (the windowed dscnn_conv* instantiations).  The FMA kernel on the CPU emulator; S / M / L and
every TCR_DSCNN_TC mode, graph replay and listen_audio.py on the GPU."""
import ctypes as C
import shlex

import numpy as np
import pytest

from listener_cases import Listener, Offline, pushes_needed, random_chunk, variables
from tcr_harness import Engine, NumpyBackend, launched
from test_dscnn_eval import FRONTENDS, MODES, Ds

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L


class DsListener(Listener):
    """listener_cases.Listener on a DS-CNN handle: created by tcr_dscnn_listener_create, pushed with moving = NULL."""

    def __init__(self, ds, streams, hop, chunk):
        self.eng, self.b, self.lib = ds, ds.b, ds.lib
        self.p = C.c_void_p()
        cfg = L.TcrListenerConfig(streams, hop, chunk)
        L.check(self.lib, self.lib.tcr_dscnn_listener_create(ds.h, C.byref(cfg), C.byref(self.p)), "tcr_dscnn_listener_create")
        self.S, self.hop, self.chunk = streams, hop, chunk
        self.K = chunk // (hop * ds.cfg.window_stride_samples)

    def push(self, samples, params=None, moving=None):
        b, nc = self.b, self.eng.classes
        x = b.upload(samples)
        kind = L.TCR_INPUT_WAV_PCM16 if np.asarray(samples).dtype == np.int16 else L.TCR_INPUT_WAV_F32
        logits, probs = b.empty(self.S, self.K, nc), b.empty(self.S, self.K, nc)
        L.check(self.lib, self.lib.tcr_listener_push(self.p, b.ptr(x), kind, b.ptr(self.eng.params), None, b.ptr(logits), b.ptr(probs),
                                                     b.stream), "tcr_listener_push")
        b.sync()
        return b.download(logits), b.download(probs)


def check_ds_push(ds, lis, off, samples):
    logits, probs = lis.push(samples)
    cut = off.push(samples)
    S, K, clip = cut.shape
    ref_logits, ref_probs = ds.wav_forward(cut.reshape(S * K, clip))
    assert np.array_equal(logits.reshape(S * K, -1), ref_logits), np.abs(logits.reshape(S * K, -1) - ref_logits).max()
    assert np.array_equal(probs.reshape(S * K, -1), ref_probs)
    carried = off.T - off.hop
    if carried:
        feats = ds.mfcc(np.ascontiguousarray(cut[:, K - 1]))
        assert np.array_equal(lis.history()[:, :carried], feats[:, off.hop:])


def run_case(b, size, case, S, hop, K, pushes=None, reset_at=(), pcm_every=3, seed=0):
    """case: a key of FRONTENDS, or a dict of front-end flags."""
    ds = Ds(b, size, FRONTENDS[case] if isinstance(case, str) else case, S * K, seed=seed)
    lis = DsListener(ds, S, hop, K * hop * ds.cfg.window_stride_samples)
    try:
        off = Offline(ds, S, hop)
        rng = np.random.default_rng(seed)
        for i in range(pushes or pushes_needed(ds.T, K, hop)):
            for r in (x for at, x in reset_at if at == i):
                lis.reset(r)
                for s in (range(S) if r == -1 else [r]):
                    off.reset(s)
            check_ds_push(ds, lis, off, random_chunk(rng, S, lis.chunk, pcm=(i % pcm_every == pcm_every - 1)))
    finally:
        lis.close()
        ds.close()


@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


def test_emulated_windows_of_two_streams_in_one_batch(emu):
    """S * K = 9 (odd), 49 x 10: windows of neighbouring streams side by side in the batch; fp32 and int16 pushes, reset of all
    streams and of the last one.  The history rows are 10 floats wide, so the carried frames move in floats, not float4s."""
    run_case(emu, "S", "49x10", S=3, hop=3, K=3, pushes=5, reset_at=((2, -1), (3, 2)), pcm_every=2)


def test_emulated_hop_t_minus_one_and_pushes_longer_than_a_clip(emu):
    run_case(emu, "S", "49x10", S=1, hop=48, K=2, pushes=3, reset_at=((1, 0),), pcm_every=2)


def test_emulated_one_window_per_hop_of_one_frame(emu):
    run_case(emu, "S", "49x40", S=2, hop=1, K=1, pushes=4, pcm_every=2)


def test_emulated_tcresnet_and_dscnn_listeners_alternate(emu):
    """A TC-ResNet listener and a DS-CNN listener pushed in turn on one stream: each keeps its own state and matches its model."""
    from listener_cases import check_push
    eng = Engine(emu, max_batch=4, dropout_keep_prob=1.0)
    ds = Ds(emu, "S", FRONTENDS["49x40"], 4, seed=1)
    tl = Listener(eng, 2, 2, 2 * 2 * eng.cfg.window_stride_samples)
    dl = DsListener(ds, 2, 3, 2 * 3 * ds.cfg.window_stride_samples)
    try:
        p_h, m_h = variables(eng, 5)
        p, m = emu.upload(p_h), emu.upload(m_h)
        t_off, d_off = Offline(eng, 2, 2), Offline(ds, 2, 3)
        rng = np.random.default_rng(3)
        for i in range(3):
            check_push(eng, tl, t_off, random_chunk(rng, 2, tl.chunk, pcm=i == 1), p_h, p, m_h, m)
            check_ds_push(ds, dl, d_off, random_chunk(rng, 2, dl.chunk, pcm=i == 2))
    finally:
        tl.close()
        dl.close()
        ds.close()
        eng.close()


def test_emulated_refusals(emu):
    lib = emu.lib
    ds = Ds(emu, "S", FRONTENDS["49x10"], 4)
    out = C.c_void_p()
    try:
        cfg = L.TcrListenerConfig(3, 1, 2 * 320)
        assert lib.tcr_dscnn_listener_create(ds.h, C.byref(cfg), C.byref(out)) == 1
        assert "streams * windows per push = 3 * 2 exceeds max_batch = 4" in lib.tcr_last_error().decode()
        lis = DsListener(ds, 1, 49, 49 * 320)
        x = np.zeros(49 * 320, np.float32)
        moving = np.zeros(4, np.float32)
        assert lib.tcr_listener_push(lis.p, x.ctypes.data, 0, emu.ptr(ds.params), moving.ctypes.data, None, None, None) == 1
        assert "moving = NULL" in lib.tcr_last_error().decode()
        lis.close()
    finally:
        ds.close()


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


def _mode(monkeypatch, mode):
    if MODES[mode] is None:
        monkeypatch.delenv("TCR_DSCNN_TC", raising=False)
    else:
        monkeypatch.setenv("TCR_DSCNN_TC", MODES[mode])


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("size", ["S", "M", "L"])
@pytest.mark.parametrize("case", ["49x10", "49x40"])
def test_cuda_listener_matches_the_cut_clips(cuda, monkeypatch, case, size, mode):
    """13 streams x 3 windows (39: odd, so wgmma tiles hold windows of two streams), hop 3, until the zero prefix has left the
    window; int16 every third push; a reset of every stream and of the last one."""
    _mode(monkeypatch, mode)
    run_case(cuda, size, case, S=13, hop=3, K=3, reset_at=((3, -1), (5, 12)))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
def test_cuda_listener_geometries(cuda, monkeypatch, mode):
    _mode(monkeypatch, mode)
    run_case(cuda, "S", "49x10", S=5, hop=48, K=2, pushes=4, reset_at=((2, 4),))       # hop = T - 1, K * hop > T
    run_case(cuda, "S", "49x40", S=7, hop=1, K=1, pushes=6)                           # K = hop = 1
    run_case(cuda, "S", "49x40", S=128, hop=2, K=4, pushes=5, pcm_every=2)            # n = 512


@pytest.mark.gpu
def test_cuda_windowed_conv_kernels_run(cuda, monkeypatch):
    """The push's conv_1 launch is the windowed instantiation of the kernel the mode selects."""
    for mode, name in (("fma", "dscnn_conv:win"), ("lockstep", "dscnn_conv_tc:win"), ("default", "dscnn_conv_ws:win")):
        _mode(monkeypatch, mode)
        ds = Ds(cuda, "S", FRONTENDS["49x10"], 8)
        lis = DsListener(ds, 2, 2, 2 * 2 * 320)
        got = launched(cuda.lib, lambda: lis.push(np.zeros((2, lis.chunk), np.float32)))
        assert got[name] == 1 and not any(k in got for k in ("dscnn_conv", "dscnn_conv_tc", "dscnn_conv_ws")), got
        lis.close()
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["DSCNNSModel", "DSCNNMModel"])
def test_streaming_model_and_listen_audio(cuda, tmp_path, model):
    """build_streaming_model: two eager pushes, then graph replay, each equal to forward_input on the cut clips; listen_audio.py on
    a DS-CNN checkpoint writes the same softmaxes."""
    import torch
    from test_listener import _write_wav
    from tcresnet_b200 import evaluate_audio, listen_audio
    from tcresnet_b200.common import checkpoint as ckpt
    from tcresnet_b200.factory import audio_nets
    flags = ("--output_name output/softmax --num_classes 12 --preprocess_method mfcc --num_mfccs 10 --clip_duration_ms 1000 "
             "--window_size_ms 40 --window_stride_ms 20")
    args = evaluate_audio.parse_arguments(shlex.split(f"--dataset_path synthetic:8 --dataset_split_name valid --checkpoint_path x "
                                                      f"--batch_size 1 --augmentation_method anchored_slice_or_pad {flags} {model}"))
    m = getattr(audio_nets, model)(args, None)
    sm = m.build_streaming_model(streams=3, hop_ms=40, chunk_ms=120)
    assert (sm.hop_frames, sm.windows) == (2, 3)
    off = Offline(type("E", (), dict(cfg=m.engine.cfg, info=m.engine.info)), 3, 2)
    rng = np.random.default_rng(0)
    for i in range(5):
        x = random_chunk(rng, 3, sm.chunk_samples, pcm=i == 3)
        got = sm(x)
        cut = off.push(x).reshape(9, -1)
        ref = sm.engine.forward_input(torch.from_numpy(cut).cuda(), m.params)[1].cpu().numpy().reshape(3, 3, -1)
        assert np.array_equal(got, ref), i
    sm.listener.close()
    # listen_audio.py: a checkpoint under the reference's names, one file
    from oracle import dscnn_oracle as D
    spec = D.build_spec(m.dscnn_size, 49, 10, 12)
    values = {k: v.astype(np.float32) for k, v in D.init_variables(spec, 2).items()}
    path = ckpt.save(tmp_path / "run", model, 100, values, fmt="tf")
    wav = rng.integers(-20000, 20000, 12000).astype(np.int16)
    _write_wav(tmp_path / "a.wav", wav)
    la = listen_audio.parse_arguments(shlex.split(f"--checkpoint_path {path} --hop_ms 40 --chunk_ms 120 --output_dir {tmp_path / 'out'} "
                                                  f"{flags} {model} {tmp_path / 'a.wav'}"))
    probs = listen_audio.listen(la)[0]
    assert probs.shape == (-(-12000 // 640), 12) and np.allclose(probs.sum(1), 1, atol=1e-5)
    m.set_variables(values)
    off = Offline(type("E", (), dict(cfg=m.engine.cfg, info=m.engine.info)), 1, 2)
    pushes = -(-probs.shape[0] // 3)
    stream = np.zeros((1, pushes * 1920), np.float32)
    stream[0, :12000] = wav.astype(np.float32) / 32768.0
    cut = np.concatenate([off.push(stream[:, p * 1920:(p + 1) * 1920]) for p in range(pushes)], axis=1)[0][:probs.shape[0]]
    ref = np.concatenate([sm.engine.forward_input(torch.from_numpy(np.ascontiguousarray(cut[i:i + 3])).cuda(), m.params)[1].cpu().numpy()
                          for i in range(0, cut.shape[0], 3)])
    assert np.array_equal(probs, ref)
    sm.engine.close()
    m.engine.close()
