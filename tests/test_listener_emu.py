"""The continuous-audio listener on the CPU emulator (tests/emu: the same kernel sources): pushes against tcr_forward on the cut
clips, features in the history against tcr_mfcc_forward bit for bit, and every refusal of tcr_listener_create / _push / _reset.
The GPU runs the same comparison across models, front-ends and stream counts (tests/test_listener.py)."""
import ctypes as C

import numpy as np
import pytest

from listener_cases import Listener, Offline, check_push, pushes_needed, random_chunk, variables
from tcr_harness import Engine, NumpyBackend
from tcresnet_b200 import _lib as L


@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


@pytest.mark.parametrize("hop,K", [(1, 8), (3, 4)])
def test_listener_matches_the_cut_clips(emu, hop, K):
    """T = 49 (the 640 / 320 frame-pair front-end), TCResNet8-1.0, two streams: every push until the zero prefix has left the
    window, then two more."""
    S = 2
    eng = Engine(emu, max_batch=S * K, dropout_keep_prob=1.0)
    T, s = eng.info.frames, eng.cfg.window_stride_samples
    lis = Listener(eng, S, hop, K * hop * s)
    try:
        p_h, m_h = variables(eng, 7)
        p, m = emu.upload(p_h), emu.upload(m_h)
        off = Offline(eng, S, hop)
        rng = np.random.default_rng(hop)
        for i in range(pushes_needed(T, K, hop)):
            check_push(eng, lis, off, random_chunk(rng, S, lis.chunk, pcm=(i % 3 == 2)), p_h, p, m_h, m)
    finally:
        lis.close()
        eng.close()


def test_listener_reset_of_one_stream(emu):
    S, hop, K = 2, 4, 2
    eng = Engine(emu, max_batch=S * K, dropout_keep_prob=1.0)
    lis = Listener(eng, S, hop, K * hop * eng.cfg.window_stride_samples)
    try:
        p_h, m_h = variables(eng, 3)
        p, m = emu.upload(p_h), emu.upload(m_h)
        off = Offline(eng, S, hop)
        rng = np.random.default_rng(0)
        for i in range(4):
            if i == 2:
                lis.reset(1)
                off.reset(1)
            check_push(eng, lis, off, random_chunk(rng, S, lis.chunk, pcm=False), p_h, p, m_h, m)
    finally:
        lis.close()
        eng.close()


def _err(lib):
    return lib.tcr_last_error().decode()


def test_listener_refusals(emu):
    lib = emu.lib
    eng = Engine(emu, max_batch=8)
    T, s = eng.info.frames, eng.cfg.window_stride_samples
    out = C.c_void_p()

    def create(streams, hop, chunk):
        cfg = L.TcrListenerConfig(streams, hop, chunk)
        return lib.tcr_listener_create(eng.h, C.byref(cfg), C.byref(out))

    try:
        assert create(1, 0, s) == 1 and f"hop_frames 0 outside [1, T = {T}]" in _err(lib)
        assert create(1, T + 1, (T + 1) * s) == 1 and f"hop_frames {T + 1} outside [1, T = {T}]" in _err(lib)
        assert create(1, 2, 3 * s) == 1 and f"not a positive multiple of hop_frames * window_stride_samples = {2 * s}" in _err(lib)
        assert create(1, 1, 0) == 1 and "not a positive multiple" in _err(lib)
        assert create(3, 1, 3 * s) == 1 and "streams * windows per push = 3 * 3 exceeds max_batch = 8" in _err(lib)
        assert create(0, 1, s) == 1 and "streams must be at least 1" in _err(lib)
        assert lib.tcr_listener_create(None, None, C.byref(out)) == 1

        lis = Listener(eng, 2, T, 2 * T * s)                   # hop = T: K = 2, nothing carried between pushes
        params, moving = emu.empty(eng.info.num_trainable), emu.empty(eng.info.num_moving)
        buf = np.zeros(2 * lis.chunk + 8, np.float32)
        base = buf.ctypes.data
        aligned = base + (-base) % 16
        push = lambda ptr, kind=L.TCR_INPUT_WAV_F32, prm=params: lib.tcr_listener_push(  # noqa: E731
            lis.p, ptr, kind, emu.ptr(prm), emu.ptr(moving), None, None, None)
        assert push(aligned + 4) == 1 and "samples must be 16-byte aligned" in _err(lib)
        assert push(aligned, kind=L.TCR_INPUT_FEATURES) == 1 and "input_kind 1" in _err(lib)
        assert push(aligned, prm=None) == 1 and "NULL argument" in _err(lib)
        assert lib.tcr_listener_reset(lis.p, 2, None) == 1 and "stream 2 outside [0, 2)" in _err(lib)
        assert lib.tcr_listener_reset(lis.p, -2, None) == 1
        assert lib.tcr_listener_reset(lis.p, -1, None) == 0 and lib.tcr_listener_reset(lis.p, 1, None) == 0
        lis.close()
        assert lib.tcr_listener_destroy(None) == 0
    finally:
        eng.close()

    # int16 input needs window, stride and chunk lengths that are multiples of 8 samples: a 164-sample stride is not one
    eng = Engine(emu, max_batch=2, window_size_samples=480, window_stride_samples=164)
    try:
        lis = Listener(eng, 1, 1, 164)
        pcm = np.zeros(176, np.int16)
        params, moving = emu.empty(eng.info.num_trainable), emu.empty(eng.info.num_moving)
        base = pcm.ctypes.data
        assert base % 16 == 0
        assert lib.tcr_listener_push(lis.p, base, L.TCR_INPUT_WAV_PCM16, emu.ptr(params), emu.ptr(moving), None, None, None) == 3
        assert "multiples of 8 samples" in _err(lib)
        lis.close()
    finally:
        eng.close()
