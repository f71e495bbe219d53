"""The listener (tcr_listener_*) against the offline computation it promises (include/tcr_b200.h): each stream is the zero-prefixed
concatenation of its pushes, and window k is the clip that starts at sample k * hop * stride of it, scored by tcr_forward in
evaluation mode at the same batch size.  Shared by the emulator tests and the -m gpu tests."""
from __future__ import annotations

import ctypes as C

import numpy as np

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L


class Listener:
    """tcr_listener_* over a tests/tcr_harness.Engine (NumPy buffers on the emulator, torch CUDA tensors on the GPU)."""

    def __init__(self, eng, streams, hop, chunk):
        self.eng, self.b, self.lib = eng, eng.b, eng.lib
        self.p = C.c_void_p()
        cfg = L.TcrListenerConfig(streams, hop, chunk)
        L.check(self.lib, self.lib.tcr_listener_create(eng.h, C.byref(cfg), C.byref(self.p)), "tcr_listener_create")
        self.S, self.hop, self.chunk = streams, hop, chunk
        self.K = chunk // (hop * eng.cfg.window_stride_samples)

    def close(self):
        if self.p:
            self.lib.tcr_listener_destroy(self.p)
            self.p = C.c_void_p()

    def reset(self, stream=-1):
        L.check(self.lib, self.lib.tcr_listener_reset(self.p, stream, self.b.stream), "tcr_listener_reset")

    def push(self, samples, params, moving):
        """samples: host [S, chunk] fp32 or int16; params / moving: backend buffers.  Returns host (logits, probs) [S, K, C]."""
        b, nc = self.b, self.eng.cfg.num_classes
        x = b.upload(samples)
        kind = L.TCR_INPUT_WAV_PCM16 if np.asarray(samples).dtype == np.int16 else L.TCR_INPUT_WAV_F32
        logits, probs = b.empty(self.S, self.K, nc), b.empty(self.S, self.K, nc)
        L.check(self.lib, self.lib.tcr_listener_push(self.p, b.ptr(x), kind, b.ptr(params), b.ptr(moving), b.ptr(logits), b.ptr(probs),
                                                     b.stream), "tcr_listener_push")
        b.sync()
        return b.download(logits), b.download(probs)

    def history(self):
        ptr, frames = C.c_void_p(), C.c_int32()
        L.check(self.lib, self.lib.tcr_listener_history(self.p, C.byref(ptr), C.byref(frames)), "tcr_listener_history")
        self.b.sync()
        f = self.eng.info.features
        return self.b.view(ptr.value, self.S * frames.value * f).reshape(self.S, frames.value, f)


class Offline:
    """What the streams hold: pre = (T - hop) * stride + (window - stride) zeros after a reset, then every pushed chunk."""

    def __init__(self, eng, streams, hop):
        c = eng.cfg
        self.T, self.stride, self.clip, self.hop = eng.info.frames, c.window_stride_samples, c.clip_samples, hop
        self.pre = (self.T - hop) * self.stride + (c.window_size_samples - self.stride)
        self.seq = [np.zeros(self.pre, np.float32) for _ in range(streams)]
        self.k = [0] * streams

    def reset(self, s):
        self.seq[s], self.k[s] = np.zeros(self.pre, np.float32), 0

    def push(self, samples):
        """The clips of the windows this push emits, [S, K, clip] fp32 (int16 decoded as decode_wav does)."""
        x = np.asarray(samples)
        x = x.astype(np.float32) / np.float32(32768.0) if x.dtype == np.int16 else x.astype(np.float32)
        step = self.hop * self.stride
        K = x.shape[1] // step
        out = np.empty((len(self.seq), K, self.clip), np.float32)
        for s in range(len(self.seq)):
            self.seq[s] = np.concatenate([self.seq[s], x[s]])
            for j in range(K):
                k = self.k[s] + j
                out[s, j] = self.seq[s][k * step:k * step + self.clip]
            self.k[s] += K
        return out


def variables(eng, seed):
    """Initial variables with the BatchNorm statistics and affine terms moved away from (0, 1), so every layer's table matters."""
    b = eng.b
    params, slots, moving = b.empty(eng.info.num_trainable), b.empty(eng.info.num_trainable), b.empty(eng.info.num_moving)
    L.check(eng.lib, eng.lib.tcr_init_variables(eng.h, b.ptr(params), b.ptr(slots), b.ptr(moving), seed, b.stream), "init")
    p, m = b.download(params), b.download(moving)
    rng = np.random.default_rng(seed)
    for d in eng.param_table():
        sl = slice(d["offset"], d["offset"] + d["numel"])
        if d["kind"] in (1, 2):
            p[sl] += rng.normal(0, 0.1, d["numel"]).astype(np.float32)
        elif d["kind"] == 3:
            m[sl] = rng.normal(0, 0.2, d["numel"]).astype(np.float32)
        elif d["kind"] == 4:
            m[sl] = rng.uniform(0.5, 2.0, d["numel"]).astype(np.float32)
    return p, m


def random_chunk(rng, streams, chunk, pcm):
    if pcm:
        return rng.integers(-32768, 32768, (streams, chunk)).astype(np.int16)
    x = rng.uniform(-1.0, 1.0, (streams, chunk)).astype(np.float32)
    x[:, : chunk // 4] *= np.float32(0.01)           # quiet and loud stretches, so windows differ in level
    return x


def check_push(eng, lis, off, samples, params_h, params, moving_h, moving):
    """One push against tcr_forward on the cut clips at n = S * K: logits and probs equal bit for bit, and the carried history
    equal bit for bit to tcr_mfcc_forward's last T - hop frames of each stream's last window.  Returns the push's probs."""
    logits, probs = lis.push(samples, params, moving)
    clips = off.push(samples)
    S, K, clip = clips.shape
    ref = eng.forward(clips.reshape(S * K, clip), params_h, moving_h)
    nc = eng.cfg.num_classes
    assert np.array_equal(logits.reshape(S * K, nc), ref["logits"]), np.abs(logits.reshape(S * K, nc) - ref["logits"]).max()
    assert np.array_equal(probs.reshape(S * K, nc), ref["probs"])
    carried = off.T - off.hop
    if carried:
        feats = eng.mfcc(np.ascontiguousarray(clips[:, K - 1]))
        assert np.array_equal(lis.history()[:, :carried], feats[:, off.hop:])
    return probs


def pushes_needed(T, K, hop):
    """Enough pushes that the zero prefix has left the window completely, plus two."""
    return -(-T // (K * hop)) + 2
