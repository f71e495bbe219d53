"""Test harness over the C ABI: the same parity code drives
  * the product library libtcr_b200.so with torch CUDA tensors (``-m gpu`` tests), and
  * the TEST-ONLY emulator build tests/emu/libtcr_emu.so with NumPy buffers (kernel logic on a CPU box).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from collections import Counter

import numpy as np

import tcresnet_b200  # noqa: F401  (registers the package alias)
from tcresnet_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_DIR = os.path.join(ROOT, "tests", "emu")
EMU_LIB = os.path.join(EMU_DIR, "libtcr_emu.so")


def build_emu():
    subprocess.run(["make", "-s", "-C", EMU_DIR], check=True)
    return EMU_LIB


class NumpyBackend:
    name = "emu"
    stream = None

    def __init__(self):
        self.lib = L.load(build_emu())

    def empty(self, *shape):
        return np.full(shape, np.nan, np.float32)

    def upload(self, a):
        a = np.asarray(a)
        return np.ascontiguousarray(a, dtype=np.int16 if a.dtype == np.int16 else np.float32).copy()

    def upload_bytes(self, a):
        return np.ascontiguousarray(a, np.uint8).copy()

    def download(self, a):
        return np.array(a, copy=True)

    def ptr(self, a):
        return None if a is None else a.ctypes.data

    def view(self, ptr, numel):
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_float)), shape=(numel,)).copy()

    def sync(self):
        pass


class TorchBackend:
    name = "cuda"

    def __init__(self):
        import torch
        self.torch = torch
        self.lib = L.load()
        self.dev = torch.device("cuda:0")

    @property
    def stream(self):
        return self.torch.cuda.current_stream().cuda_stream

    def empty(self, *shape):
        return self.torch.full(shape, float("nan"), dtype=self.torch.float32, device=self.dev)

    def upload(self, a):
        a = np.asarray(a)
        return self.torch.from_numpy(np.ascontiguousarray(a, dtype=np.int16 if a.dtype == np.int16 else np.float32)).to(self.dev)

    def upload_bytes(self, a):
        return self.torch.from_numpy(np.ascontiguousarray(a, np.uint8).copy()).to(self.dev)

    def download(self, a):
        return a.detach().cpu().numpy()

    def ptr(self, a):
        return None if a is None else a.data_ptr()

    def view(self, ptr, numel):
        out = self.torch.empty(numel, dtype=self.torch.float32, device=self.dev)
        self.torch.cuda.synchronize()
        rt = C.CDLL("libcudart.so.12")                                # already mapped by torch
        rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
        assert rt.cudaMemcpy(out.data_ptr(), ptr, numel * 4, 3) == 0   # device-to-device
        return out.cpu().numpy()

    def sync(self):
        self.torch.cuda.synchronize()


class Engine:
    """Thin handle wrapper used by the tests (the product-side wrapper is tc-resnet_b200/engine.py)."""

    def __init__(self, backend, **cfg):
        self.b = backend
        self.lib = backend.lib
        c = L.TcrConfig()
        L.check(self.lib, self.lib.tcr_config_default(C.byref(c)), "tcr_config_default")
        for k, v in cfg.items():
            if not hasattr(c, k):
                raise KeyError(k)
            setattr(c, k, v)
        self.cfg = c
        self.h = C.c_void_p()
        L.check(self.lib, self.lib.tcr_create(C.byref(c), C.byref(self.h)), "tcr_create")
        self.info = L.TcrInfo()
        L.check(self.lib, self.lib.tcr_get_info(self.h, C.byref(self.info)), "tcr_get_info")

    def close(self):
        if self.h:
            self.lib.tcr_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def param_table(self):
        descs = C.POINTER(L.TcrParamDesc)()
        n = C.c_int32()
        L.check(self.lib, self.lib.tcr_param_table(self.h, C.byref(descs), C.byref(n)), "tcr_param_table")
        return [dict(name=descs[i].name.decode(), kind=descs[i].kind, shape=tuple(descs[i].shape[:descs[i].rank]),
                     offset=descs[i].offset, numel=descs[i].numel) for i in range(n.value)]

    def mfcc(self, wav_np):
        b = self.b
        n = wav_np.shape[0]
        wav = b.upload(wav_np)
        feat = b.empty(n, self.info.frames, self.info.features)
        fn = self.lib.tcr_mfcc_forward_pcm16 if np.asarray(wav_np).dtype == np.int16 else self.lib.tcr_mfcc_forward
        L.check(self.lib, fn(self.h, b.ptr(wav), b.ptr(feat), n, b.stream), "tcr_mfcc_forward")
        b.sync()
        return b.download(feat)

    def augment(self, pcm_np, clips_np, background_np):
        """tcr_augment_pcm16 through the C ABI: int16 clips + packed tcr_augment_clip records (+ background) -> fp32 wav."""
        b = self.b
        n = pcm_np.shape[0]
        pcm = b.upload(np.ascontiguousarray(pcm_np, np.int16))
        clips = b.upload_bytes(np.frombuffer(np.ascontiguousarray(clips_np).tobytes(), np.uint8))
        bg = b.upload(background_np) if background_np is not None else None
        out = b.empty(n, self.cfg.clip_samples)
        L.check(self.lib, self.lib.tcr_augment_pcm16(self.h, b.ptr(pcm), pcm_np.shape[1], b.ptr(clips), b.ptr(bg), b.ptr(out), n, b.stream),
                "tcr_augment_pcm16")
        b.sync()
        return b.download(out)

    def forward(self, inp_np, params_np, moving_np=None, is_features=False, is_training=False, seed=0, mask_np=None,
                onehot_np=None, weight_decay=0.0):
        b = self.b
        n = inp_np.shape[0]
        inp, params = b.upload(inp_np), b.upload(params_np)
        moving = b.upload(moving_np) if moving_np is not None else None
        mask = b.upload(mask_np) if mask_np is not None else None
        onehot = b.upload(onehot_np) if onehot_np is not None else None
        nc = self.cfg.num_classes
        logits, probs, losses = b.empty(n, nc), b.empty(n, nc), b.empty(2)
        kind = 1 if is_features else (2 if np.asarray(inp_np).dtype == np.int16 else 0)
        L.check(self.lib, self.lib.tcr_forward(self.h, b.ptr(inp), kind, b.ptr(params), b.ptr(moving), n,
                                               int(is_training), seed, b.ptr(mask), b.ptr(onehot), weight_decay,
                                               b.ptr(logits), b.ptr(probs), b.ptr(losses) if onehot is not None else None,
                                               b.stream), "tcr_forward")
        b.sync()
        return dict(logits=b.download(logits), probs=b.download(probs), losses=b.download(losses))

    def train_step(self, inp_np, onehot_np, params_np, slots_np, moving_np, lr=0.1, momentum=0.9, weight_decay=1e-3,
                   is_features=False, seed=0, mask_np=None, apply_update=True, clips_np=None, background_np=None):
        b = self.b
        n = inp_np.shape[0]
        inp, onehot = b.upload(inp_np), b.upload(onehot_np)
        params, slots, moving = b.upload(params_np), b.upload(slots_np), b.upload(moving_np)
        mask = b.upload(mask_np) if mask_np is not None else None
        nc = self.cfg.num_classes
        logits, probs, losses = b.empty(n, nc), b.empty(n, nc), b.empty(2)
        grads = b.empty(self.info.num_trainable)
        a = L.TcrStepArgs()
        kind = 1 if is_features else (2 if np.asarray(inp_np).dtype == np.int16 else 0)
        a.input, a.input_is_features, a.onehot, a.n = b.ptr(inp), kind, b.ptr(onehot), n
        if clips_np is not None:          # device input stage inside the step: int16 rows + packed tcr_augment_clip records
            clips = b.upload_bytes(np.frombuffer(np.ascontiguousarray(clips_np).tobytes(), np.uint8))
            bg = b.upload(background_np) if background_np is not None else None
            a.clips, a.background, a.pcm_stride = b.ptr(clips), b.ptr(bg), inp_np.shape[1]
        a.params, a.slots, a.moving = b.ptr(params), b.ptr(slots), b.ptr(moving)
        a.learning_rate, a.momentum, a.weight_decay = lr, momentum, weight_decay
        a.dropout_seed, a.dropout_mask = seed, b.ptr(mask)
        a.losses, a.logits, a.probs, a.grads = b.ptr(losses), b.ptr(logits), b.ptr(probs), b.ptr(grads)
        a.apply_update = int(apply_update)
        L.check(self.lib, self.lib.tcr_train_step(self.h, C.byref(a), b.stream), "tcr_train_step")
        b.sync()
        return dict(logits=b.download(logits), probs=b.download(probs), losses=b.download(losses),
                    grads=b.download(grads), params=b.download(params), slots=b.download(slots),
                    moving=b.download(moving))

    def eval_accumulate(self, scores_np, onehot_np, topk=5, counts_np=None):
        """tcr_eval_accumulate through the C ABI: returns the accumulated int64 counts [C*C + 2]."""
        b = self.b
        n, c = scores_np.shape
        scores, onehot = b.upload(scores_np), b.upload(onehot_np)
        init = np.zeros(c * c + 2, np.int64) if counts_np is None else np.asarray(counts_np, np.int64)
        if b.name == "cuda":
            counts = b.torch.from_numpy(init.copy()).to(b.dev)
            ptr = counts.data_ptr()
        else:
            counts = init.copy()
            ptr = counts.ctypes.data
        L.check(self.lib, self.lib.tcr_eval_accumulate(self.h, b.ptr(scores), b.ptr(onehot), n, topk, ptr, b.stream), "tcr_eval_accumulate")
        b.sync()
        return counts.cpu().numpy() if b.name == "cuda" else counts

    def workspace(self, name):
        p = C.c_void_p()
        numel = C.c_int64()
        L.check(self.lib, self.lib.tcr_workspace_tensor(self.h, name.encode(), C.byref(p), C.byref(numel)),
                f"tcr_workspace_tensor({name})")
        return self.b.view(p.value, numel.value)


def launched(lib, fn):
    """Kernel launches of one call, {name: count}, from the library's launch profiler (CUDA build only)."""
    L.check(lib, lib.tcr_profile_enable(1), "tcr_profile_enable")
    try:
        fn()
        stats, count = C.POINTER(L.TcrKernelStat)(), C.c_int32()
        L.check(lib, lib.tcr_profile_read(C.byref(stats), C.byref(count)), "tcr_profile_read")
        return Counter({stats[i].name.decode(): int(stats[i].launches) for i in range(count.value)})
    finally:
        lib.tcr_profile_enable(0)


def rel_err(a, ref):
    """max |a - ref| / max |ref|  (the tolerance definition of SURVEY.md 8c)."""
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    return float(np.abs(a - ref).max() / max(np.abs(ref).max(), 1e-30))
