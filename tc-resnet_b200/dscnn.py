"""DS-CNN forward (inference) on the CUDA path: the reference's 2-D-conv comparison model
(audio_nets/ds_cnn.py; DSCNN{S,M,L}Model.build_inference in factory/audio_nets.py:298-358), and on the same handle the KWS
baselines cnn-trad-fpool3 (size 'P') and cnn-one-fstride4 ('F') of audio_nets/kws.py and its speech_commands nets low_latency_conv
('C') and tiny_conv ('Y'), and the paper's 2-D ablations of TC-ResNet8,
ResNet2D8 ('R') and ResNet2D8Pool ('A') of audio_nets/tc_resnet.py, and Honk's ResNets of audio_nets/res.py, Res8 ('E'), Res8Narrow
('N'), Res15 ('D') and Res15Narrow ('T'), with their dilated 3x3 convolutions.  Training DS-CNN is out of scope
(SURVEY.md 2 #13): weights come from a checkpoint keyed by the TF variable names in `self.table`.

With a front-end (set_frontend) the handle also takes audio: `mfcc`, `forward_input`, `eval_accumulate` and `listener` mirror
Engine.mfcc / Engine.forward / Engine.eval_accumulate / Engine.listener (include/tcr_b200.h, tcr_dscnn_set_frontend ff.)."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib as L
from .engine import Listener, frontend_config, frontend_shape

# tcr_dscnn_config.size of the KWS baselines (include/tcr_b200.h): KWSModel --architecture -> size code
KWS_SIZES = {"trad_fpool3": "P", "one_fstride4": "F", "low_latency_conv": "C", "tiny_conv": "Y"}
# and of the 2-D ablations, by TF scope; they alone take a width multiplier
RES2D_SIZES = {"ResNet2D8": "R", "ResNet2D8Pool": "A"}
# and of Honk's ResNets, by model name (all four under the TF scope "Res")
RES_SIZES = {"Res8": "E", "Res8Narrow": "N", "Res15": "D", "Res15Narrow": "T"}


class DsCnn:
    _LISTENER_CREATE = "tcr_dscnn_listener_create"

    def __init__(self, size: str = "S", height: int = 49, width: int = 40, num_classes: int = 12, max_batch: int = 512,
                 device: int | None = None, width_multiplier: float = 0.0):
        if not torch.cuda.is_available():
            raise L.TcrError("tcresnet_b200.DsCnn needs a CUDA device (there is no CPU fallback)")
        self.lib = L.load()
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        cfg = L.TcrDscnnConfig(ord(size), height, width, num_classes, max_batch, self.device.index, width_multiplier)
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):
            L.check(self.lib, self.lib.tcr_dscnn_create(C.byref(cfg), C.byref(self._h)), "tcr_dscnn_create")
        descs, count, nparams, flops = C.POINTER(L.TcrParamDesc)(), C.c_int32(), C.c_int64(), C.c_int64()
        L.check(self.lib, self.lib.tcr_dscnn_param_table(self._h, C.byref(descs), C.byref(count), C.byref(nparams),
                                                         C.byref(flops)), "tcr_dscnn_param_table")
        self.table = [dict(name=descs[i].name.decode(), kind=L.KIND_NAMES[descs[i].kind], trainable=descs[i].kind < 3,
                           shape=tuple(descs[i].shape[:descs[i].rank]), offset=int(descs[i].offset),
                           numel=int(descs[i].numel)) for i in range(count.value)]
        self.num_params, self.forward_flops = int(nparams.value), int(flops.value)
        self.num_classes, self.height, self.width = num_classes, height, width
        self.size, self.max_batch = size, int(max_batch)
        self.cfg: Optional[L.TcrConfig] = None          # the front-end's configuration (set_frontend)
        # the counts AudioNetModel reports, in tcr_get_info's form
        self.info = L.TcrInfo(abi_version=L.ABI_VERSION, frames=height, features=width, forward_flops_per_utt=self.forward_flops)
        self.info.num_moving = sum(d["numel"] for d in self.table if not d["trainable"])
        self.info.num_trainable = self.num_params - self.info.num_moving
        self.num_trainable, self.num_moving = int(self.info.num_trainable), int(self.info.num_moving)
        self.frames, self.features = height, width

    def close(self):
        if getattr(self, "_h", None):
            self.lib.tcr_dscnn_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def _f32(self, *shape):
        return torch.empty(shape, dtype=torch.float32, device=self.device)

    @staticmethod
    def _ptr(t, dtype=torch.float32):
        return None if t is None else _checked(t, dtype)

    @property
    def trainable_names(self):
        """The TF variables the reference's graph trains (weights, biases, beta), in table order; the moving statistics are not."""
        return [d["name"] for d in self.table if d["trainable"]]

    def pack(self, values: Dict[str, np.ndarray]) -> torch.Tensor:
        flat = np.zeros(self.num_params, np.float32)
        for d in self.table:
            flat[d["offset"]:d["offset"] + d["numel"]] = np.asarray(values[d["name"]], np.float32).ravel()
        return torch.from_numpy(flat).to(self.device)

    def new_variables(self, seed: int = 0) -> torch.Tensor:
        """Flat variables as the reference initialises them before a restore: Xavier-uniform weights (slim's default), zero biases /
        beta / moving mean, unit moving variance, unit gamma (the 2-D ablations' BatchNorm); the KWS nets (KWS_SIZES) draw every weight from
        truncated_normal(stddev=0.01) (audio_nets/kws.py), values past two sigma redrawn, and zero biases.  Host-side RNG, not TF's."""
        rng = np.random.default_rng(seed)
        flat = np.zeros(self.num_params, np.float32)
        for d in self.table:
            sl = slice(d["offset"], d["offset"] + d["numel"])
            if d["kind"] == "weight" and self.size in KWS_SIZES.values():
                v = rng.standard_normal(d["numel"])
                while (bad := np.abs(v) > 2.0).any():
                    v[bad] = rng.standard_normal(int(bad.sum()))
                flat[sl] = (0.01 * v).astype(np.float32)
            elif d["kind"] == "weight":
                shp = d["shape"]
                fan_in, fan_out = int(np.prod(shp[:-1])), int(np.prod(shp[:-2])) * shp[-1]
                lim = np.sqrt(6.0 / (fan_in + fan_out))
                flat[sl] = rng.uniform(-lim, lim, d["numel"]).astype(np.float32)
            elif d["kind"] in ("moving_variance", "gamma"):
                flat[sl] = 1.0
        return torch.from_numpy(flat).to(self.device)

    def variables_to_dict(self, params: torch.Tensor) -> Dict[str, np.ndarray]:
        p = params.detach().cpu().numpy()
        return {d["name"]: p[d["offset"]:d["offset"] + d["numel"]].reshape(d["shape"]).copy() for d in self.table}

    def variables_from_dict(self, values: Dict[str, np.ndarray], params: torch.Tensor, strict: bool = True, only=None):
        """Restores `params` by TF name, as Engine.variables_from_dict (only: predicate on names; the ones it rejects are skipped)."""
        p = params.detach().cpu().numpy().copy()
        for d in self.table:
            if only is not None and not only(d["name"]):
                continue
            if d["name"] not in values:
                if strict:
                    raise KeyError(d["name"])
                continue
            v = np.asarray(values[d["name"]], np.float32)
            if v.size != d["numel"]:
                raise ValueError(f"{d['name']}: expected {d['shape']}, got {v.shape}")
            p[d["offset"]:d["offset"] + d["numel"]] = v.ravel()
        params.copy_(torch.from_numpy(p))

    # ------------------------------------------------------------------ front-end and evaluation
    def set_frontend(self, sample_rate=16000, clip_duration_ms=1000, window_size_ms=40.0, window_stride_ms=20.0, num_mel_bins=64,
                     num_mfccs=40, lower_edge_hertz=80.0, upper_edge_hertz=7600.0, preprocess_method="mfcc"):
        """The wav front-end in front of conv_1 (tcr_dscnn_set_frontend), from the reference's flags; its (T, F) must be the handle's
        (height, width)."""
        c = frontend_config(self.lib, sample_rate, clip_duration_ms, window_size_ms, window_stride_ms, num_mel_bins, num_mfccs,
                            lower_edge_hertz, upper_edge_hertz, preprocess_method)
        c.num_classes, c.max_batch, c.device = self.num_classes, self.max_batch, self.device.index
        with torch.cuda.device(self.device):
            L.check(self.lib, self.lib.tcr_dscnn_set_frontend(self._h, C.byref(c)), "tcr_dscnn_set_frontend")
        assert frontend_shape(c) == (self.height, self.width)
        self.cfg = c
        return self

    def _input(self, inputs: torch.Tensor, input_is_features: bool):
        n = inputs.shape[0]
        if input_is_features:
            return self._ptr(inputs.reshape(n, self.height, self.width).contiguous()), L.TCR_INPUT_FEATURES
        inputs = inputs.reshape(n, -1)
        if inputs.dtype == torch.int16:
            return self._ptr(inputs, torch.int16), L.TCR_INPUT_WAV_PCM16
        return self._ptr(inputs), L.TCR_INPUT_WAV_F32

    def mfcc(self, wav: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Front-end only: fp32 or int16 wav [n, clip_samples] -> features [n, height, width]."""
        n = wav.shape[0]
        ptr, kind = self._input(wav, False)
        out = out if out is not None else self._f32(n, self.height, self.width)
        L.check(self.lib, self.lib.tcr_dscnn_mfcc_forward(self._h, ptr, kind, self._ptr(out), n, self._stream), "tcr_dscnn_mfcc_forward")
        return out

    def forward(self, features: torch.Tensor, params: torch.Tensor):
        n = features.shape[0]
        features = features.reshape(n, self.height, self.width).contiguous()
        logits = torch.empty(n, self.num_classes, dtype=torch.float32, device=self.device)
        probs = torch.empty_like(logits)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        L.check(self.lib, self.lib.tcr_dscnn_forward(self._h, features.data_ptr(), params.data_ptr(), n, logits.data_ptr(),
                                                     probs.data_ptr(), stream), "tcr_dscnn_forward")
        return logits, probs

    def forward_input(self, inputs: torch.Tensor, params: torch.Tensor, input_is_features: bool = False, logits=None, probs=None):
        """The evaluation forward from fp32 wav, int16 PCM (decode_wav scaling on the device) or features: (logits, probs)."""
        n = inputs.shape[0]
        ptr, kind = self._input(inputs, input_is_features)
        logits = logits if logits is not None else self._f32(n, self.num_classes)
        probs = probs if probs is not None else self._f32(n, self.num_classes)
        L.check(self.lib, self.lib.tcr_dscnn_forward_input(self._h, ptr, kind, self._ptr(params), n, self._ptr(logits), self._ptr(probs),
                                                           self._stream), "tcr_dscnn_forward_input")
        return logits, probs

    def eval_accumulate(self, scores: torch.Tensor, onehot: torch.Tensor, counts: Optional[torch.Tensor] = None, topk: int = 5) -> torch.Tensor:
        """Adds one batch to the device-resident evaluation counts, as Engine.eval_accumulate (tcr_dscnn_eval_accumulate)."""
        n, c = scores.shape[0], self.num_classes
        if counts is None:
            counts = torch.zeros(c * c + 2, dtype=torch.int64, device=self.device)
        assert counts.is_cuda and counts.dtype == torch.int64 and counts.numel() == c * c + 2
        L.check(self.lib, self.lib.tcr_dscnn_eval_accumulate(self._h, self._ptr(scores), self._ptr(onehot), n, int(topk),
                                                             counts.data_ptr(), self._stream), "tcr_dscnn_eval_accumulate")
        return counts

    def eval_collect(self, scores: torch.Tensor, onehot: torch.Tensor, store_scores: torch.Tensor, store_labels: torch.Tensor,
                     row_offset: int) -> None:
        """Appends one batch of SOFTMAX scores and its label indices to the ranking store (fp32 [capacity, C], int32 [capacity]) at
        row_offset; see tcr_dscnn_eval_collect in include/tcr_b200.h."""
        L.check(self.lib, self.lib.tcr_dscnn_eval_collect(self._h, self._ptr(scores), self._ptr(onehot), scores.shape[0], int(row_offset),
                                                    store_scores.shape[0], self._ptr(store_scores), self._ptr(store_labels, torch.int32),
                                                    self._stream), "tcr_dscnn_eval_collect")

    def eval_rank_workspace(self, n: int) -> torch.Tensor:
        """The device workspace eval_rank needs for n stored rows (the tcr_dscnn_eval_rank query)."""
        nb = C.c_int64()
        L.check(self.lib, self.lib.tcr_dscnn_eval_rank(self._h, None, None, int(n), None, C.byref(nb), None, self._stream), "tcr_dscnn_eval_rank")
        return torch.empty(nb.value, dtype=torch.uint8, device=self.device)

    def eval_rank(self, store_scores: torch.Tensor, store_labels: torch.Tensor, n: int,
                  workspace: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The ranking pass over the store's first n rows: fp64 [2C + 4] = per-class AP, per-class positives, then the macro,
        micro, weighted and samples averages (tcr_dscnn_eval_rank).  metrics.manager.ranking_metrics names them."""
        ws = workspace if workspace is not None else self.eval_rank_workspace(n)
        nb = C.c_int64(ws.numel())
        out = torch.empty(2 * self.num_classes + 4, dtype=torch.float64, device=self.device)
        L.check(self.lib, self.lib.tcr_dscnn_eval_rank(self._h, self._ptr(store_scores), self._ptr(store_labels, torch.int32), int(n),
                                                 self._ptr(ws, torch.uint8), C.byref(nb), self._ptr(out, torch.float64), self._stream),
                "tcr_dscnn_eval_rank")
        return out

    def listener(self, streams: int, hop_frames: int, chunk_samples: int, params: Optional[torch.Tensor] = None) -> Listener:
        """A continuous-audio listener on this handle (tcr_dscnn_listener_create); pushes take `params` only (moving is None)."""
        return Listener(self, streams, hop_frames, chunk_samples, params, None)


def _checked(t: torch.Tensor, dtype):
    assert t.is_cuda and t.dtype == dtype and t.is_contiguous(), f"expected contiguous {dtype} CUDA tensor"
    return t.data_ptr()
