"""Host-side engine: one C-ABI handle + torch CUDA tensors as buffer carriers.

This is the object the reference-facing shims (factory/audio_nets.py, helper/trainer.py, helper/evaluator.py)
drive; it maps the reference's `args` flags onto tcr_config and exposes the three calls a `session.run`
of the reference amounts to: front-end, forward (eval / training-graph) and one full training step.
There is no CPU path: constructing an Engine without a CUDA device or without libtcr_b200.so raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib as L

_MODELS = {"TCResNet8": 8, "TCResNet8Model": 8, "TCResNet14": 14, "TCResNet14Model": 14, 8: 8, 14: 14}
_FEATURES = {"mfcc": L.TCR_FEATURE_MFCC, "log_mel_spectrogram": L.TCR_FEATURE_LOG_MEL}

# Optimizers of the fused step (tcr_step_args::optimizer) with TF 1.13's defaults.  "mom" / "gd" take the step's `momentum`
# argument; Adam and RMSProp take their hyper-parameters from the `optimizer` dict, Adam also its powers beta^t BEFORE the step.
OPTIMIZER_DEFAULTS = {
    "mom": dict(),
    "gd": dict(),
    "adam": dict(beta1=0.9, beta2=0.999, epsilon=1e-8),
    "rmsprop": dict(decay=0.9, momentum=0.0, epsilon=1e-10),
}
# TF slot names of the optimizer state: `<var>/<slot>` for each of (slots, slots2)
OPTIMIZER_SLOT_NAMES = {"mom": ("Momentum", None), "gd": ("Momentum", None), "adam": ("Adam", "Adam_1"),
                        "rmsprop": ("RMSProp", "RMSProp_1")}


def _optimizer_kind(optimizer) -> str:
    kind = "mom" if optimizer is None else optimizer.get("kind", "mom")
    if kind not in OPTIMIZER_DEFAULTS:
        raise NotImplementedError(f"optimizer {kind!r}: expected one of {sorted(OPTIMIZER_DEFAULTS)}")
    return kind


def _set_optimizer(a, optimizer, slots2_ptr):
    """Fills the optimizer fields of a TcrStepArgs.  None or kind "mom" / "gd" leave them zero: the momentum step."""
    kind = _optimizer_kind(optimizer)
    if kind in ("mom", "gd"):
        return
    o = dict(OPTIMIZER_DEFAULTS[kind], **{k: v for k, v in optimizer.items() if v is not None})
    a.slots2, a.epsilon = slots2_ptr, float(o["epsilon"])
    if kind == "adam":
        a.optimizer, a.beta1, a.beta2 = L.TCR_OPT_ADAM, float(o["beta1"]), float(o["beta2"])
        a.beta1_power, a.beta2_power = float(o["beta1_power"]), float(o["beta2_power"])
    else:
        a.optimizer, a.rho, a.momentum = L.TCR_OPT_RMSPROP, float(o["decay"]), float(o["momentum"])


def frontend_config(lib, sample_rate=16000, clip_duration_ms=1000, window_size_ms=40.0, window_stride_ms=20.0, num_mel_bins=64,
                    num_mfccs=40, lower_edge_hertz=80.0, upper_edge_hertz=7600.0, preprocess_method="mfcc") -> "L.TcrConfig":
    """tcr_config_default with the front-end fields set from the reference's flags (the fields tcr_dscnn_set_frontend reads)."""
    if preprocess_method not in _FEATURES:
        raise NotImplementedError(f"preprocess_method {preprocess_method}")
    c = L.TcrConfig()
    L.check(lib, lib.tcr_config_default(C.byref(c)), "tcr_config_default")
    c.sample_rate = int(sample_rate)
    # the reference's integer truncations (factory/audio_nets.py:63-64, :89)
    c.clip_samples = int(sample_rate * clip_duration_ms / 1000)
    c.window_size_samples = int(sample_rate * window_size_ms / 1000)
    c.window_stride_samples = int(sample_rate * window_stride_ms / 1000)
    c.num_mel_bins, c.num_mfccs = int(num_mel_bins), int(num_mfccs)
    c.lower_edge_hertz, c.upper_edge_hertz = float(lower_edge_hertz), float(upper_edge_hertz)
    c.feature_kind = _FEATURES[preprocess_method]
    return c


def frontend_shape(c: "L.TcrConfig"):
    """(T, F) of a front-end configuration: frames and features per clip."""
    frames = 1 + (c.clip_samples - c.window_size_samples) // c.window_stride_samples
    return frames, (c.num_mfccs if c.feature_kind == L.TCR_FEATURE_MFCC else c.num_mel_bins)


class Engine:
    _LISTENER_CREATE = "tcr_listener_create"

    def __init__(self, model="TCResNet8", width_multiplier=1.0, num_classes=12, sample_rate=16000,
                 clip_duration_ms=1000, window_size_ms=40.0, window_stride_ms=20.0, num_mel_bins=64, num_mfccs=40,
                 lower_edge_hertz=80.0, upper_edge_hertz=7600.0, preprocess_method="mfcc", max_batch=512,
                 dropout_keep_prob=0.5, label_smoothing=0.0, bn_decay=0.997, bn_epsilon=1e-3,
                 device: Optional[int] = None):
        if not torch.cuda.is_available():
            raise L.TcrError("tcresnet_b200.Engine needs a CUDA device (there is no CPU fallback)")
        if model not in _MODELS:
            raise NotImplementedError(f"{model}: only TCResNet8/TCResNet14 are on the accelerated path")
        if preprocess_method not in _FEATURES:
            raise NotImplementedError(f"preprocess_method {preprocess_method}")
        self.lib = L.load()
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        c = frontend_config(self.lib, sample_rate, clip_duration_ms, window_size_ms, window_stride_ms, num_mel_bins, num_mfccs,
                            lower_edge_hertz, upper_edge_hertz, preprocess_method)
        c.model = _MODELS[model]
        c.width_multiplier = float(width_multiplier)
        c.num_classes = int(num_classes)
        c.max_batch = int(max_batch)
        c.bn_decay, c.bn_epsilon = float(bn_decay), float(bn_epsilon)
        c.dropout_keep_prob, c.label_smoothing = float(dropout_keep_prob), float(label_smoothing)
        c.device = self.device.index
        self.cfg = c
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):
            L.check(self.lib, self.lib.tcr_create(C.byref(c), C.byref(self._h)), "tcr_create")
        self.info = L.TcrInfo()
        L.check(self.lib, self.lib.tcr_get_info(self._h, C.byref(self.info)), "tcr_get_info")
        self.num_trainable = int(self.info.num_trainable)
        self.num_moving = int(self.info.num_moving)
        self.frames, self.features = int(self.info.frames), int(self.info.features)
        self.num_classes = int(num_classes)
        self.table = self._read_table()
        self.trained = set(self.trainable_names)
        self.world_size = 1

    # ------------------------------------------------------------------ plumbing
    def close(self):
        if getattr(self, "_h", None):
            self.lib.tcr_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def _read_table(self):
        descs = C.POINTER(L.TcrParamDesc)()
        n = C.c_int32()
        L.check(self.lib, self.lib.tcr_param_table(self._h, C.byref(descs), C.byref(n)), "tcr_param_table")
        return [dict(name=descs[i].name.decode(), kind=L.KIND_NAMES[descs[i].kind], trainable=descs[i].kind < 3,
                     shape=tuple(descs[i].shape[:descs[i].rank]), offset=int(descs[i].offset),
                     numel=int(descs[i].numel)) for i in range(n.value)]

    def _f32(self, *shape):
        return torch.empty(shape, dtype=torch.float32, device=self.device)

    @staticmethod
    def _ptr(t, dtype=torch.float32):
        if t is None:
            return None
        assert t.is_cuda and t.dtype == dtype and t.is_contiguous(), f"expected contiguous {dtype} CUDA tensor"
        return t.data_ptr()

    def _input(self, inputs, input_is_features):
        """(pointer, TCR_INPUT_* kind): fp32 wav, precomputed features, or int16 PCM (decode_wav scaling on device)."""
        n = inputs.shape[0]
        if input_is_features:
            return self._ptr(inputs), L.TCR_INPUT_FEATURES
        inputs = inputs.reshape(n, -1)
        if inputs.dtype == torch.int16:
            return self._ptr(inputs, torch.int16), L.TCR_INPUT_WAV_PCM16
        return self._ptr(inputs), L.TCR_INPUT_WAV_F32

    # ------------------------------------------------------------------ variables
    def new_variables(self, seed: int = 0):
        """(params, slots, moving): Xavier-uniform / gamma=1 / beta=0 / moving (0,1) / slots 0."""
        params, slots, moving = self._f32(self.num_trainable), self._f32(self.num_trainable), self._f32(self.num_moving)
        L.check(self.lib, self.lib.tcr_init_variables(self._h, self._ptr(params), self._ptr(slots), self._ptr(moving),
                                                      seed, self._stream), "tcr_init_variables")
        return params, slots, moving

    def new_optimizer_state(self, kind: str = "mom"):
        """(slots, slots2) for an optimizer kind, initialised as TF's slot creators do: the momentum accumulator (slots2 None),
        Adam's m and v (zeros), RMSProp's ms (ONES, as tf.train.RMSPropOptimizer in TF 1.x) and mom (zeros)."""
        kind = _optimizer_kind(dict(kind=kind))
        slots = torch.ones if kind == "rmsprop" else torch.zeros
        first = slots(self.num_trainable, dtype=torch.float32, device=self.device)
        second = torch.zeros(self.num_trainable, dtype=torch.float32, device=self.device) if OPTIMIZER_SLOT_NAMES[kind][1] else None
        return first, second

    @property
    def trainable_names(self):
        """Names of the trainable variables in table order (tf.trainable_variables() order)."""
        return [d["name"] for d in self.table if d["trainable"]]

    def set_trainable(self, names_or_mask=None):
        """The variables the training steps train (--trainable_scopes, tcr_set_trainable): None = all (the default), an iterable of
        variable names, or one bool per trainable variable in table order.  Frozen variables get a zero gradient and keep their
        values and optimizer slots; the step skips the backward work only they needed.  Returns the set of trained names."""
        names = self.trainable_names
        torch.cuda.current_stream(self.device).synchronize()      # the plans are rewritten in place: no step may be queued
        if names_or_mask is None:
            L.check(self.lib, self.lib.tcr_set_trainable(self._h, None, 0), "tcr_set_trainable")
            self.trained = set(names)
            return self.trained
        sel = list(names_or_mask)
        if sel and all(isinstance(x, (bool, np.bool_)) for x in sel):
            if len(sel) != len(names):
                raise ValueError(f"{len(sel)} flags for {len(names)} trainable variables")
            mask = [bool(x) for x in sel]
        else:
            unknown = set(sel) - set(names)
            if unknown:
                raise KeyError(f"not trainable variables of this model: {sorted(unknown)}")
            mask = [n in set(sel) for n in names]
        flags = (C.c_int32 * len(mask))(*[int(m) for m in mask])
        L.check(self.lib, self.lib.tcr_set_trainable(self._h, flags, len(mask)), "tcr_set_trainable")
        self.trained = {n for n, m in zip(names, mask) if m}
        return self.trained

    def new_ema(self, params: torch.Tensor) -> torch.Tensor:
        """Flat shadow buffer for tcr_step_args::ema, initialised to `params` (TF initialises each `<var>/ExponentialMovingAverage`
        to the variable's initial value)."""
        return params.detach().clone().contiguous()

    def variables_to_dict(self, params: torch.Tensor, moving: Optional[torch.Tensor] = None) -> Dict[str, np.ndarray]:
        """{TF variable name: ndarray} — the reference's `var_names_to_values` form (helper/trainer.py:145-154)."""
        p = params.detach().cpu().numpy()
        m = moving.detach().cpu().numpy() if moving is not None else None
        out = {}
        for d in self.table:
            src = p if d["trainable"] else m
            if src is not None:
                out[d["name"]] = src[d["offset"]:d["offset"] + d["numel"]].reshape(d["shape"]).copy()
        return out

    def variables_from_dict(self, values: Dict[str, np.ndarray], params: torch.Tensor, moving: Optional[torch.Tensor] = None,
                            strict: bool = True, only=None):
        """only: predicate on names; the variables it rejects are skipped (neither read nor required)."""
        p = params.detach().cpu().numpy().copy()
        m = moving.detach().cpu().numpy().copy() if moving is not None else None
        for d in self.table:
            if only is not None and not only(d["name"]):
                continue
            if d["name"] not in values:
                if strict:
                    raise KeyError(d["name"])
                continue
            dst = p if d["trainable"] else m
            if dst is None:
                continue
            v = np.asarray(values[d["name"]], np.float32)
            if v.size != d["numel"]:
                raise ValueError(f"{d['name']}: expected {d['shape']}, got {v.shape}")
            dst[d["offset"]:d["offset"] + d["numel"]] = v.ravel()
        params.copy_(torch.from_numpy(p))
        if moving is not None:
            moving.copy_(torch.from_numpy(m))

    # ------------------------------------------------------------------ the three calls
    def mfcc(self, wav: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        wav = wav.reshape(wav.shape[0], -1)
        n = wav.shape[0]
        out = out if out is not None else self._f32(n, self.frames, self.features)
        if wav.dtype == torch.int16:
            L.check(self.lib, self.lib.tcr_mfcc_forward_pcm16(self._h, self._ptr(wav, torch.int16), self._ptr(out), n, self._stream),
                    "tcr_mfcc_forward_pcm16")
        else:
            L.check(self.lib, self.lib.tcr_mfcc_forward(self._h, self._ptr(wav), self._ptr(out), n, self._stream),
                    "tcr_mfcc_forward")
        return out

    def augment(self, pcm: torch.Tensor, clips: torch.Tensor, background: Optional[torch.Tensor] = None,
                out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Device input stage (datasets/augmentation_factory.py): int16 clips [n, stride] + per-clip draws -> fp32 wav
        [n, clip_samples].  `clips`: uint8 CUDA tensor holding n packed tcr_augment_clip records (24 bytes each, see
        include/tcr_b200.h); `background`: the background recordings concatenated (fp32) or None."""
        n = pcm.shape[0]
        assert pcm.is_cuda and pcm.dtype == torch.int16 and pcm.is_contiguous()
        assert clips.is_cuda and clips.dtype == torch.uint8 and clips.numel() == 24 * n
        out = out if out is not None else self._f32(n, self.cfg.clip_samples)
        L.check(self.lib, self.lib.tcr_augment_pcm16(self._h, pcm.data_ptr(), pcm.shape[1], clips.data_ptr(), self._ptr(background),
                                                     self._ptr(out), n, self._stream), "tcr_augment_pcm16")
        return out

    def dataset_batch(self, desc: "L.TcrDataset", position: int, epoch: int, seed: int, n: int,
                      wav_out: Optional[torch.Tensor] = None, onehot_out: Optional[torch.Tensor] = None):
        """Rows [position, position + n) of a resident dataset's order (tcr_dataset_batch, datasets/device_input_stage.DeviceDataset),
        gathered and augmented with the device's draws: (fp32 wav [n, clip_samples], one-hot [n, num_classes])."""
        wav_out = wav_out if wav_out is not None else self._f32(n, self.cfg.clip_samples)
        onehot_out = onehot_out if onehot_out is not None else self._f32(n, self.num_classes)
        L.check(self.lib, self.lib.tcr_dataset_batch(self._h, C.byref(desc), int(position), int(epoch), int(seed), int(n),
                                                     self._ptr(wav_out), self._ptr(onehot_out), self._stream), "tcr_dataset_batch")
        return wav_out, onehot_out

    def forward(self, inputs: torch.Tensor, params: torch.Tensor, moving: Optional[torch.Tensor] = None,
                is_training: bool = False, onehot: Optional[torch.Tensor] = None, weight_decay: float = 0.0,
                dropout_seed: int = 0, dropout_mask: Optional[torch.Tensor] = None, input_is_features: bool = False):
        n = inputs.shape[0]
        in_ptr, in_kind = self._input(inputs, input_is_features)
        logits, probs = self._f32(n, self.num_classes), self._f32(n, self.num_classes)
        losses = self._f32(2) if onehot is not None else None
        L.check(self.lib, self.lib.tcr_forward(self._h, in_ptr, in_kind, self._ptr(params),
                                               self._ptr(moving), n, int(is_training), int(dropout_seed),
                                               self._ptr(dropout_mask), self._ptr(onehot), float(weight_decay),
                                               self._ptr(logits), self._ptr(probs), self._ptr(losses), self._stream),
                "tcr_forward")
        return dict(logits=logits, probs=probs, losses=losses)

    def train_step(self, inputs: torch.Tensor, onehot: torch.Tensor, params: torch.Tensor, slots: torch.Tensor,
                   moving: torch.Tensor, learning_rate: float, momentum: float = 0.9, weight_decay: float = 1e-4,
                   dropout_seed: int = 0, dropout_mask: Optional[torch.Tensor] = None, input_is_features: bool = False,
                   want_outputs: bool = False, want_grads: bool = False, apply_update: bool = True,
                   losses: Optional[torch.Tensor] = None, clips: Optional[torch.Tensor] = None,
                   background: Optional[torch.Tensor] = None, input_resident: bool = False, *,
                   optimizer: Optional[dict] = None, slots2: Optional[torch.Tensor] = None,
                   ema: Optional[torch.Tensor] = None, ema_decay: float = 0.999, dataset: Optional["L.TcrDataset"] = None,
                   position: int = 0, epoch: int = 0, seed: int = 0, n: Optional[int] = None):
        """optimizer: None or dict(kind="mom" | "gd") for the momentum step (`momentum`), dict(kind="adam", beta1=, beta2=,
        epsilon=, beta1_power=, beta2_power=) or dict(kind="rmsprop", decay=, momentum=, epsilon=) (missing hyper-parameters
        take TF's defaults, OPTIMIZER_DEFAULTS).  Adam / RMSProp keep their second slot in `slots2` (new_optimizer_state);
        Adam's beta1_power / beta2_power are the values before this step, and advancing them is the caller's.
        clips (uint8 CUDA tensor of n packed tcr_augment_clip records) + int16 `inputs` [n, stride]: the step starts with
        the device input stage (decode, shift, background mix, clip) instead of taking decoded fp32 samples.
        input_resident=True: `inputs` is final when the call is made (nothing queued on the current stream writes it); the
        front-end then runs ahead on the library's own stream and overlaps the previous step's tail (tcr_step_args::input_resident).
        ema (new_ema) / ema_decay: after the update, the shadow of every trained parameter moves toward the new weight
        (tf.train.ExponentialMovingAverage(ema_decay).apply(variables_to_train), tcr_step_args::ema).
        dataset (DeviceDataset.desc) with position / epoch / seed and n: the step reads rows [position, position + n) of the resident
        dataset's order, augmented with the device's draws, and their labels (tcr_step_args::dataset); `inputs` and `onehot` are
        then None."""
        a = L.TcrStepArgs()
        if dataset is not None:
            assert inputs is None and onehot is None and n is not None
            a.dataset, a.dataset_position, a.dataset_epoch, a.dataset_seed = C.addressof(dataset), int(position), int(epoch), int(seed)
        elif clips is not None:
            n = inputs.shape[0]
            assert inputs.dtype == torch.int16 and inputs.is_cuda and inputs.is_contiguous() and clips.numel() == 24 * n
            a.input, a.input_is_features = inputs.data_ptr(), L.TCR_INPUT_WAV_PCM16
            a.clips, a.background, a.pcm_stride = clips.data_ptr(), self._ptr(background), inputs.shape[1]
        else:
            n = inputs.shape[0]
            a.input, a.input_is_features = self._input(inputs, input_is_features)
        a.onehot, a.n = self._ptr(onehot), n
        a.params, a.slots, a.moving = self._ptr(params), self._ptr(slots), self._ptr(moving)
        a.learning_rate, a.momentum, a.weight_decay = float(learning_rate), float(momentum), float(weight_decay)
        a.dropout_seed, a.dropout_mask = int(dropout_seed), self._ptr(dropout_mask)
        losses = losses if losses is not None else self._f32(2)
        out = dict(losses=losses)
        a.losses = self._ptr(losses)
        if want_outputs:
            out["logits"], out["probs"] = self._f32(n, self.num_classes), self._f32(n, self.num_classes)
            a.logits, a.probs = self._ptr(out["logits"]), self._ptr(out["probs"])
        if want_grads:
            out["grads"] = self._f32(self.num_trainable)
            a.grads = self._ptr(out["grads"])
        a.apply_update = int(apply_update)
        a.input_resident = int(bool(input_resident))
        _set_optimizer(a, optimizer, self._ptr(slots2))
        a.ema, a.ema_decay = self._ptr(ema), float(ema_decay)
        L.check(self.lib, self.lib.tcr_train_step(self._h, C.byref(a), self._stream), "tcr_train_step")
        return out

    def eval_accumulate(self, scores: torch.Tensor, onehot: torch.Tensor, counts: Optional[torch.Tensor] = None, topk: int = 5) -> torch.Tensor:
        """Adds one batch to the device-resident evaluation counts (int64 [C*C + 2]: confusion matrix, top-k hits, samples);
        see tcr_eval_accumulate in include/tcr_b200.h.  metrics.manager.metrics_from_counts turns them into the reference's metrics."""
        n, c = scores.shape[0], self.num_classes
        if counts is None:
            counts = torch.zeros(c * c + 2, dtype=torch.int64, device=self.device)
        assert counts.is_cuda and counts.dtype == torch.int64 and counts.numel() == c * c + 2
        L.check(self.lib, self.lib.tcr_eval_accumulate(self._h, self._ptr(scores), self._ptr(onehot), n, int(topk), counts.data_ptr(),
                                                       self._stream), "tcr_eval_accumulate")
        return counts

    def eval_collect(self, scores: torch.Tensor, onehot: torch.Tensor, store_scores: torch.Tensor, store_labels: torch.Tensor,
                     row_offset: int) -> None:
        """Appends one batch of SOFTMAX scores and its label indices to the ranking store (fp32 [capacity, C], int32 [capacity]) at
        row_offset; see tcr_eval_collect in include/tcr_b200.h."""
        L.check(self.lib, self.lib.tcr_eval_collect(self._h, self._ptr(scores), self._ptr(onehot), scores.shape[0], int(row_offset),
                                                    store_scores.shape[0], self._ptr(store_scores), self._ptr(store_labels, torch.int32),
                                                    self._stream), "tcr_eval_collect")

    def eval_rank_workspace(self, n: int) -> torch.Tensor:
        """The device workspace eval_rank needs for n stored rows (the tcr_eval_rank query)."""
        nb = C.c_int64()
        L.check(self.lib, self.lib.tcr_eval_rank(self._h, None, None, int(n), None, C.byref(nb), None, self._stream), "tcr_eval_rank")
        return torch.empty(nb.value, dtype=torch.uint8, device=self.device)

    def eval_rank(self, store_scores: torch.Tensor, store_labels: torch.Tensor, n: int,
                  workspace: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The ranking pass over the store's first n rows: fp64 [2C + 4] = per-class AP, per-class positives, then the macro,
        micro, weighted and samples averages (tcr_eval_rank).  metrics.manager.ranking_metrics names them."""
        ws = workspace if workspace is not None else self.eval_rank_workspace(n)
        nb = C.c_int64(ws.numel())
        out = torch.empty(2 * self.num_classes + 4, dtype=torch.float64, device=self.device)
        L.check(self.lib, self.lib.tcr_eval_rank(self._h, self._ptr(store_scores), self._ptr(store_labels, torch.int32), int(n),
                                                 self._ptr(ws, torch.uint8), C.byref(nb), self._ptr(out, torch.float64), self._stream),
                "tcr_eval_rank")
        return out

    def listener(self, streams: int, hop_frames: int, chunk_samples: int, params: Optional[torch.Tensor] = None,
                 moving: Optional[torch.Tensor] = None) -> "Listener":
        """A continuous-audio listener on this handle (tcr_listener_*): `streams` streams, a window every `hop_frames` frames,
        `chunk_samples` new samples per stream and push, scored with `params` / `moving` (the tensors, read at every push)."""
        return Listener(self, streams, hop_frames, chunk_samples, params, moving)

    # ------------------------------------------------------------------ data parallel
    def set_sync_bn(self, enable: bool = True):
        """Parity-test flag (SURVEY.md 8(e)): BatchNorm statistics over the global batch of all ranks (= one device with batch
        world * n).  Needs attach_process_group() first; the step then runs on the per-layer kernels with one small NCCL all-reduce
        per BN layer, forward and backward.  The default (local statistics) is what production runs use."""
        L.check(self.lib, self.lib.tcr_comm_set_sync_bn(self._h, int(bool(enable))), "tcr_comm_set_sync_bn")

    def attach_process_group(self):
        """One NCCL communicator per handle; the 128-byte unique id travels through torch.distributed."""
        import torch.distributed as dist
        world, rank = dist.get_world_size(), dist.get_rank()
        if world == 1:
            return
        from .dp import broadcast_bytes
        buf = (C.c_char * 128)()
        if rank == 0:
            L.check(self.lib, self.lib.tcr_comm_unique_id(buf), "tcr_comm_unique_id")
        idbuf = (C.c_char * 128).from_buffer_copy(broadcast_bytes(bytes(buf) if rank == 0 else None))
        with torch.cuda.device(self.device):
            L.check(self.lib, self.lib.tcr_comm_init(self._h, idbuf, rank, world), "tcr_comm_init")
        self.world_size = world
        self.exchange = "nccl"
        # Peer-memory exchange (same node, <= 8 ranks): the update kernel sums the ranks' gradients itself over NVLink
        # (include/tcr_b200.h, tcr_comm_p2p_*).  Every rank must take the same branch, hence the all_gather of the outcome.
        import os
        if world <= 8 and os.environ.get("TCR_P2P", "1") != "0":
            mine = (C.c_char * 128)()
            with torch.cuda.device(self.device):
                ok = self.lib.tcr_comm_p2p_export(self._h, mine) == 0
            gathered = [None] * world
            dist.all_gather_object(gathered, bytes(mine) if ok else None)
            if all(g is not None for g in gathered):
                table = (C.c_char * (128 * world)).from_buffer_copy(b"".join(gathered))
                with torch.cuda.device(self.device):
                    ok = self.lib.tcr_comm_p2p_attach(self._h, table, rank, world) == 0
            else:
                ok = False
            outcome = [None] * world
            dist.all_gather_object(outcome, bool(ok))
            if all(outcome):
                self.exchange = "peer-memory"
            else:                                     # someone could not export / map a peer: everybody stays on NCCL
                with torch.cuda.device(self.device):
                    self.lib.tcr_comm_p2p_detach(self._h)

    # ------------------------------------------------------------------ accounting
    def launch_count(self) -> int:
        n = C.c_uint64()
        self.lib.tcr_launch_count(C.byref(n))
        return int(n.value)

    def profile(self, enable: bool):
        self.lib.tcr_profile_enable(int(enable))

    def profile_read(self):
        stats = C.POINTER(L.TcrKernelStat)()
        n = C.c_int32()
        L.check(self.lib, self.lib.tcr_profile_read(C.byref(stats), C.byref(n)), "tcr_profile_read")
        return {stats[i].name.decode(): (float(stats[i].total_ms), int(stats[i].launches)) for i in range(n.value)}

    def fp32_peak_tflops(self) -> float:
        v = C.c_double()
        L.check(self.lib, self.lib.tcr_measure_fp32_peak(self._h, C.byref(v), self._stream), "tcr_measure_fp32_peak")
        return float(v.value)


class Listener:
    """S audio streams scored with a sliding window (include/tcr_b200.h, tcr_listener_*) by an Engine or a dscnn.DsCnn (moving None).  Each push takes `chunk_samples` new
    samples per stream and returns the softmax of K = chunk_samples / (hop_frames * window_stride_samples) windows per stream;
    window k of a stream (counted from its reset) is the clip starting k * hop_frames strides into the stream after
    (T - hop_frames) * stride + (window - stride) zeros, scored exactly as Engine.forward scores it in evaluation mode."""

    def __init__(self, engine, streams: int, hop_frames: int, chunk_samples: int, params: Optional[torch.Tensor] = None,
                 moving: Optional[torch.Tensor] = None):
        self.eng, self.params, self.moving = engine, params, moving
        self._p = C.c_void_p()
        cfg = L.TcrListenerConfig(int(streams), int(hop_frames), int(chunk_samples))
        create = engine._LISTENER_CREATE
        with torch.cuda.device(engine.device):
            L.check(engine.lib, getattr(engine.lib, create)(engine._h, C.byref(cfg), C.byref(self._p)), create)
        self.streams, self.hop_frames, self.chunk_samples = int(streams), int(hop_frames), int(chunk_samples)
        self.windows = self.chunk_samples // (self.hop_frames * int(engine.cfg.window_stride_samples))

    def close(self):
        if getattr(self, "_p", None):
            self.eng.lib.tcr_listener_destroy(self._p)
            self._p = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self, stream: Optional[int] = None):
        """Back to the state after creation: one stream, or all of them (None)."""
        L.check(self.eng.lib, self.eng.lib.tcr_listener_reset(self._p, -1 if stream is None else int(stream), self.eng._stream),
                "tcr_listener_reset")

    def push(self, samples: torch.Tensor, params: Optional[torch.Tensor] = None, moving: Optional[torch.Tensor] = None,
             probs: Optional[torch.Tensor] = None, logits: Optional[torch.Tensor] = None) -> torch.Tensor:
        """samples: CUDA fp32 (in [-1, 1]) or int16 tensor [S, chunk_samples].  Returns device probs [S, K, classes] (`probs`, when
        given, is written in place; `logits` likewise receives the logits).  params / moving: the variables of this push, by
        default the ones the listener was created with."""
        eng = self.eng
        params = params if params is not None else self.params
        moving = moving if moving is not None else self.moving
        assert samples.is_cuda and samples.is_contiguous() and tuple(samples.shape) == (self.streams, self.chunk_samples), \
            f"expected a contiguous CUDA tensor [{self.streams}, {self.chunk_samples}]"
        kind = L.TCR_INPUT_WAV_PCM16 if samples.dtype == torch.int16 else L.TCR_INPUT_WAV_F32
        if kind == L.TCR_INPUT_WAV_F32:
            assert samples.dtype == torch.float32, "samples must be fp32 or int16"
        probs = probs if probs is not None else eng._f32(self.streams, self.windows, eng.num_classes)
        L.check(eng.lib, eng.lib.tcr_listener_push(self._p, samples.data_ptr(), kind, eng._ptr(params), eng._ptr(moving),
                                                   eng._ptr(logits), eng._ptr(probs), eng._stream), "tcr_listener_push")
        return probs


class HostFeed:
    """Host-buffer feed around the C ABI's tcr_train_step_host (the `session.run(train_op)` loop of
    helper/trainer.py:132-154 with the input pipeline's prefetch, datasets/data_wrapper_base.py:100-108).

    submit() hands one pinned host batch (fp32 wav, int16 PCM, or features) to the library, which copies it H2D on its
    own copy stream into a staging slot, runs the step behind the copy and reads the two losses back.  The call does
    not wait for the step it submits: it returns (step_index, total_loss, model_loss) of the step `lag` submissions
    earlier (None while the pipeline fills), so copies, launches and compute of neighbouring steps overlap while every
    step's input still crosses the bus and every step's loss reaches the host.  flush() drains what is outstanding.
    """

    def __init__(self, engine: "Engine", lag: int = 2):
        self.eng, self.lag = engine, int(lag)
        self._out = (C.c_float * 2)()
        self._step = C.c_int64(-1)

    def _result(self):
        return None if self._step.value < 0 else (int(self._step.value), float(self._out[0]), float(self._out[1]))

    def submit(self, h_inputs: torch.Tensor, h_onehot: torch.Tensor, params, slots, moving, learning_rate, momentum=0.9,
               weight_decay=1e-4, dropout_seed=0, input_is_features=False, h_clips: Optional[torch.Tensor] = None,
               background: Optional[torch.Tensor] = None, *, optimizer: Optional[dict] = None,
               slots2: Optional[torch.Tensor] = None, ema: Optional[torch.Tensor] = None, ema_decay: float = 0.999):
        """optimizer / slots2 / ema / ema_decay: as Engine.train_step; the values (Adam's powers included) are captured with this call.
        h_clips (pinned uint8 tensor of n packed tcr_augment_clip records, datasets/device_input_stage.py) with int16
        h_inputs [n, stride]: the wav files' samples and the per-clip draws cross the bus; the input stage runs on the device
        (`background`: the CUDA-resident bank)."""
        eng = self.eng
        assert h_inputs.is_pinned() and h_onehot.is_pinned() and h_inputs.is_contiguous(), "HostFeed needs pinned host tensors"
        a = L.TcrStepArgs()
        a.input = h_inputs.data_ptr()
        a.input_is_features = (L.TCR_INPUT_FEATURES if input_is_features else
                               L.TCR_INPUT_WAV_PCM16 if h_inputs.dtype == torch.int16 else L.TCR_INPUT_WAV_F32)
        a.onehot, a.n = h_onehot.data_ptr(), h_inputs.shape[0]
        if h_clips is not None:
            assert h_clips.is_pinned() and h_clips.dtype == torch.uint8 and h_inputs.dtype == torch.int16
            a.clips, a.background, a.pcm_stride = h_clips.data_ptr(), eng._ptr(background), h_inputs.shape[1]
        a.params, a.slots, a.moving = eng._ptr(params), eng._ptr(slots), eng._ptr(moving)
        a.learning_rate, a.momentum, a.weight_decay = float(learning_rate), float(momentum), float(weight_decay)
        a.dropout_seed, a.apply_update = int(dropout_seed), 1
        _set_optimizer(a, optimizer, eng._ptr(slots2))
        a.ema, a.ema_decay = eng._ptr(ema), float(ema_decay)
        L.check(eng.lib, eng.lib.tcr_train_step_host(eng._h, C.byref(a), self.lag, eng._stream, self._out, C.byref(self._step)),
                "tcr_train_step_host")
        return self._result()

    def flush(self):
        """Drain the pipeline: list of (step_index, total_loss, model_loss) for every outstanding step."""
        out = []
        while True:
            L.check(self.eng.lib, self.eng.lib.tcr_host_flush(self.eng._h, self._out, C.byref(self._step)), "tcr_host_flush")
            r = self._result()
            if r is None:
                return out
            out.append(r)
