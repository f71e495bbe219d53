"""Model builders with the reference's names and attribute surface (factory/audio_nets.py:19-183, 362-409),
executing on the CUDA engine instead of building a TF graph.

`train_audio.py` / `evaluate_audio.py` look the class up by NAME (`eval(f"audio_nets.{args.model}")`,
train_audio.py:32), call `Model(args, dataset)`, then `model.build(wavs, labels, is_training)` and hand the model
to the trainer / evaluator, which touch only the attributes set here and `session.run`.  TCResNet8Model and
TCResNet14Model are on the accelerated path; DSCNN{S,M,L}Model, KWSModel (--architecture trad_fpool3 / one_fstride4 / low_latency_conv / tiny_conv),
ResNet2D8Model, ResNet2D8PoolModel and Res{8,8Narrow,15,15Narrow}Model are on it for evaluation, deployment and streaming (their
training is out of scope and raises NotImplementedError).
"""
from __future__ import annotations

import collections
from typing import Dict, Optional, Set

import numpy as np
import torch

from ..common import utils
from ..common.model_loader import EMA_SUFFIX
from ..datasets import preprocessor_factory
from ..dscnn import KWS_SIZES, RES2D_SIZES, RES_SIZES, DsCnn
from ..engine import OPTIMIZER_DEFAULTS, OPTIMIZER_SLOT_NAMES, Engine
from ..runtime import InvalidArgumentError, Node
from .base import TFModel

_available_nets = [
    "KWSModel", "Res8Model", "Res8NarrowModel", "Res15Model", "Res15NarrowModel", "DSCNNSModel", "DSCNNMModel",
    "DSCNNLModel", "TCResNet8Model", "TCResNet14Model", "ResNet2D8Model", "ResNet2D8PoolModel",
]


class AudioNetModel(TFModel):
    engine_model: Optional[str] = None      # set by the accelerated subclasses

    def __init__(self, args, dataset=None):
        self.log = utils.get_logger("AudioNetModel")
        self.args, self.dataset = args, dataset
        self.engine: Optional[Engine] = None
        self.global_step = 0
        self.optimizer = dict(kind="mom", momentum=0.9)            # set by the trainer (build_optimizer -> set_optimizer)
        self.slots2 = None                                          # Adam v / RMSProp mom (`slots`: the first slot)
        self.beta1_power = self.beta2_power = None                  # Adam's beta^t before the next step (np.float32)
        self.ema, self.ema_decay = None, 0.999                      # --use_ema: flat shadow of the trained variables
        self.lr_schedule = lambda step: getattr(args, "learning_rate", 1e-4)
        self.var_names_to_values = None                            # in-memory weight injection hook (trainer.py:145-154)
        self.endpoints_loss: Dict[str, Node] = {}
        self._last: Dict[str, np.ndarray] = {}
        self._feed, self._feed_last = None, (0, np.float32("nan"), np.float32("nan"))
        self._feed_steps = []                                       # global step numbers of the submitted, not yet reported steps
        self._feed_slots = []
        self._loss_ring, self._loss_pending, self._loss_submitted = [], [], 0   # --device_dataset: (device, pinned, event) loss slots
        self._counts = None                                        # device int64 [classes^2 + 2] (tcr_eval_accumulate)
        self._rank = None                                          # (scores, labels, workspace) of the ranking store (tcr_eval_collect)
        self._rank_rows = 0
        self.reported_losses = collections.deque(maxlen=256)      # (global step, total_loss, model_loss) of each finished step
        self._clip_request, self._clips = 0, None                   # audio summaries: clips kept from the next training step

    # ------------------------------------------------------------------ graph-construction API of the reference
    def build(self, wavs, labels, is_training):
        self._audio_original, self.labels, self.is_training = wavs, labels, is_training
        self.preprocess_input()
        self.inputs, self.logits, self._outputs, self.endpoints = self.build_output(
            self.audio, self.is_training, self.args.output_name)
        self._total_loss, self._model_loss, self.endpoints_loss = self.build_loss(self.logits, self.outputs, self.labels)
        self.total_params = self.engine.num_trainable + self.engine.num_moving
        self.log.info(f"{type(self).__name__}: {self.engine.num_trainable} trainable parameters, "
                      f"{self.engine.info.forward_flops_per_utt / 1e6:.3f} MFLOP forward per utterance")
        if self.dataset is not None and getattr(self.dataset, "session", None) is not None:
            self.dataset.session.bind(self)

    def preprocess_input(self, for_deploy=False):
        a = self.args
        window = int(a.sample_rate * a.window_size_ms / 1000)
        stride = int(a.sample_rate * a.window_stride_ms / 1000)
        pre = preprocessor_factory.factory(preprocess_method=a.preprocess_method, scope="input/audio/preprocessing",
                                           preprocessed_node_name="input/audio/preprocessed")
        self._audio = pre.preprocess(self._audio_original, window_size_samples=window, window_stride_samples=stride,
                                     for_deploy=for_deploy, **vars(a))
        self._audio.name = "audio"
        self.log.info(f"Update height/width to {self._audio.shape}")
        a.height, a.width, a.channels = self._audio.shape[1:4]
        self.input_preprocessors_for_tflite = [pre]

    def build_output(self, inputs, is_training, output_name):
        logits, endpoints = self.build_inference(inputs, is_training=is_training)
        return inputs, logits, Node("outputs", [None, self.args.num_classes]), endpoints

    def build_inference(self, inputs, is_training=True):
        if self.engine_model is None:
            raise NotImplementedError(f"{type(self).__name__} is a baseline outside the accelerated TC-ResNet path")
        a = self.args
        self.engine = self._new_engine(max(int(getattr(a, 'batch_size', 1) or 1), int(getattr(a, 'input_batch_size', 1) or 1)))
        self.params, self.slots, self.moving = self.engine.new_variables(seed=getattr(a, "seed", 0) or 0)
        if getattr(a, "data_parallel", False):
            self.engine.attach_process_group()
        n = int(getattr(a, 'batch_size', 1) or 1)
        dev = self.engine.device
        self._h_wav = torch.empty(n, self.engine.cfg.clip_samples, dtype=torch.float32).pin_memory()
        self._h_hot = torch.empty(n, a.num_classes, dtype=torch.float32).pin_memory()
        self._d_wav, self._d_hot = self._h_wav.to(dev), self._h_hot.to(dev)
        self._feed_slots = [(torch.empty_like(self._h_wav).pin_memory(), torch.empty_like(self._h_hot).pin_memory()) for _ in range(4)]
        if getattr(a, "device_dataset", False) and self.dataset is not None and self.dataset.device_data is None:
            self.dataset.attach_device(self.engine)
        return Node("logits", [None, a.num_classes]), {"ranges": Node("ranges")}

    def _new_engine(self, max_batch: int) -> Engine:
        a = self.args
        return Engine(model=self.engine_model, width_multiplier=a.width_multiplier, num_classes=a.num_classes,
                      sample_rate=a.sample_rate, clip_duration_ms=a.clip_duration_ms,
                      window_size_ms=a.window_size_ms, window_stride_ms=a.window_stride_ms,
                      num_mel_bins=a.num_mel_bins, num_mfccs=a.num_mfccs, lower_edge_hertz=a.lower_edge_hertz,
                      upper_edge_hertz=a.upper_edge_hertz, preprocess_method=a.preprocess_method,
                      max_batch=max_batch, dropout_keep_prob=a.dropout_keep_prob,
                      label_smoothing=getattr(a, "label_smoothing", 0.0))

    def build_loss(self, logits, scores, labels):
        return Node("total_loss", []), Node("model_loss", []), {}

    def infer(self, inputs: torch.Tensor, input_is_features: bool = False) -> torch.Tensor:
        """Softmax outputs [n, classes] of the evaluation forward on wav (fp32 / int16) or features (DeployedModel)."""
        return self.engine.forward(inputs, self.params, self.moving, is_training=False, input_is_features=input_is_features)["probs"]

    def build_deployable_model(self, include_preprocess=True):
        """The deploy graph of the reference (factory/audio_nets.py:87-125: placeholder [input_batch_size, samples, 1] ->
        preprocessing -> network in inference mode -> softmax) as a callable on the CUDA engine: returns
        ([input node], DeployedModel).  include_preprocess=False takes features [1, height, width, 1] like the profiling graph.
        The front-end is the TRAINING front-end (tf.contrib.signal path, datasets/preprocessors.py:64-96): the reference's deploy
        front-end (audio_ops.mfcc, :98-158) is a different approximation of the same features and is not reproduced; TFLite
        conversion itself (freeze.py) stays out of scope."""
        a = self.args
        n = int(getattr(a, "input_batch_size", 1) or 1)
        if self.engine is None or int(self.engine.cfg.max_batch) < n:
            self.build_inference(None, is_training=False)
        samples = int(a.sample_rate * a.clip_duration_ms / 1000)
        if include_preprocess:
            node = Node("input/audio/before_preprocessing", [n, samples, 1])
        else:
            assert a.height > 0 and a.width > 0 and a.channels > 0
            node = Node("input", [1, a.height, a.width, a.channels])
        return [node], DeployedModel(self, n, include_preprocess)

    def build_streaming_model(self, streams: int = 1, hop_ms: float = 10, chunk_ms: float = 100) -> "StreamingModel":
        """The deploy graph run over continuous audio (include/tcr_b200.h, tcr_listener_*): `streams` independent streams, a
        window every hop_ms (a whole number of frame strides) and chunk_ms of new audio per stream and push (a whole number of
        hops).  Scores with the variables this model holds, so a checkpoint restored with --use_ema scores with the shadows."""
        a = self.args
        stride = int(a.sample_rate * a.window_stride_ms / 1000)
        hop_samples = int(round(a.sample_rate * hop_ms / 1000))
        chunk = int(round(a.sample_rate * chunk_ms / 1000))
        if hop_samples <= 0 or hop_samples % stride:
            raise ValueError(f"hop_ms {hop_ms} is not a positive multiple of the {a.window_stride_ms} ms frame stride")
        hop = hop_samples // stride
        if chunk <= 0 or chunk % hop_samples:
            raise ValueError(f"chunk_ms {chunk_ms} is not a positive multiple of hop_ms {hop_ms}")
        windows = int(streams) * (chunk // hop_samples)
        if self.engine is None:
            self.build_inference(None, is_training=False)
        # the listener's forward runs at streams * windows utterances: a handle sized for that, on the same variables
        engine = self.engine if int(self.engine.cfg.max_batch) >= windows else self._new_engine(windows)
        return StreamingModel(self, engine, int(streams), hop, chunk)

    # ------------------------------------------------------------------ attribute surface
    @property
    def model_loss(self):
        return self._model_loss

    @property
    def total_loss(self):
        return self._total_loss

    @property
    def audio_original(self):
        return self._audio_original

    @property
    def audio(self):
        return self._audio

    @property
    def outputs(self):
        return self._outputs

    # ------------------------------------------------------------------ optimizer state
    def set_optimizer(self, optimizer: Dict[str, object]):
        """Takes the optimizer the trainer built (TrainerBase.build_optimizer) and allocates its state as TF creates it: the
        slot buffers of the kind (Engine.new_optimizer_state) and, for Adam, beta1_power / beta2_power = beta1 / beta2."""
        self.flush_feed()
        self.optimizer = dict(optimizer)
        kind = self.optimizer["kind"]
        if self.engine is not None:
            self.slots, self.slots2 = self.engine.new_optimizer_state(kind)
        if kind == "adam":
            self.beta1_power, self.beta2_power = np.float32(self._opt("beta1")), np.float32(self._opt("beta2"))
        else:
            self.beta1_power = self.beta2_power = None

    def _opt(self, key):
        v = self.optimizer.get(key)
        return OPTIMIZER_DEFAULTS[self.optimizer["kind"]][key] if v is None else v

    def _step_optimizer(self) -> Dict[str, object]:
        """The `optimizer` argument of this step (Engine.train_step / HostFeed.submit)."""
        o = dict(self.optimizer)
        if o["kind"] == "adam":
            o.update(beta1_power=self.beta1_power, beta2_power=self.beta2_power)
        return o

    def _advance_optimizer(self):
        """After each submitted step: beta^t <- beta^t * beta in fp32, TF's assign(beta1_power * beta1) in the finish op.  Every
        rank does the same, so data-parallel replicas hold the same powers without exchanging them."""
        if self.optimizer["kind"] == "adam":
            self.beta1_power = np.float32(self.beta1_power * np.float32(self._opt("beta1")))
            self.beta2_power = np.float32(self.beta2_power * np.float32(self._opt("beta2")))

    # ------------------------------------------------------------------ trainable subset and weight EMA
    def set_trainable(self, names=None):
        """Trains only `names` (None: every trainable variable); see Engine.set_trainable."""
        self.flush_feed()
        return self.engine.set_trainable(names)

    def enable_ema(self, decay: float):
        """--use_ema: the shadow `<var>/ExponentialMovingAverage` of every trained variable, starting from the variables' CURRENT
        values (the trainer calls this before the restore: TF initialises a shadow from its variable's initializer)."""
        self.ema, self.ema_decay = self.engine.new_ema(self.params), float(decay)

    def _trained(self):
        trained = getattr(self.engine, "trained", None)
        return trained if trained is not None else {d["name"] for d in self.engine.table if d["trainable"]}

    # ------------------------------------------------------------------ variables by TF name
    def get_variables(self, with_slots=True) -> Dict[str, np.ndarray]:
        """{TF name: array}: the variables, the shadows `<var>/ExponentialMovingAverage` of the trained ones with --use_ema, and
        with_slots the optimizer state under TF's names (`<var>/Momentum`; `<var>/Adam`, `<var>/Adam_1`, beta1_power,
        beta2_power; `<var>/RMSProp`, `<var>/RMSProp_1`).  Slots and shadows exist for the trained variables only, as TF
        creates them for var_list alone."""
        self.flush_feed()
        out = self.engine.variables_to_dict(self.params, self.moving)
        trained = self._trained()
        if with_slots:
            names = OPTIMIZER_SLOT_NAMES[self.optimizer["kind"]]
            for suffix, buf in zip(names, (self.slots, self.slots2)):
                if suffix is not None:
                    for k, v in self.engine.variables_to_dict(buf).items():
                        if k in trained:
                            out[f"{k}/{suffix}"] = v
            if self.optimizer["kind"] == "adam":
                out["beta1_power"], out["beta2_power"] = np.float32(self.beta1_power), np.float32(self.beta2_power)
        if self.ema is not None:
            for k, v in self.engine.variables_to_dict(self.ema).items():
                if k in trained:
                    out[k + EMA_SUFFIX] = v
        return out

    def set_variables(self, values: Dict[str, np.ndarray], strict=True, restore=None):
        """Variables by TF name; the optimizer state of the current kind is optional (slots and powers that are absent keep
        their values).  With --use_ema the shadows of the trained variables are restored under their own names, and a missing
        one is an error when `strict` (it keeps its initial value otherwise).  restore: predicate on names
        (model_loader.restore_filter); the names it rejects are neither restored nor required."""
        self.flush_feed()
        if restore is not None:
            values = {k: v for k, v in values.items() if restore(k)}
        self.engine.variables_from_dict(values, self.params, self.moving, strict=strict, only=restore)
        names = OPTIMIZER_SLOT_NAMES[self.optimizer["kind"]]
        for suffix, buf in zip(names, (self.slots, self.slots2)):
            if suffix is None:
                continue
            tail = "/" + suffix
            slots = {k[:-len(tail)]: v for k, v in values.items() if k.endswith(tail)}
            if slots:
                self.engine.variables_from_dict(slots, buf, None, strict=False)
        if self.ema is not None:
            wanted = [n for n in sorted(self._trained()) if restore is None or restore(n + EMA_SUFFIX)]
            missing = [n + EMA_SUFFIX for n in wanted if n + EMA_SUFFIX not in values]
            if strict and missing:
                raise KeyError(f"checkpoint has no {missing[0]} (--ignore_missing_vars keeps the initial value)")
            shadows = {n: values[n + EMA_SUFFIX] for n in wanted if n + EMA_SUFFIX in values}
            if shadows:
                self.engine.variables_from_dict(shadows, self.ema, None, strict=False)
        if self.optimizer["kind"] == "adam":
            if "beta1_power" in values:
                self.beta1_power = np.float32(np.asarray(values["beta1_power"], np.float32).reshape(()))
            if "beta2_power" in values:
                self.beta2_power = np.float32(np.asarray(values["beta2_power"], np.float32).reshape(()))

    def _dropout_seed(self):
        """Counter-RNG seed of this step: distinct per rank under data parallelism (the kernel indexes utterances locally)."""
        world = getattr(self.engine, "world_size", 1)
        rank = getattr(self.dataset, "rank", 0) if world > 1 else 0
        return self.global_step * world + rank

    def read_metric_counts(self, reset: bool = True) -> np.ndarray:
        """Confusion matrix / top-5 hits / sample count accumulated by the forward passes since the last reset (one D2H read)."""
        if self._counts is None:
            return np.zeros(self.args.num_classes ** 2 + 2, np.int64)
        out = self._counts.cpu().numpy()
        if reset:
            self._counts.zero_()
        return out

    def reserve_ranking(self, rows: int) -> None:
        """Empties the device store of the ranking metrics and sizes it, with its workspace, for `rows` utterances: the scores of
        every evaluation batch are collected there (tcr_eval_collect) until read_ranking()."""
        if self._rank is None or self._rank[0].shape[0] < rows:
            self._rank = None                                       # the old store goes before the new one is allocated
            self._rank = (torch.empty(rows, self.args.num_classes, dtype=torch.float32, device=self.engine.device),
                          torch.empty(rows, dtype=torch.int32, device=self.engine.device), self.engine.eval_rank_workspace(rows))
        self._rank_rows = 0

    def _collect(self, probs, onehot) -> None:
        if self._rank is not None:
            self.engine.eval_collect(probs, onehot, self._rank[0], self._rank[1], self._rank_rows)
            self._rank_rows += probs.shape[0]

    def read_ranking(self) -> Optional[np.ndarray]:
        """The ranking pass over the utterances collected since reserve_ranking() (one D2H read of 2 * classes + 4 doubles, see
        metrics.manager.ranking_metrics), or None when none were; empties the store."""
        n, self._rank_rows = self._rank_rows, 0
        if self._rank is None or n == 0:
            return None
        return self.engine.eval_rank(self._rank[0], self._rank[1], n, self._rank[2]).cpu().numpy()

    # ------------------------------------------------------------------ one session.run
    def _execute_train_fast(self, names: Set[str]) -> Optional[Dict[str, object]]:
        """session.run(train_op) through the host-buffer step of the C ABI (tcr_train_step_host via engine.HostFeed): the batch goes
        H2D on the library's copy stream, the step is queued behind it and the call returns without waiting for it.  The losses
        handed back are those of the step `feed_lag` calls earlier (`loss_global_step` says which), exactly the overlap the
        reference gets from tf.data prefetching + an asynchronous session (helper/trainer.py:312-321).  Used when nothing but
        the train op, losses, step and learning rate is fetched; metric / output fetches take the synchronous path below."""
        if names - {"train_op", "global_step", "total_loss", "model_loss", "learning_rate"}:
            return None
        lag = int(getattr(self.args, "feed_lag", 2))
        if lag <= 0:
            return None
        if getattr(self.dataset, "device_data", None) is not None:
            return self._execute_train_device(lag)
        pinned = self.dataset.next_batch_pinned() if hasattr(self.dataset, "next_batch_pinned") else None
        if pinned is None:
            wav_np, hot_np = self.dataset.next_batch()
            n = wav_np.shape[0]
            if n != self.args.batch_size:
                raise InvalidArgumentError(f"bad batch: {wav_np.shape}")
            slot = self._feed_slots[self.global_step % len(self._feed_slots)]       # reused only after lag + 1 later calls
            slot[0].copy_(torch.from_numpy(wav_np.reshape(n, -1)))
            slot[1].copy_(torch.from_numpy(hot_np))
            pinned = slot
        self._keep_clips(pinned[0])
        if self._feed is None:
            from ..engine import HostFeed
            self._feed = HostFeed(self.engine, lag=lag)
        lr = float(self.lr_schedule(self.global_step))
        r = self._feed.submit(pinned[0], pinned[1], self.params, self.slots, self.moving, lr, self.optimizer.get("momentum") or 0.0,
                              self.args.weight_decay, dropout_seed=self._dropout_seed(), optimizer=self._step_optimizer(),
                              slots2=self.slots2, ema=self.ema, ema_decay=self.ema_decay)
        self._advance_optimizer()
        self.global_step += 1
        self._feed_steps.append(self.global_step)
        if r is not None:
            self._report_loss(self._feed_steps.pop(0), r[1], r[2])
            if not np.isfinite(r[1]):
                raise InvalidArgumentError(f"non-finite loss at step {self._feed_last[0]} (malformed input batch?)")
        step, total, model = self._feed_last
        return {"train_op": None, "learning_rate": np.float32(lr), "global_step": np.int64(self.global_step), "total_loss": total,
                "model_loss": model, "loss_global_step": np.int64(step)}

    def _execute_train_device(self, lag: int) -> Dict[str, object]:
        """session.run(train_op) on a resident dataset (--device_dataset): one tcr_train_step that gathers and augments its rows
        from the clip bank, with the front-end running ahead (input_resident: the bank is final).  Its losses are copied into a
        ring of lag + 1 pinned slots and reported `lag` calls later, as the host-buffer step reports them."""
        ds = self.dataset
        position, epoch = ds.next_device_rows()
        if not self._loss_ring:
            dev = self.engine.device
            self._loss_ring = [(torch.empty(2, dtype=torch.float32, device=dev), torch.empty(2, dtype=torch.float32).pin_memory(),
                                torch.cuda.Event()) for _ in range(lag + 1)]
        slot = self._loss_ring[self._loss_submitted % len(self._loss_ring)]     # collected before its reuse: at most lag pending
        self._loss_submitted += 1
        lr = float(self.lr_schedule(self.global_step))
        self.engine.train_step(None, None, self.params, self.slots, self.moving, lr, self.optimizer.get("momentum") or 0.0,
                               self.args.weight_decay, dropout_seed=self._dropout_seed(), losses=slot[0], input_resident=True,
                               optimizer=self._step_optimizer(), slots2=self.slots2, ema=self.ema, ema_decay=self.ema_decay,
                               dataset=ds.device_data.desc, position=position, epoch=epoch, seed=ds.draw_seed, n=self.args.batch_size)
        slot[1].copy_(slot[0], non_blocking=True)
        slot[2].record()
        if self._clip_request:
            self._keep_clips(ds.device_data.batch(position, epoch, ds.draw_seed, min(self._clip_request, self.args.batch_size))[0])
        self._advance_optimizer()
        self.global_step += 1
        self._feed_steps.append(self.global_step)
        self._loss_pending.append(slot)
        if len(self._loss_pending) > lag:
            self._collect_loss()
        step, total, model = self._feed_last
        return {"train_op": None, "learning_rate": np.float32(lr), "global_step": np.int64(self.global_step), "total_loss": total,
                "model_loss": model, "loss_global_step": np.int64(step)}

    def _collect_loss(self):
        _, host, event = self._loss_pending.pop(0)
        event.synchronize()
        self._report_loss(self._feed_steps.pop(0), host[0], host[1])
        if not np.isfinite(self._feed_last[1]):
            raise InvalidArgumentError(f"non-finite loss at step {self._feed_last[0]}")

    def _report_loss(self, step, total, model):
        self._feed_last = (step, np.float32(total), np.float32(model))
        self.reported_losses.append(self._feed_last)

    def capture_clips(self, k: int):
        """The next training step keeps the first k clips of its batch for an audio summary (take_clips).  A batch built on the
        device is regenerated for those rows and copied to pinned memory behind the step, so nothing waits for it here."""
        self._clip_request = int(k)

    def take_clips(self):
        """The clips kept by the last training step since capture_clips, as (host tensor [k, samples], event or None), or None.
        The tensor is valid once the event (the step's copy) has completed."""
        clips, self._clips, self._clip_request = self._clips, None, 0
        return clips

    def _keep_clips(self, wav):
        k = min(self._clip_request, wav.shape[0])
        if k <= 0:
            return
        if isinstance(wav, np.ndarray) or not wav.is_cuda:
            self._clips = (torch.as_tensor(wav[:k]).reshape(k, -1).clone(), None)
        else:
            host = torch.empty((k, wav.shape[1]), dtype=torch.float32).pin_memory()
            host.copy_(wav[:k], non_blocking=True)
            event = torch.cuda.Event()
            event.record()
            self._clips = (host, event)
        self._clip_request = 0

    def flush_feed(self):
        """Drain the host-feed pipeline (before anything reads the variables: checkpoints, evaluation, get_variables)."""
        if self._feed is not None:
            for r in self._feed.flush():
                self._report_loss(self._feed_steps.pop(0), r[1], r[2])
        while self._loss_pending:
            self._collect_loss()

    def execute(self, names: Set[str], feed) -> Dict[str, object]:
        if "train_op" in names:
            fast = self._execute_train_fast(names)
            if fast is not None:
                self._last = fast
                return fast
        self.flush_feed()
        device_data = getattr(self.dataset, "device_data", None)
        if device_data is not None:                             # --device_dataset: the batch is built on the device
            n = self.args.batch_size
            position, epoch = self.dataset.next_device_rows()
            device_data.batch(position, epoch, self.dataset.draw_seed, n, self._d_wav, self._d_hot)
        else:
            wav_np, hot_np = self.dataset.next_batch()
            n = wav_np.shape[0]
            if n != self.args.batch_size:
                raise InvalidArgumentError(f"bad batch: {wav_np.shape}")
            self._h_wav.copy_(torch.from_numpy(wav_np.reshape(n, -1)))
            self._h_hot.copy_(torch.from_numpy(hot_np))
            self._d_wav.copy_(self._h_wav, non_blocking=True)
            self._d_hot.copy_(self._h_hot, non_blocking=True)
        wd = self.args.weight_decay
        vals: Dict[str, object] = {}
        if "train_op" in names:
            lr = float(self.lr_schedule(self.global_step))
            out = self.engine.train_step(self._d_wav, self._d_hot, self.params, self.slots, self.moving, lr,
                                         self.optimizer.get("momentum") or 0.0, wd, dropout_seed=self._dropout_seed(),
                                         want_outputs=bool(names & {"outputs", "logits"}), optimizer=self._step_optimizer(),
                                         slots2=self.slots2, ema=self.ema, ema_decay=self.ema_decay)
            self._advance_optimizer()
            self.global_step += 1
            vals["train_op"], vals["learning_rate"] = None, np.float32(lr)
        else:
            out = self.engine.forward(self._d_wav, self.params, self.moving, is_training=bool(self.is_training),
                                      onehot=self._d_hot, weight_decay=wd, dropout_seed=self._dropout_seed())
            vals["learning_rate"] = np.float32(self.lr_schedule(self.global_step))
        if "metric_counts" in names:                            # evaluation counts stay on the device until read_metric_counts()
            if self._counts is None:
                self._counts = torch.zeros(self.args.num_classes ** 2 + 2, dtype=torch.int64, device=self.engine.device)
            self.engine.eval_accumulate(out["probs"], self._d_hot, self._counts, topk=5)
            self._collect(out["probs"], self._d_hot)
            vals["metric_counts"] = None
        losses = out["losses"].cpu().numpy()                    # the D2H read synchronises the step
        vals.update(total_loss=losses[0], model_loss=losses[1], global_step=np.int64(self.global_step))
        if "train_op" in names:
            self.reported_losses.append((self.global_step, losses[0], losses[1]))
            if self._clip_request:
                self._keep_clips(wav_np if device_data is None else self._d_wav)
        if device_data is None:
            vals.update(labels=hot_np, audio_original=wav_np)
        else:                                                   # copied to the host only when fetched
            if "labels" in names:
                vals["labels"] = self._d_hot.cpu().numpy()
            if "audio_original" in names:
                vals["audio_original"] = self._d_wav.cpu().numpy()[..., None]
        if "outputs" in names or "logits" in names:
            vals["outputs"], vals["logits"] = out["probs"].cpu().numpy(), out["logits"].cpu().numpy()
        if "audio" in names:
            feat = self.engine.mfcc(self._d_wav)
            vals["audio"] = feat.unsqueeze(-1).cpu().numpy()
        if "ranges" in names:
            vals["ranges"] = None       # dead `fc2` head: its forward is skipped (SURVEY.md 2b C6)
        self._last = vals
        return vals

    @staticmethod
    def add_arguments(parser):
        parser.add_argument("--label_smoothing", default=0.0, type=float)
        parser.add_argument("--feed_lag", default=2, type=int,
                            help="steps a training session.run may run ahead of the losses it reports (host-buffer step of the C ABI; "
                                 "0: synchronous steps, the loss returned is this step's)")


def _tc_flags(parser):
    parser.add_argument("--weight_decay", default=0.0001, type=float)
    parser.add_argument("--dropout_keep_prob", default=0.5, type=float)
    parser.add_argument("--width_multiplier", default=1.0, type=float)


class DeployedModel:
    """Batch-n (default 1) inference entry: wav [n, samples(,1)] or features [n, T, F(,1)] in, softmax outputs [n, classes] out.
    After the first call the launch sequence (front-end + every layer) is replayed from a CUDA graph: at batch 1 the forward is
    launch-latency bound (DESIGN.md section 6), and a graph replay is one submission instead of ~11 launches."""

    def __init__(self, model: "AudioNetModel", batch: int, include_preprocess: bool, use_graph: bool = True):
        self.model, self.batch, self.include_preprocess, self.use_graph = model, int(batch), include_preprocess, use_graph
        eng = model.engine
        shape = (self.batch, eng.cfg.clip_samples) if include_preprocess else (self.batch, eng.frames, eng.features)
        self._in = torch.zeros(shape, dtype=torch.float32, device=eng.device)
        self._graph, self._out, self._calls = None, None, 0

    def _run(self):
        return self.model.infer(self._in, input_is_features=not self.include_preprocess)

    def __call__(self, x) -> np.ndarray:
        x = torch.as_tensor(np.asarray(x, np.float32)).reshape(self._in.shape)
        self._in.copy_(x, non_blocking=True)
        if not self.use_graph or self._calls < 2:                  # two eager calls first: lazy per-kernel attributes are set outside capture
            self._out = self._run()
        else:
            if self._graph is None:
                stream = torch.cuda.Stream(device=self._in.device)
                stream.wait_stream(torch.cuda.current_stream(self._in.device))
                with torch.cuda.stream(stream):
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g, stream=stream):
                        self._out = self._run()
                torch.cuda.current_stream(self._in.device).wait_stream(stream)
                self._graph = g
            self._graph.replay()
        self._calls += 1
        return self._out.cpu().numpy()


class StreamingModel:
    """Continuous-audio entry (AudioNetModel.build_streaming_model): __call__ takes [streams, chunk_samples] new samples (fp32 in
    [-1, 1] or int16) and returns the softmax [streams, windows, classes] of the windows they complete; window k of a stream ends
    (k + 1) * hop samples after its reset.  Like DeployedModel, two eager pushes, then each push is replayed from a CUDA graph."""

    def __init__(self, model: "AudioNetModel", engine: Engine, streams: int, hop_frames: int, chunk_samples: int,
                 use_graph: bool = True):
        self.model, self.engine, self.use_graph = model, engine, use_graph
        self.listener = engine.listener(streams, hop_frames, chunk_samples)
        self.streams, self.hop_frames, self.chunk_samples = streams, hop_frames, chunk_samples
        self.windows = self.listener.windows
        self.hop_samples = hop_frames * int(engine.cfg.window_stride_samples)
        self._in = {dt: torch.zeros(streams, chunk_samples, dtype=dt, device=engine.device) for dt in (torch.float32, torch.int16)}
        self._probs = torch.zeros(streams, self.windows, engine.num_classes, dtype=torch.float32, device=engine.device)
        self._graphs, self._calls = {}, 0

    def _push(self, dt):
        m = self.model
        self.listener.push(self._in[dt], m.params, m.moving, probs=self._probs)

    def reset(self, stream: Optional[int] = None):
        self.listener.reset(stream)

    def __call__(self, x) -> np.ndarray:
        x = torch.as_tensor(x)
        dt = torch.int16 if x.dtype == torch.int16 else torch.float32
        self._in[dt].copy_(x.to(dt).reshape(self.streams, self.chunk_samples), non_blocking=True)
        if not self.use_graph or self._calls < 2:                  # two eager calls first: lazy per-kernel attributes are set outside capture
            self._push(dt)
        else:
            if dt not in self._graphs:
                dev = self.engine.device
                stream = torch.cuda.Stream(device=dev)
                stream.wait_stream(torch.cuda.current_stream(dev))
                with torch.cuda.stream(stream):
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g, stream=stream):
                        self._push(dt)
                torch.cuda.current_stream(dev).wait_stream(stream)
                self._graphs[dt] = g
            self._graphs[dt].replay()
        self._calls += 1
        return self._probs.cpu().numpy()


class TCResNet8Model(AudioNetModel):
    engine_model = "TCResNet8"
    add_arguments = staticmethod(_tc_flags)


class TCResNet14Model(AudioNetModel):
    engine_model = "TCResNet14"
    add_arguments = staticmethod(_tc_flags)


class DsCnnModel(AudioNetModel):
    """DSCNN{S,M,L}Model (factory/audio_nets.py:299-359, audio_nets/ds_cnn.py) in evaluation mode on dscnn.DsCnn: the handle runs the
    model's front-end (tcr_dscnn_set_frontend), the forward with the BatchNorm moving statistics held in its flat parameters
    (`moving` is None), the device evaluation counts, the deployable model and the listener.  Variables are restored by their TF
    names ("DSCNN/conv_1/weights", ...), with the same --use_ema, --ignore_missing_vars and include / exclude scope rules as
    TC-ResNet.  Training is out of scope."""
    dscnn_size: Optional[str] = None

    @staticmethod
    def add_arguments(parser):
        parser.add_argument("--weight_decay", default=0.0, type=float)

    def build_inference(self, inputs, is_training=True):
        if is_training:
            raise NotImplementedError(f"{type(self).__name__}: training DS-CNN is out of scope on the CUDA path; evaluation "
                                      "(evaluate_audio.py), the deployable model and the listener (listen_audio.py) are supported")
        a = self.args
        if getattr(a, "device_dataset", False):
            raise NotImplementedError(f"{type(self).__name__}: --device_dataset serves the TC-ResNet models only")
        self.engine = self._new_engine(max(int(getattr(a, 'batch_size', 1) or 1), int(getattr(a, 'input_batch_size', 1) or 1)))
        self.params, self.moving, self.slots = self.engine.new_variables(seed=getattr(a, "seed", 0) or 0), None, None
        n = int(getattr(a, 'batch_size', 1) or 1)
        dev = self.engine.device
        self._h_wav = torch.empty(n, self.engine.cfg.clip_samples, dtype=torch.float32).pin_memory()
        self._h_hot = torch.empty(n, a.num_classes, dtype=torch.float32).pin_memory()
        self._d_wav, self._d_hot = self._h_wav.to(dev), self._h_hot.to(dev)
        return Node("logits", [None, a.num_classes]), {}

    def _new_engine(self, max_batch: int) -> DsCnn:
        a = self.args
        clip = int(a.sample_rate * a.clip_duration_ms / 1000)
        window, stride = int(a.sample_rate * a.window_size_ms / 1000), int(a.sample_rate * a.window_stride_ms / 1000)
        if stride <= 0 or clip < window:
            raise ValueError(f"bad window / stride / clip ({window} / {stride} / {clip} samples)")
        height = 1 + (clip - window) // stride
        width = a.num_mfccs if a.preprocess_method == "mfcc" else a.num_mel_bins
        eng = DsCnn(self.dscnn_size, height, width, a.num_classes, max_batch, width_multiplier=self._width_multiplier())
        return eng.set_frontend(a.sample_rate, a.clip_duration_ms, a.window_size_ms, a.window_stride_ms, a.num_mel_bins, a.num_mfccs,
                                a.lower_edge_hertz, a.upper_edge_hertz, a.preprocess_method)

    def infer(self, inputs: torch.Tensor, input_is_features: bool = False) -> torch.Tensor:
        return self.engine.forward_input(inputs, self.params, input_is_features=input_is_features)[1]

    def get_variables(self, with_slots=True) -> Dict[str, np.ndarray]:
        """{TF name: array} of every variable, the moving statistics included (there is no optimizer state)."""
        return self.engine.variables_to_dict(self.params)

    def set_variables(self, values: Dict[str, np.ndarray], strict=True, restore=None):
        """Variables by TF name (restore: predicate on names, model_loader.restore_filter); optimizer slots and shadows in the
        checkpoint are ignored (evaluation with --use_ema has already put the shadows under the variables' names)."""
        if restore is not None:
            values = {k: v for k, v in values.items() if restore(k)}
        self.engine.variables_from_dict(values, self.params, strict=strict, only=restore)

    def _regularization(self) -> float:
        """The regularisation term of total_loss: none in the DS-CNN graph."""
        return 0.0

    def _width_multiplier(self) -> float:
        """tcr_dscnn_config.width_multiplier: 0 (none) but for the 2-D ablations."""
        return 0.0

    def execute(self, names: Set[str], feed) -> Dict[str, object]:
        """One evaluation session.run: the batch from the dataset, the forward from its samples, the device counts when
        `metric_counts` is fetched, and model_loss = the batch's mean softmax cross-entropy (label smoothing as --label_smoothing),
        from the logits in float64; total_loss = model_loss + _regularization()."""
        if "train_op" in names:
            raise NotImplementedError(f"{type(self).__name__}: training DS-CNN is out of scope on the CUDA path")
        wav_np, hot_np = self.dataset.next_batch()
        n = wav_np.shape[0]
        if n != self.args.batch_size:
            raise InvalidArgumentError(f"bad batch: {wav_np.shape}")
        self._h_wav.copy_(torch.from_numpy(wav_np.reshape(n, -1)))
        self._h_hot.copy_(torch.from_numpy(hot_np))
        self._d_wav.copy_(self._h_wav, non_blocking=True)
        self._d_hot.copy_(self._h_hot, non_blocking=True)
        logits, probs = self.engine.forward_input(self._d_wav, self.params)
        vals: Dict[str, object] = {"learning_rate": np.float32(self.lr_schedule(self.global_step))}
        if "metric_counts" in names:                            # evaluation counts stay on the device until read_metric_counts()
            if self._counts is None:
                self._counts = torch.zeros(self.args.num_classes ** 2 + 2, dtype=torch.int64, device=self.engine.device)
            self.engine.eval_accumulate(probs, self._d_hot, self._counts, topk=5)
            self._collect(probs, self._d_hot)
            vals["metric_counts"] = None
        lg = logits.cpu().numpy().astype(np.float64)            # the D2H read synchronises the forward
        ls = float(getattr(self.args, "label_smoothing", 0.0) or 0.0)
        target = hot_np.astype(np.float64) * (1.0 - ls) + ls / lg.shape[1]
        mx = lg.max(axis=1, keepdims=True)
        logp = lg - mx - np.log(np.exp(lg - mx).sum(axis=1, keepdims=True))
        ce = -(target * logp).sum(axis=1).mean()
        vals.update(total_loss=np.float32(ce + self._regularization()), model_loss=np.float32(ce), global_step=np.int64(self.global_step), labels=hot_np, audio_original=wav_np)
        if "outputs" in names or "logits" in names:
            vals["outputs"], vals["logits"] = probs.cpu().numpy(), lg.astype(np.float32)
        if "audio" in names:
            vals["audio"] = self.engine.mfcc(self._d_wav).unsqueeze(-1).cpu().numpy()
        self._last = vals
        return vals


class DSCNNSModel(DsCnnModel):
    dscnn_size = "S"


class DSCNNMModel(DsCnnModel):
    dscnn_size = "M"


class DSCNNLModel(DsCnnModel):
    dscnn_size = "L"


# KWSModel --architecture choices (factory/audio_nets.py:222-224); KWS_SIZES names the four on the CUDA path
KWS_ARCHITECTURES = ["single_fc", "conv", "low_latency_conv", "low_latency_svdf", "tiny_conv", "one_fstride4", "trad_fpool3"]


class KWSModel(DsCnnModel):
    """KWSModel (factory/audio_nets.py:205-224, audio_nets/kws.py) for --architecture trad_fpool3 and one_fstride4, the two Sainath &
    Parada CNNs of the reference's recipes, and low_latency_conv and tiny_conv, two of TensorFlow's speech_commands nets, in
    evaluation mode on the DS-CNN handle (size codes 'P' / 'F' / 'C' / 'Y', dscnn.KWS_SIZES).  The variables are top-level TF names
    ("first_weights", "first_bias", ...).  --weight_decay keeps TFModel's default of 1e-4, and total_loss adds the reference's L2
    term over every variable, biases included (build_loss: weight_decay * sum(tf.nn.l2_loss(v))).  single_fc, conv and
    low_latency_svdf, and training, are out of scope."""

    @staticmethod
    def add_arguments(parser):
        parser.add_argument("--architecture", default="conv", type=str, choices=KWS_ARCHITECTURES)

    @property
    def dscnn_size(self) -> str:
        arch = self.args.architecture
        if arch not in KWS_SIZES:
            raise NotImplementedError(f"KWSModel --architecture {arch} is not on the CUDA path; supported: "
                                      + ", ".join(KWS_SIZES))
        return KWS_SIZES[arch]

    def build_inference(self, inputs, is_training=True):
        self.dscnn_size                                          # an unsupported architecture is refused first
        if is_training:
            raise NotImplementedError(f"KWSModel --architecture {self.args.architecture}: training the KWS baselines is out of "
                                      "scope on the CUDA path; evaluation (evaluate_audio.py), the deployable model and the "
                                      "listener (listen_audio.py) are supported")
        return super().build_inference(inputs, is_training=False)

    def _regularization(self) -> float:
        wd = float(self.args.weight_decay)
        return wd * 0.5 * float((self.params.double() ** 2).sum()) if wd else 0.0


class _Res2dModel(DsCnnModel):
    """ResNet2D8Model / ResNet2D8PoolModel (factory/audio_nets.py:412-460, audio_nets/tc_resnet.py:73-101): the paper's 2-D ablations
    of TC-ResNet8, in evaluation mode on the DS-CNN handle (size codes 'R' / 'A', dscnn.RES2D_SIZES) with --width_multiplier.
    Variables are restored by their TF names ("ResNet2D8/conv0/weights", ...).  total_loss adds build_loss's L2 term,
    weight_decay * sum(tf.nn.l2_loss(v)) over every variable outside BatchNorm (the weights, fc2 included).  Training is out of
    scope."""
    scope: str = ""

    add_arguments = staticmethod(_tc_flags)

    @property
    def dscnn_size(self) -> str:
        return RES2D_SIZES[self.scope]

    def _width_multiplier(self) -> float:
        return float(self.args.width_multiplier)

    def build_inference(self, inputs, is_training=True):
        if is_training:
            raise NotImplementedError(f"{type(self).__name__}: training the 2-D ablations is out of scope on the CUDA path; evaluation "
                                      "(evaluate_audio.py), the deployable model and the listener (listen_audio.py) are supported")
        if getattr(self.args, "device_dataset", False):
            raise NotImplementedError(f"{type(self).__name__}: --device_dataset serves the TC-ResNet models only; evaluate from the "
                                      "dataset on disk")
        return super().build_inference(inputs, is_training=False)

    def _regularization(self) -> float:
        return _weights_l2(self)


def _weights_l2(model: DsCnnModel) -> float:
    """build_loss's L2 term, weight_decay * sum(tf.nn.l2_loss(w)) over the weights of the parameter table (every variable outside
    BatchNorm)."""
    wd = float(model.args.weight_decay)
    if not wd:
        return 0.0
    p = model.params.double()
    return wd * 0.5 * sum(float((p[d["offset"]:d["offset"] + d["numel"]] ** 2).sum()) for d in model.engine.table
                          if d["kind"] == "weight")


class ResNet2D8Model(_Res2dModel):
    scope = "ResNet2D8"


class ResNet2D8PoolModel(_Res2dModel):
    scope = "ResNet2D8Pool"


class _ResModel(DsCnnModel):
    """Res8Model / Res8NarrowModel / Res15Model / Res15NarrowModel (factory/audio_nets.py:227-297, audio_nets/res.py): Honk's ResNets
    in evaluation mode on the DS-CNN handle (size codes dscnn.RES_SIZES), Res15 with its dilated convolutions.  Variables are
    restored by their TF names ("Res/conv0/Conv/weights", ...).  --weight_decay keeps the reference's 1e-5 default, and total_loss
    adds build_loss's L2 term over the trainable variables, which are all weights.  Training is out of scope."""
    net: str = ""

    @staticmethod
    def add_arguments(parser):
        parser.add_argument("--weight_decay", default=0.00001, type=float)

    @property
    def dscnn_size(self) -> str:
        return RES_SIZES[self.net]

    def build_inference(self, inputs, is_training=True):
        if is_training:
            raise NotImplementedError(f"{type(self).__name__}: training Res8 / Res15 is out of scope on the CUDA path; evaluation "
                                      "(evaluate_audio.py), the deployable model and the listener (listen_audio.py) are supported")
        if getattr(self.args, "device_dataset", False):
            raise NotImplementedError(f"{type(self).__name__}: --device_dataset serves the TC-ResNet models only; evaluate from the "
                                      "dataset on disk")
        return super().build_inference(inputs, is_training=False)

    def _regularization(self) -> float:
        return _weights_l2(self)


class Res8Model(_ResModel):
    net = "Res8"


class Res8NarrowModel(_ResModel):
    net = "Res8Narrow"


class Res15Model(_ResModel):
    net = "Res15"


class Res15NarrowModel(_ResModel):
    net = "Res15Narrow"
