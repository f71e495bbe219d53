"""Shared evaluation loop of trainer and evaluator (reference: helper/base.py:20-182).
`run_inference` iterates `num_samples // batch_size` batches (the remainder is dropped, :35-46), fetching
labels / softmax outputs / total_loss per batch through `session.run` and stacking them."""
from __future__ import annotations

import time
from abc import ABC, abstractmethod

import numpy as np

from ..common.utils import Timer, get_logger
from ..runtime import InvalidArgumentError, OutOfRangeError


class Base(ABC):
    def __init__(self):
        self.log = get_logger("Base")
        self.timer = Timer(self.log)

    def get_feed_dict(self, is_training: bool = False):
        return {}

    def build_iters_from_batch_size(self, num_samples, batch_size):
        iters = self.dataset.num_samples // self.args.batch_size
        ignored = self.dataset.num_samples % self.args.batch_size
        if ignored:
            self.log.warning(f"{ignored} samples are ignored in evaluation: {self.dataset.num_samples} % {self.args.batch_size}")
        return iters

    @abstractmethod
    def build_evaluation_fetch_ops(self, do_eval):
        raise NotImplementedError

    def run_inference(self, global_step: int, iters: int = None, is_training: bool = False, do_eval: bool = True):
        feed_dict = self.get_feed_dict(is_training=is_training)
        if iters is None:
            iters = self.build_iters_from_batch_size(self.dataset.num_samples, self.args.batch_size)
        fetch_ops = self.build_evaluation_fetch_ops(do_eval)
        agg = {k: [] for k in fetch_ops}
        agg.update(batch_infer_time=[], unit_infer_time=[])
        if "metric_counts" in fetch_ops:                               # the scores of every batch stay on the device for the ranking
            self.model.reserve_ranking(iters * self.args.batch_size)
        for _ in range(iters):
            try:
                t0 = time.perf_counter()
                vals = self.session.run(fetch_ops, feed_dict=feed_dict)
                ms = (time.perf_counter() - t0) * 1e3
            except OutOfRangeError:
                self.log.info("Reach end of the dataset.")
                break
            except InvalidArgumentError as e:
                self.log.error(f"Invalid instance is detected: {e}")
                continue
            for k, v in vals.items():
                if k in agg and v is not None:
                    agg[k].append(np.atleast_1d(v))
            agg["batch_infer_time"].append(np.atleast_1d(ms))
            agg["unit_infer_time"].append(np.atleast_1d(ms / self.args.batch_size))
        out = {k: np.vstack(v) for k, v in agg.items() if v}
        if "metric_counts" in fetch_ops:                               # ONE device-to-host read per evaluation
            out["metric_counts"] = self.model.read_metric_counts(reset=True)
            out["ranking"] = self.model.read_ranking()
        return out

    def run_evaluation(self, global_step: int, iters: int = None, is_training: bool = False):
        eval_dict = self.run_inference(global_step, iters, is_training, do_eval=True)
        data = self.build_non_tensor_data_from_eval_dict(eval_dict, step=global_step)
        self.metric_manager.evaluate_and_aggregate_metrics(step=global_step, non_tensor_data=data, eval_dict=eval_dict)
        return self.metric_manager.get_evaluation_result(step=global_step)

    @staticmethod
    def add_arguments(parser):
        g = parser.add_argument_group("Base")
        g.add_argument("--use_ema", dest="use_ema", action="store_true")
        g.add_argument("--no-use_ema", dest="use_ema", action="store_false")
        g.set_defaults(use_ema=False)
        g.add_argument("--ema_decay", default=0.999, type=float)
        g.add_argument("--evaluation_iterations", type=int, default=None)


class AudioBase(Base):
    def build_evaluation_fetch_ops(self, do_eval):
        if not do_eval:
            return {"predictions_onehot": self.model.outputs}
        if getattr(self.args, "device_metrics", False):
            from ..runtime import Node
            ops = {"metric_counts": Node("metric_counts"), "total_loss": self.model.total_loss}
        else:
            ops = {"labels_onehot": self.model.labels, "predictions_onehot": self.model.outputs,
                   "total_loss": self.model.total_loss}
        ops.update(self.metric_tf_op)
        return ops

    def build_basic_loss_ops(self):
        losses = {"total_loss": self.model.total_loss, "model_loss": self.model.model_loss}
        losses.update(self.model.endpoints_loss)
        return losses

    def build_non_tensor_data_from_eval_dict(self, eval_dict, **kwargs):
        return {"dataset_split_name": self.dataset.dataset_split_name, "label_names": self.dataset.label_names,
                "predictions_onehot": eval_dict.get("predictions_onehot"), "labels_onehot": eval_dict.get("labels_onehot"),
                "metric_counts": eval_dict.get("metric_counts"), "ranking": eval_dict.get("ranking")}
