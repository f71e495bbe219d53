"""Host-side metrics on the aggregated [num_samples, num_classes] arrays the hot path returns, and their TensorBoard summaries.

The reference routes these through a metric-op registry + TensorBoard summaries (metrics/, ~1.26 kLoC, sklearn).  What the
trainer / evaluator loops need is kept: the flag surface of MetricManagerBase.add_arguments (metrics/base.py:250-260),
accuracy / top-5 / per-class precision-recall-F1 / mAP computed with NumPy, `get_best_keep_metric_with_modes`, a log line
per evaluation, and the summaries of metrics/summaries.py:11-202 written by common/tf_events (DESIGN.md section 4m):
`summary_table` restates which op registers which tag in which collection, `summary_collections` the trainer's schedule.
"""
from __future__ import annotations

from pathlib import Path
from types import SimpleNamespace
from typing import Dict, List, Optional, Sequence

import numpy as np

from ..common.tf_events import EventWriter, audio_values, scalar_value, text_value

# metrics/summaries.py:12-23
KEY_TYPES = SimpleNamespace(DEFAULT="SUMMARY_DEFAULT", VERBOSE="SUMMARY_VERBOSE", FIRST_N="SUMMARY_FIRST_N")
VALUE_TYPES = SimpleNamespace(SCALAR="SCALAR", PLACEHOLDER="PLACEHOLDER", AUDIO="AUDIO")


def summary_collections(step_from_restore: int, step_min_summaries: int, step_save_summaries: int,
                        step_save_verbose_summaries: int, step_save_first_n_summaries: int) -> List[str]:
    """The collections a training step writes (helper/trainer.py:374-385): DEFAULT from step_min_summaries on, every
    step_save_summaries steps; VERBOSE every step_save_verbose_summaries steps; FIRST_N up to step_save_first_n_summaries."""
    keys = []
    if step_from_restore >= step_min_summaries and step_from_restore % max(1, step_save_summaries) == 0:
        keys.append(KEY_TYPES.DEFAULT)
    if step_from_restore % max(1, step_save_verbose_summaries) == 0:
        keys.append(KEY_TYPES.VERBOSE)
    if step_from_restore <= step_save_first_n_summaries:
        keys.append(KEY_TYPES.FIRST_N)
    return keys


def summary_directory(train_dir, is_training: bool, base_name: str) -> Path:
    """metrics/summaries.py:130-142: the training directory itself, or `<dir>/<split>` for an evaluator (the directory of a
    checkpoint path that is a file)."""
    if is_training:
        return Path(train_dir)
    return (Path(train_dir) if Path(train_dir).is_dir() else Path(train_dir).parent) / base_name


class Summaries:
    """One event-file writer (metrics/summaries.py:BaseSummaries): the `config` text once, then Summary events by step."""

    def __init__(self, directory, max_outputs: int, sample_rate: int = 16000):
        self.writer = EventWriter(directory)
        self.max_outputs, self.sample_rate = int(max_outputs), int(sample_rate)

    def setup_experiment(self, config):
        """The sorted (flag, str(value)) table as tf.summary.text("config") (metrics/summaries.py:47-59).  There is no graph to
        add: the step is one fused CUDA launch sequence, not a TF graph."""
        rows = [(k, str(v)) for k, v in sorted(vars(config).items(), key=lambda x: x[0])]
        self.writer.add(0, [text_value("config", rows)])
        self.writer.flush()

    def write(self, step: int, values: Sequence[bytes]):
        self.writer.add(step, values)

    def flush(self):
        self.writer.flush()

    def close(self):
        self.writer.close()


def topn_accuracy(labels_onehot, predictions, n=5):
    """The reference's topN_accuracy (metrics/funcs.py:4-19) with a stable sort: equal scores keep the lower class first, as on
    the device (tcr_eval_accumulate), at every class count.  NaN scores rank after every number."""
    top = np.argsort(-predictions, axis=1, kind="stable")[:, :n]
    return float(np.mean(np.any(top == labels_onehot.argmax(1)[:, None], axis=1)))


def average_precision(y_true, score):
    order = np.argsort(-score, kind="stable")
    y = y_true[order]
    if y.sum() == 0:
        return float("nan")
    hits = np.cumsum(y)
    return float(np.sum((hits / (np.arange(len(y)) + 1)) * y) / y.sum())


def ranking_vector(labels_onehot, predictions) -> np.ndarray:
    """NumPy restatement of what tcr_eval_rank leaves on the device, from the [n, classes] arrays: fp64 [2 * classes + 4] =
    per-class AP, per-class positives, then the macro, micro, weighted and samples averages of sklearn's
    average_precision_score (equal scores grouped; a class without positives has AP 0 and counts in the macro average).
    The label of a row is its first maximum; a NaN score makes every average it enters NaN."""
    s = np.asarray(predictions, np.float32)
    n, c = s.shape
    y = np.asarray(labels_onehot).argmax(1)
    hot = np.arange(c)[None, :] == y[:, None]

    def ap(pos, score):
        if np.isnan(score).any():
            return float("nan")
        if not pos.any():
            return 0.0
        order = np.argsort(-score, kind="stable")
        score, pos = score[order], pos[order]
        ends = np.r_[np.nonzero(score[1:] != score[:-1])[0], score.size - 1]   # last item of each group of equal scores (inf too)
        tp = np.cumsum(pos)[ends]
        return float(np.sum(np.diff(np.r_[0, tp]) * tp / (ends + 1.0)) / tp[-1])

    per_class = np.array([ap(hot[:, k], s[:, k]) for k in range(c)])
    support = hot.sum(0).astype(np.float64)
    above = (s >= s[np.arange(n), y][:, None]).sum(1)
    samples = np.where(np.isnan(s).any(1), np.nan, 1.0 / above)
    return np.concatenate([per_class, support, [per_class.mean(), ap(hot.ravel(), s.ravel()),
                                                np.sum(per_class * support) / support.sum(), samples.mean()]])


def ranking_metrics(ranking, label_names=None, use_class_metrics: bool = False) -> Dict[str, float]:
    """The reference's MAPMetricOp (mAP at macro / micro / weighted / samples) and, with use_class_metrics, APMetricOp (ap/<label>),
    metrics/ops/non_tensor_ops.py:15-61, :296-343, from tcr_eval_rank's result or ranking_vector (the same layout)."""
    r = np.asarray(ranking, np.float64)
    c = (r.size - 4) // 2
    res = {f"mAP/{avg}": float(v) for avg, v in zip(("macro", "micro", "weighted", "samples"), r[2 * c:])}
    if use_class_metrics:
        for k, name in enumerate(label_names or [str(i) for i in range(c)]):
            res[f"ap/{name}"] = float(r[k])
    return res


def metrics_from_counts(counts, label_names=None, use_class_metrics: bool = False) -> Dict[str, object]:
    """The count-based metrics of the reference (accuracy, top-5, per-class precision / recall / F1, confusion matrix:
    metrics/ops/non_tensor_ops.py:64-295) from the integers tcr_eval_accumulate leaves on the device:
    counts[:C*C] confusion matrix (true row, predicted column), counts[C*C] top-k hits, counts[C*C+1] samples."""
    counts = np.asarray(counts, np.int64)
    c = int(round((counts.size - 2) ** 0.5))
    cm = counts[:c * c].reshape(c, c)
    n = max(int(counts[c * c + 1]), 1)
    res: Dict[str, object] = {"accuracy": float(np.trace(cm)) / n, "top5_accuracy": float(counts[c * c]) / n}
    if use_class_metrics:
        for k, name in enumerate(label_names or [str(i) for i in range(c)]):
            tp = float(cm[k, k])
            prec = tp / max(float(cm[:, k].sum()), 1.0)
            rec = tp / max(float(cm[k, :].sum()), 1.0)
            res[f"precision/{name}"], res[f"recall/{name}"] = prec, rec
            res[f"f1score/{name}"] = 2 * prec * rec / max(prec + rec, 1e-12)
    res["confusion_matrix"] = cm.astype(np.float64)
    return res


class MetricManagerBase:
    @staticmethod
    def add_arguments(parser):
        g = parser.add_argument_group("Metric Manager Arguments")
        g.add_argument("--exclude_metric_names", nargs="*", default=[], type=str)
        g.add_argument("--max_summary_outputs", default=3, type=int)
        g.add_argument("--host_metrics", dest="device_metrics", action="store_false",
                       help="ship every batch's [batch, classes] outputs to the host and compute the metrics there (adds mAP, "
                            "stable-sort ranking without tie groups); default: confusion-matrix counts accumulated on the device, "
                            "and the scores ranked on the device once per evaluation")
        g.set_defaults(device_metrics=True)


class AudioMetricManager(MetricManagerBase):
    def __init__(self, is_training: bool, use_class_metrics: bool, exclude_metric_names: List[str],
                 summary: Optional[Summaries] = None):
        self.is_training, self.use_class_metrics = is_training, use_class_metrics
        self.exclude = set(exclude_metric_names or [])
        self.results: Dict[int, Dict[str, float]] = {}
        self.summary = summary
        self.summary_table: List[tuple] = []

    def build_metric_ops(self, data):          # tensor metrics (losses / learning rate) are fetched with the step
        """Registers the step summaries of metrics/manager.py:20-37 as (op, tag, value type, collection) rows: LossesMetricOp
        (metric_loss/<split>/<loss>), and in training LearningRateSummaryOp (learning_rate/<split>) and WavSummaryOp
        (wav/<split>), each in DEFAULT as the reference registers them; an op named in --exclude_metric_names is left out.
        The evaluation metrics are written under their result keys (write_evaluation_summaries)."""
        self.label_names = data["label_names"]
        split = self.split = data["dataset_split_name"]
        rows = [("LossesMetricOp", f"metric_loss/{split}/{name}", VALUE_TYPES.SCALAR, KEY_TYPES.DEFAULT) for name in data["losses"]]
        if self.is_training:
            if data.get("learning_rate") is not None:
                rows.append(("LearningRateSummaryOp", f"learning_rate/{split}", VALUE_TYPES.SCALAR, KEY_TYPES.DEFAULT))
            rows.append(("WavSummaryOp", f"wav/{split}", VALUE_TYPES.AUDIO, KEY_TYPES.DEFAULT))
        self.summary_table = [r for r in rows if r[0] not in self.exclude]
        return {}

    def step_summary_tags(self, collection_keys) -> List[tuple]:
        return [r for r in self.summary_table if r[3] in collection_keys]

    def wants_clips(self, collection_keys) -> bool:
        return self.summary is not None and any(r[2] == VALUE_TYPES.AUDIO for r in self.step_summary_tags(collection_keys))

    def write_step_summaries(self, step, collection_keys, losses: Dict[str, float], learning_rate=None, clips=None):
        """The step summaries of `collection_keys` at `step`: the step's losses by name, its learning rate and its first
        --max_outputs clips [n, samples] (tf.summary.audio at 16 kHz).  Values that are None are skipped."""
        if self.summary is None:
            return
        values = []
        for op, tag, kind, _ in self.step_summary_tags(collection_keys):
            loss = losses.get(tag[len(f"metric_loss/{self.split}/"):]) if op == "LossesMetricOp" else None
            if loss is not None:
                values.append(scalar_value(tag, loss))
            elif op == "LearningRateSummaryOp" and learning_rate is not None:
                values.append(scalar_value(tag, learning_rate))
            elif kind == VALUE_TYPES.AUDIO and clips is not None:
                values += audio_values(tag, clips, self.summary.sample_rate, self.summary.max_outputs)
        self.summary.write(step, values)

    def get_best_keep_metric_with_modes(self):
        return {"accuracy": "max"}

    def evaluate_and_aggregate_metrics(self, step, non_tensor_data, eval_dict):
        if non_tensor_data.get("metric_counts") is not None:          # device path: classes^2 + 2 integers per evaluation
            res = metrics_from_counts(non_tensor_data["metric_counts"], non_tensor_data["label_names"], self.use_class_metrics)
            if non_tensor_data.get("ranking") is not None:
                res.update(ranking_metrics(non_tensor_data["ranking"], non_tensor_data["label_names"], self.use_class_metrics))
            if "total_loss" in eval_dict:
                res["total_loss"] = float(np.mean(eval_dict["total_loss"]))
            self.results[int(step)] = {k: v for k, v in res.items() if k not in self.exclude}
            return
        labels, preds = non_tensor_data["labels_onehot"], non_tensor_data["predictions_onehot"]
        y, p = labels.argmax(1), preds.argmax(1)
        res = {"accuracy": float(np.mean(y == p)), "top5_accuracy": topn_accuracy(labels, preds, 5)}
        aps = [average_precision(labels[:, c], preds[:, c]) for c in range(labels.shape[1])]
        res["mAP"] = float(np.nanmean(aps)) if not np.all(np.isnan(aps)) else float("nan")
        res.update(ranking_metrics(ranking_vector(labels, preds), non_tensor_data["label_names"], self.use_class_metrics))
        if "total_loss" in eval_dict:
            res["total_loss"] = float(np.mean(eval_dict["total_loss"]))
        if self.use_class_metrics:
            for c, name in enumerate(non_tensor_data["label_names"]):
                tp = float(np.sum((p == c) & (y == c)))
                prec = tp / max(float(np.sum(p == c)), 1.0)
                rec = tp / max(float(np.sum(y == c)), 1.0)
                res[f"precision/{name}"], res[f"recall/{name}"] = prec, rec
                res[f"f1score/{name}"] = 2 * prec * rec / max(prec + rec, 1e-12)
        res["confusion_matrix"] = np.histogram2d(y, p, bins=labels.shape[1], range=[[0, labels.shape[1]]] * 2)[0]
        self.results[int(step)] = {k: v for k, v in res.items() if k not in self.exclude}

    def get_evaluation_result(self, step):
        return self.results[int(step)]

    def filter_best_keep_metric(self, metric_dict):
        return {k: v for k, v in metric_dict.items() if k in self.get_best_keep_metric_with_modes()}

    def log_metrics(self, step, log=print):
        scalars = {k: round(v, 5) for k, v in self.results[int(step)].items() if np.isscalar(v)}
        log(f"[step {step}] " + " / ".join(f"{k}: {v}" for k, v in scalars.items() if "/" not in k or k.startswith("mAP/")))

    def write_evaluation_summaries(self, step, collection_keys=(KEY_TYPES.DEFAULT,)):
        """Every scalar result of the evaluation at `step` (the keys of the log line and the per-class ones), in DEFAULT as the
        reference's non-tensor metric ops; the file is flushed."""
        if self.summary is None or KEY_TYPES.DEFAULT not in collection_keys:
            return
        res = self.results[int(step)]
        self.summary.write(int(step), [scalar_value(k, v) for k, v in res.items() if np.isscalar(v)])
        self.summary.flush()

    def close_summaries(self):
        if self.summary is not None:
            self.summary.close()
