"""TEST INFRASTRUCTURE (never imported by tc-resnet_b200/): NumPy restatement of the count-based evaluation metrics of the
reference, to check tcr_eval_accumulate (csrc/tcr_metrics.cu) and metrics.manager.metrics_from_counts.

Follows the reference's own rules, not the kernel's: labels / predictions = np.argmax of the one-hot and score rows
(metrics/parser.py:135-147; the first NaN if a row has one, else the first maximum), accuracy = sklearn accuracy_score
(metrics/ops/non_tensor_ops.py:64-101), top-k = the label is among np.argsort(-scores)[:, :k] (metrics/funcs.py:4-19, which puts
every NaN after every number), per-class precision / recall / F1 (:146-295) and the confusion matrix.  The sort is
kind="stable": equal scores keep the lower class first.  The reference's default sort leaves the order of equal scores to NumPy's
implementation, and k >= classes counts every row where the reference asserts k <= classes (SURVEY.md §9)."""
import numpy as np


def top_k_hits(scores, labels, k):
    """Per row: the label is among the first k classes of np.argsort(-scores, kind="stable")."""
    top = np.argsort(-np.asarray(scores), axis=1, kind="stable")[:, :k]
    return (top == np.asarray(labels)[:, None]).any(1)


def eval_counts(scores, onehot, topk=5):
    scores, onehot = np.asarray(scores), np.asarray(onehot)
    n, c = scores.shape
    y, p = np.argmax(onehot, 1), np.argmax(scores, 1)
    counts = np.zeros(c * c + 2, np.int64)
    np.add.at(counts, y * c + p, 1)
    counts[c * c] = int(top_k_hits(scores, y, topk).sum())
    counts[c * c + 1] = n
    return counts
