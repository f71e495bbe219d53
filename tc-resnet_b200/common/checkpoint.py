"""Checkpoint I/O keyed by the reference's TF variable names.

The reference saves TF-V2 tensor bundles with tf.train.Saver every `step_save_checkpoint` steps as
`<train_dir>/<Model>-<step>` (helper/trainer.py:406-414) and the evaluator process discovers them through the
directory (common/tf_utils.py:65-67, 219-247).  Two on-disk formats, same names / directory protocol:
  "tf"  (default)  <train_dir>/<Model>-<step>.index + .data-00000-of-00001 + the `checkpoint` state file: the tensor-bundle
                   format of tf.train.Saver, written / read by common/tf_bundle.py, so reference-trained weights load here
                   and checkpoints written here open with tf.train.load_checkpoint
  "npz"            <train_dir>/<Model>-<step>.npz (one NumPy archive)
Content: {TF variable name: array, the optimizer's state under TF's names, "global_step": int64}.  The optimizer state is
"<var>/Momentum" (mom, gd), "<var>/Adam" + "<var>/Adam_1" + the scalars "beta1_power" / "beta2_power" (adam), or
"<var>/RMSProp" + "<var>/RMSProp_1" (rmsprop).
"""
from __future__ import annotations

import os
import re
import shutil
import time
from pathlib import Path
from typing import Dict, Iterator, List, Optional

import numpy as np

from . import tf_bundle

_STEP = re.compile(r"-(\d+)(?:\.npz|\.index)?$")


def checkpoint_step(path) -> int:
    """Global step parsed from the file name (common/tf_utils.py:237-247); 0 when absent."""
    m = _STEP.search(str(path))
    return int(m.group(1)) if m else 0


def _candidates(directory) -> List[str]:
    """Complete checkpoints of a directory as load()-able paths: `<stem>.npz` files and bundle prefixes (`<stem>` of `<stem>.index`)."""
    d = Path(directory)
    out = [str(p) for p in d.glob("*-*.npz") if not p.name.startswith(".") and _STEP.search(p.name)]
    out += [str(p)[:-len(".index")] for p in d.glob("*-*.index") if not p.name.startswith(".") and _STEP.search(p.name)]
    return sorted(out, key=checkpoint_step)


def checkpoint_files(path) -> List[Path]:
    """Every file that belongs to one checkpoint (for copying the best one, helper/evaluator.py)."""
    p = str(path)
    if p.endswith(".npz"):
        return [Path(p)]
    pre = Path(p[:-len(".index")] if p.endswith(".index") else p)
    return [Path(str(pre) + ".index")] + sorted(pre.parent.glob(pre.name + ".data-*"))


def save(train_dir, model_name: str, step: int, variables: Dict[str, np.ndarray], max_to_keep: int = 5, fmt: str = "tf") -> str:
    d = Path(train_dir)
    d.mkdir(parents=True, exist_ok=True)
    stem = f"{model_name}-{int(step)}"
    if fmt == "npz":
        path = d / (stem + ".npz")
        # unique per process and NOT matching "*.npz": neither another rank nor the watching evaluator can pick it up
        tmp = d / f".{stem}.{os.getpid()}.tmp"
        with open(tmp, "wb") as f:
            np.savez(f, global_step=np.int64(step), **variables)
        os.replace(tmp, path)                       # atomic: the watching evaluator never sees a partial file
        out = str(path)
    elif fmt == "tf":
        tensors = dict(variables)
        tensors["global_step"] = np.asarray(step, np.int64)
        out = tf_bundle.write_bundle(d / stem, tensors)               # data first, index last: a visible index is complete
    else:
        raise ValueError(f"unknown checkpoint format {fmt!r} (tf | npz)")
    kept = _candidates(d)
    mine = [c for c in kept if Path(c).name.startswith(model_name + "-")]
    for old in (mine[:-max_to_keep] if max_to_keep > 0 else []):
        for f in checkpoint_files(old):
            f.unlink(missing_ok=True)
    mine = mine[-max_to_keep:] if max_to_keep > 0 else mine
    if fmt == "tf":
        tf_bundle.write_checkpoint_state(d, Path(out).name, [Path(c).name for c in mine if not c.endswith(".npz")])
    return out


def load(path) -> Dict[str, np.ndarray]:
    p = str(path)
    if p.endswith(".npz"):
        with np.load(p) as z:
            return {k: z[k] for k in z.files}
    if p.endswith(".index"):
        p = p[:-len(".index")]
    return tf_bundle.BundleReader(p).read_all()


def latest_checkpoint(directory) -> Optional[str]:
    """tf.train.latest_checkpoint: the `checkpoint` state file when present, else the highest step in the directory."""
    d = Path(directory)
    named = tf_bundle.read_checkpoint_state(d)
    if named and (d / (named + ".index")).exists():
        return str(d / named)
    cands = _candidates(d)
    return cands[-1] if cands else None


def resolve_checkpoint_path(path: str) -> str:
    """A directory resolves to its latest checkpoint (common/tf_utils.py:219-234)."""
    if path and Path(path).is_dir():
        return latest_checkpoint(path) or ""
    return path or ""


def copy_checkpoint(path, target_dir) -> None:
    for f in checkpoint_files(path):
        shutil.copy(f, Path(target_dir) / f.name)


def checkpoints_iterator(directory, min_interval_secs: float = 0.0, timeout: Optional[float] = None) -> Iterator[str]:
    """Yields each new checkpoint as it appears (tf.contrib.training.checkpoints_iterator semantics)."""
    seen, waited = None, 0.0
    while True:
        newest = latest_checkpoint(directory)
        if newest is not None and newest != seen:
            seen, waited = newest, 0.0
            yield newest
            time.sleep(min_interval_secs)
            continue
        if timeout is not None and waited >= timeout:
            return
        time.sleep(1.0)
        waited += 1.0
