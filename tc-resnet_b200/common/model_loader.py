"""Which variables a run trains and which it restores, by TF variable name.

  variables_to_train    --trainable_scopes: common/tf_utils.py:19-37 (re.match of each scope on `<var>:0`)
  restore_filter        --checkpoint_include_scopes / --checkpoint_exclude_scopes: common/model_loader.py:42-83 (startswith on
                        the name without `:0`, so a scope also covers that variable's optimizer slots and EMA shadow)
  ema_restore_values    evaluation with --use_ema: helper/evaluator.py:41-48 + common/model_loader.py:62-67 (every trainable
                        variable is read from `<var>/ExponentialMovingAverage`, the BN moving statistics under their own names)
"""
from __future__ import annotations

import re
from typing import Callable, Dict, List, Sequence

import numpy as np

EMA_SUFFIX = "/ExponentialMovingAverage"


def split_strip(scopes: str) -> List[str]:
    return [s for s in (x.strip() for x in (scopes or "").split(",")) if s]


def variables_to_train(trainable_scopes: str, trainable_names: Sequence[str], log=None) -> List[str]:
    """The trained variables in table order.  Empty scopes: every trainable variable.  Otherwise each comma-separated, stripped
    scope selects the variables whose `<name>:0` it re.match-es (anchored at the start, a regex: "TCResNet8/block2",
    ".*BatchNorm").  Two deliberate deviations from the reference (SURVEY.md section 9): an empty selection raises ValueError (the
    reference's train op becomes tf.no_op() and the loop never ends), and so does a variable selected by two scopes (the
    reference would list it twice in var_list)."""
    if not trainable_scopes:
        return list(trainable_names)
    scopes = [s.strip() for s in trainable_scopes.split(",")]
    picked: Dict[str, str] = {}
    for scope in scopes:
        rx = re.compile(scope)
        for name in trainable_names:
            if rx.match(name + ":0"):
                if name in picked:
                    raise ValueError(f"--trainable_scopes: {name} is selected by both {picked[name]!r} and {scope!r}")
                picked[name] = scope
    if not picked:
        raise ValueError(f"--trainable_scopes {trainable_scopes!r} selects no trainable variable")
    out = [n for n in trainable_names if n in picked]
    if log is not None:
        for name in out:
            log.info(f"vars to train > {name}:0")
    return out


def restore_filter(include_scopes: str = "", exclude_scopes: str = "") -> Callable[[str], bool]:
    """Predicate on a variable name: restored when it starts with an include scope (all, when there are none) and with no
    exclude scope."""
    inc, exc = split_strip(include_scopes), split_strip(exclude_scopes)

    def keep(name: str) -> bool:
        if inc and not any(name.startswith(p) for p in inc):
            return False
        return not any(name.startswith(p) for p in exc)
    return keep


def evaluation_restore(args, values: Dict[str, np.ndarray], trainable_names: Callable[[], Sequence[str]]):
    """(values, restore predicate) for AudioNetModel.set_variables as evaluation restores a checkpoint (helper/evaluator.py, and
    listen_audio.py): filtered by --checkpoint_{include,exclude}_scopes, or with --use_ema every trainable variable (the names
    `trainable_names()` returns) taken from its shadow.  --use_ema together with a scope filter is rejected (the reference crashes
    on it, SURVEY.md section 9)."""
    include = getattr(args, "checkpoint_include_scopes", "")
    exclude = getattr(args, "checkpoint_exclude_scopes", "")
    if getattr(args, "use_ema", False):
        if split_strip(include) or split_strip(exclude):
            raise ValueError("--use_ema cannot be combined with --checkpoint_include_scopes / --checkpoint_exclude_scopes")
        return ema_restore_values(values, trainable_names()), None
    return values, restore_filter(include, exclude)


def ema_restore_values(values: Dict[str, np.ndarray], trainable_names: Sequence[str]) -> Dict[str, np.ndarray]:
    """The checkpoint as the evaluator restores it with --use_ema: each trainable variable takes its shadow's value; one without
    a shadow in the checkpoint is absent (missing unless --ignore_missing_vars, which leaves its initial value)."""
    out = {k: v for k, v in values.items() if not k.endswith(EMA_SUFFIX)}
    for name in trainable_names:
        out.pop(name, None)
        if name + EMA_SUFFIX in values:
            out[name] = values[name + EMA_SUFFIX]
    return out
