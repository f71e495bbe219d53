#!/usr/bin/env python
"""`python evaluate_audio.py <reference flags> <ModelName> <model flags>` — the reference's evaluation CLI
(evaluate_audio.py:19-87): `--valid_type once` evaluates one checkpoint, `--valid_type loop` follows the
training directory and evaluates every new checkpoint (the trainer and evaluator are two processes coupled only
through that directory)."""
from __future__ import annotations

import argparse
import os
import sys
from typing import List

if __package__ in (None, ""):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import tcresnet_b200  # noqa: F401
    __package__ = "tcresnet_b200"

from . import const  # noqa: E402
from .common import checkpoint as ckpt  # noqa: E402
from .common import utils  # noqa: E402
from .datasets.audio_data_wrapper import AudioDataWrapper, SingleLabelAudioDataWrapper  # noqa: E402
from .datasets.data_wrapper_base import DataWrapperBase  # noqa: E402
from .factory import audio_nets  # noqa: E402
from .factory.base import TFModel  # noqa: E402
from .helper.base import Base  # noqa: E402
from .helper.evaluator import Evaluator, SingleLabelAudioEvaluator  # noqa: E402
from .metrics.manager import MetricManagerBase  # noqa: E402
from .runtime import Session  # noqa: E402


def main(args, loop_timeout=None):
    is_training = False
    dataset_name = args.dataset_split_name[0]
    session = Session(config=const.TF_SESSION_CONFIG)
    dataset = SingleLabelAudioDataWrapper(args, session, dataset_name, is_training)
    wavs, labels = dataset.get_input_and_output_op()
    model = getattr(audio_nets, args.model)(args, dataset)
    model.build(wavs=wavs, labels=labels, is_training=is_training)
    evaluator = SingleLabelAudioEvaluator(model, session, args, dataset, dataset_name)
    log = utils.get_logger("EvaluateAudio")
    results = []
    try:
        if args.valid_type == "once":
            results.append(evaluator.evaluate_once(ckpt.resolve_checkpoint_path(args.checkpoint_path)))
        elif args.valid_type == "loop":
            log.info(f"Start Loop: watching {evaluator.watch_path}")
            for path in ckpt.checkpoints_iterator(evaluator.watch_path, timeout=loop_timeout):
                log.info(f"[watch] {path}")
                results.append(evaluator.evaluate_once(path))
        else:
            raise ValueError(f"Undefined valid_type: {args.valid_type}")
    finally:
        evaluator.metric_manager.close_summaries()
    return results


def parse_arguments(arguments: List[str] = None):
    parser = argparse.ArgumentParser(description=__doc__)
    subparsers = parser.add_subparsers(title="Model", description="")
    Base.add_arguments(parser)
    Evaluator.add_arguments(parser)
    DataWrapperBase.add_arguments(parser)
    AudioDataWrapper.add_arguments(parser)
    TFModel.add_arguments(parser)
    audio_nets.AudioNetModel.add_arguments(parser)
    MetricManagerBase.add_arguments(parser)
    for class_name in audio_nets._available_nets:
        sub = subparsers.add_parser(class_name)
        sub.add_argument("--model", default=class_name, type=str, help="DO NOT FIX ME")
        getattr(audio_nets, class_name).add_arguments(sub)
    return parser.parse_args(arguments)


if __name__ == "__main__":
    args = parse_arguments()
    utils.get_logger("AudioNetEvaluate").info(args)
    main(args)
