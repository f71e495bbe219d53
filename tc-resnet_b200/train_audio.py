#!/usr/bin/env python
"""`python train_audio.py <reference flags> <ModelName> <model flags>` — same command lines as the reference's
train_audio.py (e.g. scripts/commands/TCResNet8Model-1.0_mfcc_40_3010_0.001_mom_l1.sh line 3), executing on the
H100 CUDA path.  The model is an argparse sub-command placed last; it is looked up by name in factory.audio_nets."""
from __future__ import annotations

import argparse
import os
import sys
from typing import List

if __package__ in (None, ""):      # run as a script: make the package importable under its alias
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import tcresnet_b200  # noqa: F401
    __package__ = "tcresnet_b200"

from . import const  # noqa: E402
from .common import utils  # noqa: E402
from .datasets.audio_data_wrapper import AudioDataWrapper, SingleLabelAudioDataWrapper  # noqa: E402
from .datasets.data_wrapper_base import DataWrapperBase  # noqa: E402
from .factory import audio_nets  # noqa: E402
from .factory.base import TFModel  # noqa: E402
from .helper.base import Base  # noqa: E402
from .helper.trainer import SingleLabelAudioTrainer, TrainerBase  # noqa: E402
from .metrics.manager import MetricManagerBase  # noqa: E402
from .runtime import Session  # noqa: E402


def train(args):
    is_training = True
    dataset_name = args.dataset_split_name[0]
    if getattr(args, "data_parallel", False):
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        if not dist.is_initialized():
            dist.init_process_group("nccl")
    session = Session(config=const.TF_SESSION_CONFIG)
    dataset = SingleLabelAudioDataWrapper(args, session, dataset_name, is_training)
    wavs, labels = dataset.get_input_and_output_op()
    model = getattr(audio_nets, args.model)(args, dataset)
    model.build(wavs=wavs, labels=labels, is_training=is_training)
    trainer = SingleLabelAudioTrainer(model, session, args, dataset, dataset_name)
    trainer.train()
    return trainer


def parse_arguments(arguments: List[str] = None):
    parser = argparse.ArgumentParser(description=__doc__)
    subparsers = parser.add_subparsers(title="Model", description="")
    TFModel.add_arguments(parser)
    audio_nets.AudioNetModel.add_arguments(parser)
    for class_name in audio_nets._available_nets:
        sub = subparsers.add_parser(class_name)
        sub.add_argument("--model", default=class_name, type=str, help="DO NOT FIX ME")
        getattr(audio_nets, class_name).add_arguments(sub)
    DataWrapperBase.add_arguments(parser)
    AudioDataWrapper.add_arguments(parser)
    Base.add_arguments(parser)
    TrainerBase.add_arguments(parser)
    SingleLabelAudioTrainer.add_arguments(parser)
    MetricManagerBase.add_arguments(parser)
    return parser.parse_args(arguments)


if __name__ == "__main__":
    args = parse_arguments()
    log = utils.get_logger("Trainer")
    utils.update_train_dir(args)
    log.info(args)
    train(args)
