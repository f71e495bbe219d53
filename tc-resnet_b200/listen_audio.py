#!/usr/bin/env python
"""`python listen_audio.py <flags> <ModelName> <model flags> file.wav [file.wav ...]` — scores recordings with a sliding window on
the CUDA listener (include/tcr_b200.h, tcr_listener_*): one window every --hop_ms, each the model's clip length, scored exactly as
evaluate_audio.py scores a clip.  The model subcommand, the front-end flags, --checkpoint_path, --use_ema and the checkpoint
include / exclude scopes mean what they mean to evaluate_audio.py, and the checkpoint is restored the same way.

The files are streamed in parallel, one listener stream per file, --chunk_ms of each per push.  Window k of a file ends
(k + 1) * hop after its start; the windows that start before the file do so over zeros (the listener's state after a reset), and
a file's last window ends at its last sample rounded up to a whole hop (zeros again).  For each file `<name>.wav` it writes
  <name>.npy  float32 [windows, classes]: the softmax of every window;
  <name>.csv  one row per window: end time in seconds, top class, its probability."""
from __future__ import annotations

import argparse
import os
import sys
from pathlib import Path
from typing import List

import numpy as np

if __package__ in (None, ""):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import tcresnet_b200  # noqa: F401
    __package__ = "tcresnet_b200"

from .common import checkpoint as ckpt  # noqa: E402
from .common import model_loader  # noqa: E402
from .common import utils  # noqa: E402
from .datasets.audio_data_wrapper import AudioDataWrapper  # noqa: E402
from .datasets.augmentation_factory import load_wav_file  # noqa: E402
from .factory import audio_nets  # noqa: E402
from .factory.base import TFModel  # noqa: E402
from .helper.base import Base  # noqa: E402


def listen(args) -> List[np.ndarray]:
    """Scores every file of args.wav_files; returns the softmax arrays it writes, in file order."""
    log = utils.get_logger("ListenAudio")
    if args.num_classes is None:
        raise ValueError("--num_classes is required (the classes the checkpoint was trained on)")
    waves = [load_wav_file(str(f), -1) for f in args.wav_files]
    model = getattr(audio_nets, args.model)(args, None)
    sm = model.build_streaming_model(streams=len(waves), hop_ms=args.hop_ms, chunk_ms=args.chunk_ms)
    path = ckpt.resolve_checkpoint_path(args.checkpoint_path)
    if not path:
        raise ValueError(f"no checkpoint at --checkpoint_path {args.checkpoint_path!r}")
    values, restore = model_loader.evaluation_restore(args, ckpt.load(path), lambda: model.engine.trainable_names)
    model.set_variables(values, strict=not args.ignore_missing_vars, restore=restore)
    log.info(f"restored {path}; {len(waves)} stream(s), {sm.windows} window(s) of each per {args.chunk_ms} ms push")
    hop, chunk = sm.hop_samples, sm.chunk_samples
    windows = [max(1, -(-len(w) // hop)) for w in waves]
    pushes = -(-max(windows) // sm.windows)
    audio = np.zeros((len(waves), pushes * chunk), np.float32)
    for i, w in enumerate(waves):
        audio[i, :len(w)] = w
    probs = np.concatenate([sm(audio[:, p * chunk:(p + 1) * chunk]) for p in range(pushes)], axis=1)
    rate = float(args.sample_rate)
    out = []
    for f, n, pr in zip(args.wav_files, windows, probs):
        pr = np.ascontiguousarray(pr[:n], np.float32)
        stem = Path(f).stem
        d = Path(args.output_dir) if args.output_dir else Path(f).parent
        d.mkdir(parents=True, exist_ok=True)
        np.save(d / f"{stem}.npy", pr)
        top = pr.argmax(axis=1)
        with open(d / f"{stem}.csv", "w") as fh:
            fh.write("end_s,class,probability\n")
            for k in range(n):
                fh.write(f"{(k + 1) * hop / rate:.3f},{int(top[k])},{float(pr[k, top[k]]):.6f}\n")
        log.info(f"{f}: {n} windows -> {d / stem}.npy, .csv")
        out.append(pr)
    sm.listener.close()
    return out


def parse_arguments(arguments: List[str] = None):
    parser = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    subparsers = parser.add_subparsers(title="Model", description="")
    Base.add_arguments(parser)
    AudioDataWrapper.add_arguments(parser)
    TFModel.add_arguments(parser)
    audio_nets.AudioNetModel.add_arguments(parser)
    g = parser.add_argument_group("Listener")
    g.add_argument("--hop_ms", default=10.0, type=float, help="time between two windows: a whole number of frame strides")
    g.add_argument("--chunk_ms", default=100.0, type=float, help="audio per stream and push: a whole number of hops")
    g.add_argument("--output_dir", default=None, type=str, help="where the .npy / .csv files go (default: next to each wav)")
    for class_name in audio_nets._available_nets:
        sub = subparsers.add_parser(class_name)
        sub.add_argument("--model", default=class_name, type=str, help="DO NOT FIX ME")
        getattr(audio_nets, class_name).add_arguments(sub)
        sub.add_argument("wav_files", nargs="+", help="16-bit PCM wav files, one listener stream each")
    return parser.parse_args(arguments)


if __name__ == "__main__":
    args = parse_arguments()
    utils.get_logger("AudioNetListen").info(args)
    listen(args)
