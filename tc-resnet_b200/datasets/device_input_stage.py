"""The per-clip input stage on the device (SURVEY.md 8f "next" row 1): host side.

The reference runs decode_wav, pad/crop, time shift, background mix and clipping per file on `tf.data` host threads
(datasets/augmentation_factory.py:30-211, datasets/audio_data_wrapper.py:37-58).  Here the host only makes the random DRAWS
(24 bytes per clip) and ships the wav files' own int16 samples; tcr_augment_pcm16 (csrc/tcr_augment.cu) does the arithmetic for the
whole batch in one HBM-bound pass, bit-identical to the host stage (augmentation_factory.py in this package) for the same draws.
"""
from __future__ import annotations

from concurrent.futures import ThreadPoolExecutor
from typing import Optional, Sequence

import numpy as np
import torch

from .. import _lib as L
from .augmentation_factory import read_wav_pcm16

# tcr_augment_clip (include/tcr_b200.h)
CLIP_DTYPE = np.dtype([("length", "<i4"), ("shift", "<i4"), ("silent", "<i4"), ("bg_volume", "<f4"), ("bg_offset", "<i8")])
# tcr_dataset_clip (include/tcr_b200.h)
DATASET_CLIP_DTYPE = np.dtype([("offset", "<i8"), ("length", "<i4"), ("label", "<i4")])


def draw_clips(rng: np.random.RandomState, lengths: Sequence[int], silent: Sequence[bool], clip_samples: int,
               bg_lengths: Sequence[int], shift: bool = True, is_training: bool = True, background_frequency: float = 0.8,
               background_max_volume: float = 0.1, shift_ratio: float = 0.1) -> np.ndarray:
    """One record per clip, drawn in the order of the reference's graph: time shift (augmentation_factory.py:104-112),
    background choice and random crop (:58-67), background volume ("naive" version, :69-80)."""
    n = len(lengths)
    clips = np.zeros(n, CLIP_DTYPE)
    starts = np.concatenate([[0], np.cumsum(bg_lengths)])[:-1] if len(bg_lengths) else np.zeros(0, np.int64)
    limit = int(clip_samples * shift_ratio)
    for i in range(n):
        clips[i]["length"] = int(lengths[i])
        clips[i]["silent"] = int(bool(silent[i]))
        clips[i]["shift"] = int(rng.randint(-limit, limit)) if (shift and limit) else 0
        clips[i]["bg_offset"] = -1
        if len(bg_lengths):
            b = int(rng.randint(0, len(bg_lengths)))
            # recordings shorter than a clip are zero-padded to clip length by DeviceInputStage (tf.random_crop would raise)
            clips[i]["bg_offset"] = int(starts[b]) + int(rng.randint(0, max(bg_lengths[b] - clip_samples, 0) + 1))
            mixed = is_training and rng.uniform() < background_frequency
            clips[i]["bg_volume"] = np.float32(rng.uniform(0.0, background_max_volume)) if mixed else np.float32(0.0)
    return clips


def pack(clips: np.ndarray, device) -> torch.Tensor:
    """The records as the uint8 CUDA tensor Engine.augment takes."""
    assert clips.dtype == CLIP_DTYPE
    return torch.from_numpy(np.frombuffer(np.ascontiguousarray(clips).tobytes(), np.uint8).copy()).to(device)


class DeviceInputStage:
    """Background bank resident in HBM + one call per batch: int16 clips and draws in, fp32 wav [n, clip_samples] out."""

    def __init__(self, engine, background_data: Optional[Sequence[np.ndarray]] = None):
        self.engine = engine
        clip = int(engine.cfg.clip_samples)
        bank = [np.asarray(b, np.float32).reshape(-1) for b in (background_data or [])]
        bank = [np.pad(b, (0, clip - b.shape[0])) if b.shape[0] < clip else b for b in bank]     # every crop fits its recording
        self.bg_lengths = [int(b.shape[0]) for b in bank]
        self.background = torch.from_numpy(np.concatenate(bank)).to(engine.device) if bank else None
        if bank:                                     # the kernel refuses crops that would run past the bank
            engine.lib.tcr_set_background_samples(engine._h, int(sum(self.bg_lengths)))

    def __call__(self, pcm: torch.Tensor, clips: np.ndarray, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        return self.engine.augment(pcm, pack(clips, self.engine.device), self.background, out=out)


def decode_clip_bank(filenames: Sequence[str], labels: Sequence[int], clip_samples: int, num_threads: int = 8):
    """Every clip of a split decoded once, with `num_threads` workers: (int16 bank, DATASET_CLIP_DTYPE table).  A clip keeps at
    most clip_samples samples (decode_wav's crop); a "" filename (a silent sample) is stored with length 0."""
    def read(f):
        return np.zeros(0, np.int16) if f == "" else read_wav_pcm16(f)[:clip_samples]
    with ThreadPoolExecutor(max(1, int(num_threads))) as ex:
        clips = list(ex.map(read, filenames))
    lengths = np.array([c.shape[0] for c in clips], np.int64)
    table = np.zeros(len(clips), DATASET_CLIP_DTYPE)
    table["offset"] = np.cumsum(lengths) - lengths
    table["length"], table["label"] = lengths, np.asarray(labels, np.int64)
    bank = np.empty(int(lengths.sum()), np.int16)
    for i in range(len(clips)):
        bank[table["offset"][i]:table["offset"][i] + lengths[i]] = clips[i]
        clips[i] = None
    return bank, table


class DeviceDataset:
    """A split resident in device memory (tcr_dataset, include/tcr_b200.h): the clip bank, its table, the background bank
    (through DeviceInputStage) and two order buffers.  Each epoch's order is uploaded once, into the buffer the epoch before the
    last one used; an event recorded when that epoch's last step was submitted guards the overwrite."""

    def __init__(self, engine, bank: np.ndarray, table: np.ndarray, background_data=None, shift: bool = True, mix: bool = True,
                 is_training: bool = True, background_frequency: float = 0.8, background_max_volume: float = 0.1):
        self.engine = engine
        dev = engine.device
        clip = int(engine.cfg.clip_samples)
        bg = [np.asarray(b, np.float32).reshape(-1) for b in (background_data or [])]
        bg_floats = sum(max(b.shape[0], clip) for b in bg)
        need = bank.nbytes + table.nbytes + 2 * 4 * len(table) + 4 * bg_floats + 16 * len(bg)
        free, _ = torch.cuda.mem_get_info(dev)
        if need > free:
            raise MemoryError(f"--device_dataset: the split needs {need} bytes of device memory, {free} bytes are free")
        self.num_clips = len(table)
        self.samples = torch.from_numpy(np.ascontiguousarray(bank, np.int16)).to(dev)
        self.table = torch.from_numpy(np.frombuffer(np.ascontiguousarray(table, DATASET_CLIP_DTYPE).tobytes(), np.uint8).copy()).to(dev)
        self.stage = DeviceInputStage(engine, bg)
        starts = np.cumsum(self.stage.bg_lengths) - np.asarray(self.stage.bg_lengths, np.int64) if bg else np.zeros(0, np.int64)
        self.bg_table = torch.from_numpy(np.stack([starts, np.asarray(self.stage.bg_lengths, np.int64)], 1).reshape(-1)
                                         if bg else np.zeros(2, np.int64)).to(dev)
        # empty, not zeros: the uploads run on their own stream and must not race a fill queued on the current one
        self.orders = [torch.empty(max(self.num_clips, 1), dtype=torch.int32, device=dev) for _ in range(2)]
        self._released = [None, None]                 # event: every step that read the buffer has finished
        self._copy = torch.cuda.Stream(dev)
        self.current = 1
        self.desc = L.TcrDataset()
        d = self.desc
        d.samples, d.num_samples = self.samples.data_ptr(), self.samples.numel()
        d.clips, d.num_clips = self.table.data_ptr(), self.num_clips
        d.background = self.stage.background.data_ptr() if bg else None
        d.background_samples = int(sum(self.stage.bg_lengths))
        d.background_table, d.num_background = self.bg_table.data_ptr(), len(bg)
        d.shift, d.mix, d.is_training = int(bool(shift)), int(bool(mix) and bool(bg)), int(bool(is_training))
        d.background_frequency, d.background_max_volume = float(background_frequency), float(background_max_volume)

    def upload_order(self, order: np.ndarray):
        """Makes `order` (the epoch's sample indices) the order the following batches read.  Returns when it is on the device."""
        stream = torch.cuda.current_stream(self.engine.device)
        self._released[self.current] = stream.record_event()      # every step reading the current buffer is submitted by now
        b = self.current ^ 1
        if self._released[b] is not None:
            self._released[b].synchronize()
        with torch.cuda.stream(self._copy):
            self.orders[b][:len(order)].copy_(torch.from_numpy(np.ascontiguousarray(order, np.int32)))
        self._copy.synchronize()
        self.current = b
        self.desc.order, self.desc.order_length = self.orders[b].data_ptr(), len(order)

    def batch(self, position: int, epoch: int, seed: int, n: int, wav_out: Optional[torch.Tensor] = None,
              onehot_out: Optional[torch.Tensor] = None):
        """(wav [n, clip_samples], one-hot [n, classes]) of rows [position, position + n) of the current order (tcr_dataset_batch)."""
        return self.engine.dataset_batch(self.desc, position, epoch, seed, n, wav_out, onehot_out)
