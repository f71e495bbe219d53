"""NumPy restatement of the resident dataset's input stage (tcr_dataset, include/tcr_b200.h) — TEST INFRASTRUCTURE ONLY.

The draws (uint64 SplitMix64 keyed by seed, epoch and global position) and the gather from the clip bank, as the kernel makes
them (tc-resnet_b200/csrc/tcr_augment.cu).  Together with oracle/augment_oracle.augment they give the batch bit for bit."""
from __future__ import annotations

import numpy as np

from oracle import augment_oracle as A

_U = np.uint64


def splitmix64(seed, idx) -> np.ndarray:
    """SplitMix64 output for the state seed + 0x9E3779B97F4A7C15 * (idx + 1), elementwise, wrapping mod 2^64."""
    with np.errstate(over="ignore"):
        z = _U(seed) + _U(0x9E3779B97F4A7C15) * (np.asarray(idx, np.uint64) + _U(1))
        z = (z ^ (z >> _U(30))) * _U(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> _U(27))) * _U(0x94D049BB133111EB)
        return z ^ (z >> _U(31))


def uniform01(z) -> np.ndarray:
    """The top 24 bits as an fp32 in [0, 1)."""
    return (np.asarray(z, np.uint64) >> _U(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def draws(seed, epoch, positions, clip_samples, bg_lengths, shift=True, mix=True, is_training=True, background_frequency=0.8,
          background_max_volume=0.1):
    """dict of per-position draws: shift, recording, crop, mixed, volume (fp32), bg_offset (recording start + crop, -1: none)."""
    p = np.asarray(positions, np.uint64)
    key = splitmix64(seed, np.uint64(epoch))
    z = [splitmix64(key, _U(8) * p + _U(k)) for k in range(5)]
    limit = int(clip_samples * 0.1)
    n = p.shape[0]
    out = dict(shift=np.zeros(n, np.int64), recording=np.full(n, -1, np.int64), crop=np.zeros(n, np.int64),
               mixed=np.zeros(n, bool), volume=np.zeros(n, np.float32), bg_offset=np.full(n, -1, np.int64))
    if shift and limit > 0:
        out["shift"] = (z[0] % _U(2 * limit)).astype(np.int64) - limit
    nb = len(bg_lengths)
    if mix and nb:
        lengths = np.asarray(bg_lengths, np.int64)
        starts = np.cumsum(lengths) - lengths
        b = (z[1] % _U(nb)).astype(np.int64)
        crop = (z[2] % (np.maximum(lengths[b] - clip_samples, 0) + 1).astype(np.uint64)).astype(np.int64)
        mixed = bool(is_training) & (uniform01(z[3]) < np.float32(background_frequency))
        out.update(recording=b, crop=crop, mixed=mixed, bg_offset=starts[b] + crop,
                   volume=np.where(mixed, uniform01(z[4]) * np.float32(background_max_volume), np.float32(0)).astype(np.float32))
    return out


def batch(bank, table, order, position, n, seed, epoch, clip_samples, num_classes, background=None, bg_lengths=(), **kw):
    """(fp32 wav [n, clip_samples], one-hot [n, num_classes]) of rows [position, position + n) of `order`: the gather, these
    draws and augment_oracle.augment."""
    idx = np.asarray(order[position:position + n], np.int64)
    pcm = np.zeros((n, clip_samples), np.int16)
    clips = np.zeros(n, A.CLIP_DTYPE)
    hot = np.zeros((n, num_classes), np.float32)
    for i, c in enumerate(idx):
        off, length, label = int(table["offset"][c]), min(int(table["length"][c]), clip_samples), int(table["label"][c])
        pcm[i, :length] = bank[off:off + length]
        clips[i]["length"] = length
        hot[i, label] = 1.0
    d = draws(seed, epoch, np.arange(position, position + n), clip_samples, list(bg_lengths), **kw)
    clips["shift"] = d["shift"]
    clips["bg_volume"] = d["volume"]
    clips["bg_offset"] = d["bg_offset"] if background is not None else -1
    return A.augment(pcm, clips, background, clip_samples), hot
