"""Host-side (NumPy) restatement of the reference's per-clip input stage (datasets/augmentation_factory.py):
wav decode int16/32768 -> f32, pad/crop to `desired_samples` (:146-158), +-10 % time shift (:104-143),
background-noise mix p=0.8 / volume U(0, 0.1) and clip to [-1,1] (:30-101, "naive" version).
It produces the contract the hot path consumes: f32 [desired_samples] in [-1, 1].  Moving this stage onto the
GPU is the first "next" row of SURVEY.md 8(f); it is not on the measured path (bench uses synthetic clips)."""
from __future__ import annotations

import wave

import numpy as np

_available_audio_augmentation_methods = ["anchored_slice_or_pad", "anchored_slice_or_pad_with_shift", "no_augmentation_audio"]
_available_augmentation_methods = _available_audio_augmentation_methods + ["no_augmentation"]


def read_wav_pcm16(filename: str) -> np.ndarray:
    """The int16 samples of a 16-bit PCM wav file, channel 0 only (decode_wav's input, before its 1/32768 scaling)."""
    with wave.open(filename, "rb") as w:
        nch, width, nframes = w.getnchannels(), w.getsampwidth(), w.getnframes()
        raw = w.readframes(nframes)
    if width != 2:
        raise ValueError(f"{filename}: only 16-bit PCM wav is supported")
    data = np.frombuffer(raw, dtype="<i2")
    return data.reshape(-1, nch)[:, 0] if nch > 1 else data


def load_wav_file(filename: str, desired_samples: int) -> np.ndarray:
    data = read_wav_pcm16(filename).astype(np.float32) / 32768.0
    if desired_samples > 0:
        out = np.zeros(desired_samples, np.float32)
        m = min(desired_samples, data.shape[0])
        out[:m] = data[:m]
        return out
    return data


def shift_audio(audio: np.ndarray, rng: np.random.RandomState, shift_ratio: float = 0.1) -> np.ndarray:
    n = audio.shape[0]
    limit = int(n * shift_ratio)
    amount = int(rng.randint(-limit, limit)) if limit > 0 else 0
    out = np.zeros_like(audio)
    if amount >= 0:
        out[amount:] = audio[:n - amount]
    else:
        out[:n + amount] = audio[-amount:]
    return out


def mix_background(audio, background_data, rng, is_training, background_frequency, background_max_volume):
    n = audio.shape[0]
    bg = background_data[int(rng.randint(0, len(background_data)))]
    start = int(rng.randint(0, max(1, bg.shape[0] - n + 1)))
    crop = np.zeros(n, np.float32)
    seg = bg[start:start + n]
    crop[:seg.shape[0]] = seg
    volume = 0.0
    if is_training and rng.uniform() < background_frequency:
        volume = float(rng.uniform(0.0, background_max_volume))
    return np.clip(crop * volume + audio, -1.0, 1.0).astype(np.float32)


def get_audio_augmentation_fn(name):
    if name not in _available_audio_augmentation_methods:
        raise ValueError(f"Augmentation name [{name}] was not recognized")

    def fn(filename, desired_samples, rng, background_data=None, is_training=False, background_frequency=0.0,
           background_max_volume=0.0):
        audio = np.zeros(desired_samples, np.float32) if filename == "" else load_wav_file(filename, desired_samples)
        if name == "no_augmentation_audio":
            return audio
        if name == "anchored_slice_or_pad_with_shift":
            audio = shift_audio(audio, rng)
        if background_data:
            audio = mix_background(audio, background_data, rng, is_training, background_frequency, background_max_volume)
        return audio
    return fn
