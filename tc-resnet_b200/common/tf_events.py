"""TensorBoard event files in pure Python + NumPy — no TensorFlow needed.

The reference writes its summaries with tf.summary.FileWriter (metrics/summaries.py:121-128).  On disk that is a TFRecord
file `events.out.tfevents.<secs>.<host>`: records of (uint64 length, masked CRC32C of the length, payload, masked CRC32C of
the payload), each payload an `Event` proto (tensorflow/core/util/event.proto): the first carries file_version
"brain.Event:2", the others a `Summary` at a step.  Three kinds of Summary.Value are written: simple_value scalars
(tf.summary.scalar), `audio` values as tf.summary.audio builds them (16-bit PCM wav) and the string tensor with the text
plugin's metadata that tf.summary.text writes.  Protos are hand-encoded with the varint and CRC32C helpers of tf_bundle.
"""
from __future__ import annotations

import io
import socket
import struct
import time
import wave
from pathlib import Path
from typing import Dict, Iterator, List, Sequence, Tuple

import numpy as np

from .tf_bundle import _decode_fields, _field, _varint, crc32c, mask_crc, unmask_crc

_DT_STRING = 7


def _bytes(num: int, payload: bytes) -> bytes:
    return _field(num, 2) + _varint(len(payload)) + payload


def _record(payload: bytes) -> bytes:
    head = struct.pack("<Q", len(payload))
    return head + struct.pack("<I", mask_crc(crc32c(head))) + payload + struct.pack("<I", mask_crc(crc32c(payload)))


# ------------------------------------------------------------------------------------------------ Summary.Value
def scalar_value(tag: str, value: float) -> bytes:
    """Summary.Value {tag, simple_value} (float32, as tf.summary.scalar stores it)."""
    return _bytes(1, tag.encode()) + _field(2, 5) + struct.pack("<f", float(value))


def encode_wav(clip: np.ndarray, sample_rate: int) -> bytes:
    """[frames, channels] float samples -> 16-bit PCM wav, TF's EncodeAudioAsS16LEWav: round(x * 32768) clamped to int16."""
    pcm = np.clip(np.round(np.asarray(clip, np.float32) * 32768.0), -32768, 32767).astype("<i2")
    buf = io.BytesIO()
    with wave.open(buf, "wb") as w:
        w.setnchannels(pcm.shape[1])
        w.setsampwidth(2)
        w.setframerate(int(sample_rate))
        w.writeframes(pcm.tobytes())
    return buf.getvalue()


def audio_values(tag: str, clips: np.ndarray, sample_rate: int, max_outputs: int) -> List[bytes]:
    """tf.summary.audio(tag, clips [n, frames(, channels)], sample_rate, max_outputs): one Summary.Value per clip of the first
    max_outputs, tagged `<tag>/audio` when max_outputs is 1 and `<tag>/audio/<i>` otherwise (AudioSummaryV2)."""
    clips = np.asarray(clips, np.float32)
    if clips.ndim == 2:
        clips = clips[..., None]
    out = []
    for i, clip in enumerate(clips[:max_outputs]):
        audio = (_field(1, 5) + struct.pack("<f", float(sample_rate)) + _field(2, 0) + _varint(clip.shape[1])
                 + _field(3, 0) + _varint(clip.shape[0]) + _bytes(4, encode_wav(clip, sample_rate)) + _bytes(5, b"audio/wav"))
        name = f"{tag}/audio" if max_outputs == 1 else f"{tag}/audio/{i}"
        out.append(_bytes(1, name.encode()) + _bytes(6, audio))
    return out


def text_value(tag: str, rows: Sequence[Sequence[str]]) -> bytes:
    """tf.summary.text(tag, tf.convert_to_tensor(rows)): a DT_STRING tensor of shape [len(rows), len(rows[0])] with
    SummaryMetadata.plugin_data.plugin_name = "text"."""
    shape = (len(rows), len(rows[0]) if rows else 0)
    dims = b"".join(_bytes(2, _field(1, 0) + _varint(d)) for d in shape)
    tensor = _field(1, 0) + _varint(_DT_STRING) + _bytes(2, dims) + b"".join(_bytes(8, str(s).encode()) for r in rows for s in r)
    metadata = _bytes(1, _bytes(1, b"text"))
    return _bytes(1, tag.encode()) + _bytes(9, metadata) + _bytes(8, tensor)


# ------------------------------------------------------------------------------------------------ writer
class EventWriter:
    """tf.summary.FileWriter's file: created in `directory` (made if missing) with its file_version event; add() appends one
    Event with a Summary of the given values at `step`.  Records are buffered until flush() or close()."""

    def __init__(self, directory):
        self.directory = Path(directory)
        self.directory.mkdir(parents=True, exist_ok=True)
        name = f"events.out.tfevents.{int(time.time()):010d}.{socket.gethostname()}"
        path, n = self.directory / name, 0
        while path.exists():                  # another writer in the same directory within the same second
            n += 1
            path = self.directory / f"{name}.{n}"
        self.path = path
        self._f = open(path, "wb")
        self._event(_bytes(3, b"brain.Event:2"))
        self.flush()

    def _event(self, fields: bytes, step: int = 0):
        head = _field(1, 1) + struct.pack("<d", time.time())
        if step:
            head += _field(2, 0) + _varint(int(step))
        self._f.write(_record(head + fields))

    def add(self, step: int, values: Sequence[bytes]):
        if values:
            self._event(_bytes(5, b"".join(_bytes(1, v) for v in values)), step)

    def flush(self):
        self._f.flush()

    def close(self):
        if not self._f.closed:
            self._f.close()


# ------------------------------------------------------------------------------------------------ reader
def read_records(path) -> Iterator[bytes]:
    """The payloads of a TFRecord file; a length or payload whose masked CRC32C does not match raises ValueError."""
    data = Path(path).read_bytes()
    pos = 0
    while pos < len(data):
        head = data[pos:pos + 8]
        (n,) = struct.unpack("<Q", head)
        (c,) = struct.unpack("<I", data[pos + 8:pos + 12])
        if unmask_crc(c) != crc32c(head):
            raise ValueError(f"{path}: bad length CRC at offset {pos}")
        payload = data[pos + 12:pos + 12 + n]
        (c,) = struct.unpack("<I", data[pos + 12 + n:pos + 16 + n])
        if len(payload) != n or unmask_crc(c) != crc32c(payload):
            raise ValueError(f"{path}: bad payload CRC at offset {pos}")
        yield payload
        pos += 16 + n


def _decode_value(buf: bytes) -> Tuple[str, Dict[str, object]]:
    tag, val = "", {}
    for num, _, v in _decode_fields(buf):
        if num == 1:
            tag = v.decode()
        elif num == 2:
            val["simple_value"] = struct.unpack("<f", v)[0]
        elif num == 6:
            a = {1: "sample_rate", 2: "num_channels", 3: "length_frames", 4: "encoded_audio_string", 5: "content_type"}
            val["audio"] = {a[n]: (struct.unpack("<f", x)[0] if n == 1 else x) for n, _, x in _decode_fields(v)}
        elif num == 9:
            plugin = dict((n, x) for n, _, x in _decode_fields(v)).get(1, b"")
            val["plugin_name"] = dict((n, x) for n, _, x in _decode_fields(plugin)).get(1, b"").decode()
        elif num == 8:
            f = _decode_fields(v)
            shape = next((x for n, _, x in f if n == 2), b"")
            dims = [dict((k, x) for k, _, x in _decode_fields(d)).get(1, 0) for n, _, d in _decode_fields(shape) if n == 2]
            val["tensor"] = np.array([x.decode() for n, _, x in f if n == 8], dtype=object).reshape(dims)
    return tag, val


def read_events(path) -> List[Dict[str, object]]:
    """The Events of an event file as dicts: wall_time, step, and file_version or summary {tag: value dict}."""
    out = []
    for payload in read_records(path):
        ev: Dict[str, object] = {"step": 0}
        for num, _, v in _decode_fields(payload):
            if num == 1:
                ev["wall_time"] = struct.unpack("<d", v)[0]
            elif num == 2:
                ev["step"] = v
            elif num == 3:
                ev["file_version"] = v.decode()
            elif num == 5:
                ev["summary"] = dict(_decode_value(x) for n, _, x in _decode_fields(v) if n == 1)
        out.append(ev)
    return out


def decode_wav(data: bytes) -> Tuple[np.ndarray, int]:
    """(int16 samples [frames, channels], sample rate) of a PCM16 wav."""
    with wave.open(io.BytesIO(data), "rb") as w:
        pcm = np.frombuffer(w.readframes(w.getnframes()), "<i2").reshape(-1, w.getnchannels())
        return pcm, w.getframerate()
