"""TensorFlow V2 checkpoint ("tensor bundle") reader / writer in pure Python + NumPy — no TensorFlow needed.

The reference saves its variables with tf.train.Saver (helper/trainer.py:83-86, :406-414) and restores them by name through
pywrap_tensorflow.NewCheckpointReader (common/model_loader.py:87-165); the evaluator finds checkpoints through
tf.train.latest_checkpoint / checkpoints_iterator (common/tf_utils.py:65-67, :219-247).  Saver's on-disk format (TF r1.13,
tensorflow/core/util/tensor_bundle) is

    <prefix>.index                   an immutable sorted string table (the LevelDB table format of tensorflow/core/lib/io):
                                     key ""   -> BundleHeaderProto {num_shards, endianness, version}
                                     key name -> BundleEntryProto {dtype, shape, shard_id, offset, size, crc32c}
    <prefix>.data-00000-of-00001     the tensors' raw little-endian bytes, back to back, in key order
    checkpoint                       CheckpointState text proto: model_checkpoint_path / all_model_checkpoint_paths

Written here from the format's published layout (no reference vectors exist in this container; "parity unpinned" for this
file too): blocks with prefix-compressed keys and restart points, per-block trailer (compression byte 0 + masked CRC32C),
index block of BlockHandles, 48-byte footer with the table magic 0xdb4775248b80fb57; protos are hand-encoded varints.
"""
from __future__ import annotations

import functools
import os
import struct
from pathlib import Path
from typing import Dict, List, Optional, Tuple

import numpy as np

_TABLE_MAGIC = 0xDB4775248B80FB57
_BLOCK_SIZE = 4096            # table::Options::block_size used by BundleWriter
_RESTART_INTERVAL = 16
_MASK_DELTA = 0xA282EAD8

# DataType enum values of tensorflow/core/framework/types.proto
_DT = {np.dtype("float32"): 1, np.dtype("float64"): 2, np.dtype("int32"): 3, np.dtype("uint8"): 4, np.dtype("int16"): 5,
       np.dtype("int8"): 6, np.dtype("int64"): 9, np.dtype("bool"): 10}
_DT_INV = {v: k for k, v in _DT.items()}


# ------------------------------------------------------------------------------------------------ CRC32C (Castagnoli)
def _make_table():
    poly = 0x82F63B78
    tab = np.zeros(256, np.uint32)
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ poly if c & 1 else c >> 1
        tab[i] = c
    return tab


_CRC_TABLE = _make_table()
_CRC_LIST = [int(x) for x in _CRC_TABLE]
_CHUNK = 32                   # bytes per chunk of the chunk-parallel path


def _shift(tables: np.ndarray, regs: np.ndarray) -> np.ndarray:
    return tables[0][regs & 0xFF] ^ tables[1][(regs >> 8) & 0xFF] ^ tables[2][(regs >> 16) & 0xFF] ^ tables[3][regs >> 24]


@functools.lru_cache(maxsize=None)
def _zeros_tables(n: int) -> np.ndarray:
    """The CRC register after n zero bytes (n = _CHUNK * 2^k), as lookup tables [4, 256] on the bytes of the starting register
    (the map is linear over GF(2)); 2n is n applied twice."""
    if n > _CHUNK:
        half = _zeros_tables(n // 2)
        return _shift(half, half)
    regs = (np.arange(256, dtype=np.uint32)[None, :] << (8 * np.arange(4, dtype=np.uint32))[:, None]).ravel()
    for _ in range(n):
        regs = _CRC_TABLE[regs & 0xFF] ^ (regs >> 8)
    return regs.reshape(4, 256)


def crc32c(data: bytes, crc: int = 0) -> int:
    c = crc ^ 0xFFFFFFFF
    n = len(data) // _CHUNK
    if n >= 64:               # large inputs (audio summaries): every chunk's register in one NumPy pass, then folded pairwise
        levels = (n - 1).bit_length()
        regs = np.zeros(1 << levels, np.uint32)
        first = (1 << levels) - n                            # leading all-zero registers leave the result unchanged
        regs[first] = c
        cols = np.frombuffer(data, np.uint8, n * _CHUNK).reshape(n, _CHUNK).T
        for col in cols:
            regs[first:] = _CRC_TABLE[(regs[first:] ^ col) & 0xFF] ^ (regs[first:] >> 8)
        size = _CHUNK
        while regs.size > 1:
            regs = _shift(_zeros_tables(size), regs[0::2]) ^ regs[1::2]
            size *= 2
        c = int(regs[0])
        data = data[n * _CHUNK:]
    tab = _CRC_LIST
    for b in data:
        c = tab[(c ^ b) & 0xFF] ^ (c >> 8)
    return c ^ 0xFFFFFFFF


def mask_crc(crc: int) -> int:
    return (((crc >> 15) | (crc << 17)) + _MASK_DELTA) & 0xFFFFFFFF


def unmask_crc(masked: int) -> int:
    rot = (masked - _MASK_DELTA) & 0xFFFFFFFF
    return ((rot >> 17) | (rot << 15)) & 0xFFFFFFFF


# ------------------------------------------------------------------------------------------------ varints / protos
def _varint(n: int) -> bytes:
    if n < 0:
        n += 1 << 64
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        if n:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _read_varint(buf: bytes, pos: int) -> Tuple[int, int]:
    shift = result = 0
    while True:
        b = buf[pos]
        pos += 1
        result |= (b & 0x7F) << shift
        if not b & 0x80:
            return result, pos
        shift += 7


def _field(num: int, wire: int) -> bytes:
    return _varint((num << 3) | wire)


def _encode_header() -> bytes:
    version = _field(1, 0) + _varint(1)                               # VersionDef.producer = 1
    return _field(1, 0) + _varint(1) + _field(3, 2) + _varint(len(version)) + version   # num_shards = 1, (endianness LITTLE = 0 omitted)


def _encode_entry(dtype: int, shape: Tuple[int, ...], offset: int, size: int, crc_masked: int) -> bytes:
    dims = b""
    for d in shape:
        dim = _field(1, 0) + _varint(int(d))
        dims += _field(2, 2) + _varint(len(dim)) + dim
    out = _field(1, 0) + _varint(dtype)
    out += _field(2, 2) + _varint(len(dims)) + dims                   # TensorShapeProto (empty for a scalar)
    if offset:
        out += _field(4, 0) + _varint(offset)                          # shard_id = 0 omitted (proto3 default)
    out += _field(5, 0) + _varint(size)
    out += _field(6, 5) + struct.pack("<I", crc_masked)
    return out


def _decode_fields(buf: bytes) -> List[Tuple[int, int, object]]:
    pos, out = 0, []
    while pos < len(buf):
        key, pos = _read_varint(buf, pos)
        num, wire = key >> 3, key & 7
        if wire == 0:
            v, pos = _read_varint(buf, pos)
        elif wire == 1:
            v = buf[pos:pos + 8]
            pos += 8
        elif wire == 2:
            n, pos = _read_varint(buf, pos)
            v = buf[pos:pos + n]
            pos += n
        elif wire == 5:
            v = buf[pos:pos + 4]
            pos += 4
        else:
            raise ValueError(f"unsupported wire type {wire}")
        out.append((num, wire, v))
    return out


def _decode_entry(buf: bytes) -> dict:
    e = dict(dtype=0, shape=(), shard_id=0, offset=0, size=0, crc32c=None, sliced=False)
    for num, _, v in _decode_fields(buf):
        if num == 1:
            e["dtype"] = v
        elif num == 2:
            dims = []
            for n2, _, v2 in _decode_fields(v):
                if n2 == 2:
                    size = 0
                    for n3, _, v3 in _decode_fields(v2):
                        if n3 == 1:
                            size = v3 - (1 << 64) if v3 >= 1 << 63 else v3
                    dims.append(size)
            e["shape"] = tuple(dims)
        elif num == 3:
            e["shard_id"] = v
        elif num == 4:
            e["offset"] = v
        elif num == 5:
            e["size"] = v
        elif num == 6:
            e["crc32c"] = struct.unpack("<I", v)[0]
        elif num == 7:
            e["sliced"] = True
    return e


# ------------------------------------------------------------------------------------------------ table blocks
class _BlockBuilder:
    def __init__(self):
        self.buf = bytearray()
        self.restarts = [0]
        self.counter = 0
        self.last_key = b""

    def add(self, key: bytes, value: bytes):
        shared = 0
        if self.counter < _RESTART_INTERVAL:
            m = min(len(self.last_key), len(key))
            while shared < m and self.last_key[shared] == key[shared]:
                shared += 1
        else:
            self.restarts.append(len(self.buf))
            self.counter = 0
        self.buf += _varint(shared) + _varint(len(key) - shared) + _varint(len(value)) + key[shared:] + value
        self.last_key = key
        self.counter += 1

    def size(self) -> int:
        return len(self.buf) + 4 * len(self.restarts) + 4

    def empty(self) -> bool:
        return not self.buf

    def finish(self) -> bytes:
        return bytes(self.buf) + b"".join(struct.pack("<I", r) for r in self.restarts) + struct.pack("<I", len(self.restarts))


def _write_block(f, contents: bytes) -> Tuple[int, int]:
    """Appends block + trailer (type 0 = uncompressed, masked crc32c over contents + type); returns its BlockHandle."""
    offset = f.tell()
    trailer_type = b"\x00"
    f.write(contents)
    f.write(trailer_type + struct.pack("<I", mask_crc(crc32c(contents + trailer_type))))
    return offset, len(contents)


def _parse_block(block: bytes) -> List[Tuple[bytes, bytes]]:
    n_restarts = struct.unpack("<I", block[-4:])[0]
    end = len(block) - 4 - 4 * n_restarts
    pos, key, out = 0, b"", []
    while pos < end:
        shared, pos = _read_varint(block, pos)
        non_shared, pos = _read_varint(block, pos)
        vlen, pos = _read_varint(block, pos)
        key = key[:shared] + block[pos:pos + non_shared]
        pos += non_shared
        out.append((key, block[pos:pos + vlen]))
        pos += vlen
    return out


def _read_block(buf: bytes, offset: int, size: int, verify: bool = True) -> bytes:
    contents, trailer = buf[offset:offset + size], buf[offset + size:offset + size + 5]
    if trailer[0] != 0:
        raise ValueError("compressed table blocks are not supported (tf.train.Saver writes uncompressed index files)")
    if verify and unmask_crc(struct.unpack("<I", trailer[1:5])[0]) != crc32c(contents + trailer[:1]):
        raise ValueError("index block checksum mismatch")
    return contents


# ------------------------------------------------------------------------------------------------ public API
def write_bundle(prefix, tensors: Dict[str, np.ndarray]) -> str:
    """Writes <prefix>.index and <prefix>.data-00000-of-00001 (atomically: temporary names, then rename)."""
    prefix = str(prefix)
    Path(prefix).parent.mkdir(parents=True, exist_ok=True)
    data_path, index_path = prefix + ".data-00000-of-00001", prefix + ".index"
    # temporary names are dot-files: no checkpoint glob (latest_checkpoint, pruning of old checkpoints by another process) sees them
    parent, stem = Path(prefix).parent, Path(prefix).name
    data_tmp, index_tmp = str(parent / f".{stem}.data.{os.getpid()}.tmp"), str(parent / f".{stem}.index.{os.getpid()}.tmp")
    entries = []
    with open(data_tmp, "wb") as f:
        for name in sorted(tensors, key=lambda s: s.encode()):
            a = np.asarray(tensors[name])
            if a.dtype not in _DT:
                raise TypeError(f"{name}: dtype {a.dtype} is not supported")
            raw = np.ascontiguousarray(a.astype(a.dtype.newbyteorder("<"), copy=False)).tobytes()
            entries.append((name.encode(), _encode_entry(_DT[a.dtype], a.shape, f.tell(), len(raw), mask_crc(crc32c(raw)))))
            f.write(raw)
    with open(index_tmp, "wb") as f:
        index_entries, blk = [], _BlockBuilder()

        def flush():
            nonlocal blk
            if blk.empty():
                return
            off, size = _write_block(f, blk.finish())
            index_entries.append((blk.last_key, _varint(off) + _varint(size)))
            blk = _BlockBuilder()

        for key, value in [(b"", _encode_header())] + entries:
            blk.add(key, value)
            if blk.size() >= _BLOCK_SIZE:
                flush()
        flush()
        meta = _write_block(f, _BlockBuilder().finish())               # empty metaindex block
        ib = _BlockBuilder()
        for key, handle in index_entries:
            ib.add(key, handle)
        index = _write_block(f, ib.finish())
        footer = _varint(meta[0]) + _varint(meta[1]) + _varint(index[0]) + _varint(index[1])
        f.write(footer + b"\x00" * (40 - len(footer)) + struct.pack("<Q", _TABLE_MAGIC))
    os.replace(data_tmp, data_path)
    os.replace(index_tmp, index_path)                          # the index appears last: a visible index means a complete bundle
    return prefix


class BundleReader:
    """NewCheckpointReader's surface: has_tensor / get_tensor / get_variable_to_shape_map (common/model_loader.py:111-123)."""

    def __init__(self, prefix, verify: bool = True):
        self.prefix, self.verify = str(prefix), verify
        buf = Path(self.prefix + ".index").read_bytes()
        if len(buf) < 48 or struct.unpack("<Q", buf[-8:])[0] != _TABLE_MAGIC:
            raise ValueError(f"{self.prefix}.index is not a tensor-bundle index (bad magic)")
        footer = buf[-48:-8]
        _, pos = _read_varint(footer, 0)
        _, pos = _read_varint(footer, pos)
        ioff, pos = _read_varint(footer, pos)
        isize, pos = _read_varint(footer, pos)
        self.entries: Dict[str, dict] = {}
        self.header = None
        for _, handle in _parse_block(_read_block(buf, ioff, isize, verify)):
            off, p = _read_varint(handle, 0)
            size, _ = _read_varint(handle, p)
            for key, value in _parse_block(_read_block(buf, off, size, verify)):
                if key == b"":
                    self.header = _decode_fields(value)
                else:
                    self.entries[key.decode()] = _decode_entry(value)
        if self.header is None:
            raise ValueError("bundle header entry is missing")
        for num, _, v in self.header:
            if num == 2 and v != 0:
                raise ValueError("big-endian bundles are not supported")
        self._data: Dict[int, np.memmap] = {}
        self.num_shards = next((v for num, _, v in self.header if num == 1), 1)

    def has_tensor(self, name: str) -> bool:
        return name in self.entries

    def get_variable_to_shape_map(self) -> Dict[str, Tuple[int, ...]]:
        return {k: e["shape"] for k, e in self.entries.items()}

    def get_tensor(self, name: str) -> np.ndarray:
        e = self.entries[name]
        if e["sliced"]:
            raise NotImplementedError(f"{name}: partitioned (sliced) variables are not supported")
        if e["dtype"] not in _DT_INV:
            raise NotImplementedError(f"{name}: DataType {e['dtype']} is not supported")
        shard = e["shard_id"]
        if shard not in self._data:
            self._data[shard] = np.memmap(f"{self.prefix}.data-{shard:05d}-of-{self.num_shards:05d}", dtype=np.uint8, mode="r")
        raw = bytes(self._data[shard][e["offset"]:e["offset"] + e["size"]])
        if self.verify and e["crc32c"] is not None and unmask_crc(e["crc32c"]) != crc32c(raw):
            raise ValueError(f"{name}: tensor checksum mismatch")
        dt = _DT_INV[e["dtype"]]
        return np.frombuffer(raw, dtype=dt.newbyteorder("<")).astype(dt).reshape(e["shape"])

    def read_all(self) -> Dict[str, np.ndarray]:
        return {k: self.get_tensor(k) for k in self.entries}


def write_checkpoint_state(directory, latest: str, all_paths: Optional[List[str]] = None):
    """The `checkpoint` text file tf.train.latest_checkpoint reads (CheckpointState, paths relative to the directory)."""
    lines = [f'model_checkpoint_path: "{latest}"'] + [f'all_model_checkpoint_paths: "{p}"' for p in (all_paths or [latest])]
    tmp = Path(directory) / f".checkpoint.tmp{os.getpid()}"
    tmp.write_text("\n".join(lines) + "\n")
    os.replace(tmp, Path(directory) / "checkpoint")


def read_checkpoint_state(directory) -> Optional[str]:
    p = Path(directory) / "checkpoint"
    if not p.exists():
        return None
    for line in p.read_text().splitlines():
        if line.startswith("model_checkpoint_path:"):
            return line.split(":", 1)[1].strip().strip('"')
    return None
