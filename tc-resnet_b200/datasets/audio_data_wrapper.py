"""SingleLabelAudioDataWrapper with the reference's constructor, flags and attributes
(datasets/audio_data_wrapper.py:9-174): label discovery from `<dataset_path>/<split>/<label>/*.wav`, silent samples,
one-hot labels, `get_input_and_output_op()` -> (wavs, labels) handles, `setup_iterator()` to rewind.

`--dataset_path synthetic[:NUM]` is an addition for machines without the Speech Commands data: seeded
U(-1,1) clips and uniform labels over the 12 reference classes (SURVEY.md 8d)."""
from __future__ import annotations

import numpy as np

from .. import const
from ..runtime import Node, OutOfRangeError
from .augmentation_factory import get_audio_augmentation_fn, load_wav_file
from .data_wrapper_base import DataWrapperBase

GSC12 = [const.NULL_CLASS_LABEL, "down", "go", "left", "no", "off", "on", "right", "stop", "unknown", "up", "yes"]

_AUDIO_FLAGS = [("sample_rate", int, 16000), ("clip_duration_ms", int, 1000), ("window_size_ms", float, 30.0),
                ("window_stride_ms", float, 10.0), ("lower_edge_hertz", float, 80.0), ("upper_edge_hertz", float, 7600.0),
                ("num_mel_bins", int, 64), ("num_mfccs", int, 40), ("input_file", str, None), ("description_file", str, None),
                ("num_partitions", int, 2), ("background_max_volume", float, 0.1), ("background_frequency", float, 0.8),
                ("num_silent", int, -1)]


class AudioDataWrapper(DataWrapperBase):
    def __init__(self, args, session, dataset_split_name, is_training, name: str = "AudioDataWrapper"):
        super().__init__(args, dataset_split_name, is_training, name)
        self.session = session
        self.desired_samples = int(args.sample_rate * args.clip_duration_ms / 1000)
        self.rng = np.random.RandomState(1234)          # shuffle order: the SAME on every rank (ranks take disjoint slices of it)
        # data-parallel shard of this process (train_audio.py --data_parallel under torchrun): rank r takes rows
        # [r*B, (r+1)*B) of every global window of world*B samples; augmentation draws are per rank
        self.rank, self.world = 0, 1
        if getattr(args, "data_parallel", False):
            import torch.distributed as dist
            if dist.is_available() and dist.is_initialized():
                self.rank, self.world = dist.get_rank(), dist.get_world_size()
        self.aug_rng = np.random.RandomState(1234 + 7919 * self.rank)
        self.draw_seed = 1234                           # --device_dataset: draws keyed by global position, the same on every rank
        self.setup()
        self.placeholders = (Node("filenames"), Node("labels_index"))
        self.setup_iterator(session, self.placeholders, self.data)

    @property
    def num_samples(self):
        return self._num_samples

    def setup_iterator(self, session, placeholders, variables):
        assert len(placeholders) == len(variables), "Length of placeholders and variables differ!"
        self._cursor = 0
        self._order = np.arange(self._num_samples)
        if self.shuffle:
            self.rng.shuffle(self._order)
        self._epoch = getattr(self, "_epoch", -1) + 1     # key of the device path's draws; a new order goes to the device
        self._order_changed = True

    def get_input_and_output_op(self):
        return (Node("audio_original", [None, self.desired_samples, 1], self),
                Node("labels", [None, self.num_labels], self))

    def _next_position(self):
        """Position of this rank's next batch in `_order`: advances the shared cursor, reshuffles when the epoch ends."""
        n = self.batch_size
        window = n * self.world                       # one global batch; every rank advances the shared cursor by it
        if self._cursor + window > self._num_samples:
            if not self.is_training:
                raise OutOfRangeError("Finished looping dataset.")
            self._cursor = 0
            if self.shuffle:
                self.rng.shuffle(self._order)
            self._epoch += 1
            self._order_changed = True
        lo = self._cursor + self.rank * n
        self._cursor += window
        return lo

    def _take_indices(self):
        lo = self._next_position()
        return self._order[lo:lo + self.batch_size]

    def attach_device(self, engine):
        """--device_dataset: moves the decoded split to `engine`'s device (DeviceDataset); called once the model's engine exists."""
        from .device_input_stage import DeviceDataset
        a = self.args
        self.device_data = DeviceDataset(
            engine, self._bank, self._bank_table, self.background_data,
            shift=a.augmentation_method == "anchored_slice_or_pad_with_shift",
            mix=a.augmentation_method not in ("no_augmentation", "no_augmentation_audio"),
            is_training=self.is_training, background_frequency=a.background_frequency, background_max_volume=a.background_max_volume)
        self._bank = self._bank_table = None          # the host copy is not needed any more
        return self.device_data

    def next_device_rows(self):
        """--device_dataset: (position, epoch) of this rank's next batch in the resident order, which is the order the host path
        takes its indices from; the epoch's order is uploaded when it changed."""
        lo = self._next_position()
        if self._order_changed:
            self.device_data.upload_order(self._order)
            self._order_changed = False
        return lo, self._epoch

    @staticmethod
    def add_arguments(parser):
        g = parser.add_argument_group("(AudioDataWrapper) Arguments for Audio DataWrapper")
        for name, typ, default in _AUDIO_FLAGS:
            g.add_argument(f"--{name}", type=typ, default=default)


class SingleLabelAudioDataWrapper(AudioDataWrapper):
    def setup(self):
        a = self.args
        self.synthetic = str(a.dataset_path).startswith("synthetic")
        self.device_data = None
        if self.synthetic and getattr(a, "device_dataset", False):
            raise ValueError("--device_dataset reads a dataset from disk; `synthetic:` clips are generated on the host")
        if self.synthetic:
            spec = str(a.dataset_path).split(":")
            self._num_samples = int(spec[1]) if len(spec) > 1 else 4096
            self.label_names = GSC12[:a.num_classes] if a.num_classes and a.num_classes <= 12 else GSC12
            self.num_labels = len(self.label_names)
            self.labels = list(np.random.RandomState(4321).randint(0, self.num_labels, size=self._num_samples))
            self.filenames = [f"synthetic://{i}" for i in range(self._num_samples)]
            self.background_data = []
        else:
            paths = self.get_all_dataset_paths()
            self.label_names, self.num_labels = self.get_label_names(paths)
            assert const.NULL_CLASS_LABEL in self.label_names
            self.filenames, self.labels = self.get_filenames_labels(paths)
            self.background_data = []
            for p in paths:
                noise = p / const.BACKGROUND_NOISE_DIR_NAME
                if noise.is_dir():
                    self.background_data += [load_wav_file(str(f), -1) for f in sorted(noise.glob("*.wav"))]
            num_silent = a.num_silent if a.num_silent >= 0 else len(self.filenames) // self.num_labels
            null_idx = self.label_names.index(const.NULL_CLASS_LABEL)
            self.filenames += [""] * num_silent          # "" marks a silent (all-zero) clip
            self.labels += [null_idx] * num_silent
            self._num_samples = len(self.filenames)
            self.augment = get_audio_augmentation_fn(a.augmentation_method if a.augmentation_method != "no_augmentation"
                                                     else "no_augmentation_audio")
            if getattr(a, "device_dataset", False):             # decoded once here, moved to the device by attach_device()
                from .device_input_stage import decode_clip_bank
                self._bank, self._bank_table = decode_clip_bank(self.filenames, self.labels, self.desired_samples,
                                                                getattr(a, "num_threads", 8))
        assert a.num_classes == self.num_labels, f"--num_classes {a.num_classes} != {self.num_labels} label directories"
        self.data = (self.filenames, self.labels)

    def _synthetic_wavs(self, idx):
        """Seeded U(-1,1) clips; clip i is always the same samples (a pool of up to 4096 distinct clips, generated once)."""
        pool = getattr(self, "_pool", None)
        if pool is None:
            rng = np.random.default_rng(1234)
            pool = self._pool = rng.uniform(-1.0, 1.0, (min(self._num_samples, 4096), self.desired_samples)).astype(np.float32)
        return pool[np.asarray(idx) % pool.shape[0]]

    def next_batch_pinned(self):
        """Training fast path for `synthetic:` data: pre-built batches in PINNED host memory (built once, cycled), so that a
        session.run(train_op) is one tcr_train_step_host call with no per-step host work; None for datasets read from disk
        (their decode / augment pipeline is the reference's tf.data stage, outside the hot path).  Advances the same cursor."""
        if not self.synthetic or not self.is_training:
            return None
        import torch
        idx = self._take_indices()
        key = int(self._cursor // max(self.batch_size * self.world, 1)) % 8
        cache = self.__dict__.setdefault("_pinned", {})
        if key not in cache:
            labels = np.zeros((len(idx), self.num_labels), np.float32)
            labels[np.arange(len(idx)), [self.labels[i] for i in idx]] = 1.0
            cache[key] = (torch.from_numpy(self._synthetic_wavs(idx)).pin_memory(), torch.from_numpy(labels).pin_memory())
        return cache[key]

    def next_batch(self):
        idx = self._take_indices()
        n = len(idx)
        labels = np.zeros((n, self.num_labels), np.float32)
        labels[np.arange(n), [self.labels[i] for i in idx]] = 1.0
        if self.synthetic:
            return self._synthetic_wavs(idx)[..., None], labels
        a = self.args
        wavs = np.stack([self.augment(self.filenames[i], self.desired_samples, self.aug_rng, self.background_data,
                                      self.is_training, a.background_frequency, a.background_max_volume) for i in idx])
        return wavs[..., None], labels
