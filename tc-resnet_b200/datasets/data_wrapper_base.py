"""Flag surface and bookkeeping of the reference's DataWrapperBase (datasets/data_wrapper_base.py:18-288).
The tf.data pipeline itself (list files -> shuffle -> map(decode+augment) -> batch -> repeat, :59-89) is host I/O
outside the hot path; subclasses implement `next_batch()` directly."""
from __future__ import annotations

import random
from abc import ABC, abstractmethod
from pathlib import Path

from .. import const
from ..common import utils
from .augmentation_factory import _available_augmentation_methods

_BOOL_FLAGS = [("has_sub_dataset", False), ("add_null_class", True), ("shuffle", True), ("cache_dataset", False),
               # decode the split once into device memory and build every batch there (datasets/device_input_stage.DeviceDataset);
               # opt-in: it holds the whole split in GPU memory and draws other augmentation random numbers than the host path
               ("device_dataset", False)]


class DataWrapperBase(ABC):
    def __init__(self, args, dataset_split_name: str, is_training: bool, name: str):
        self.name, self.args = name, args
        self.dataset_split_name, self.is_training = dataset_split_name, is_training
        self.shuffle = args.shuffle
        self.log = utils.get_logger(name)
        self.timer = utils.Timer(self.log)
        self.dataset_path = Path(args.dataset_path)
        self.dataset_path_with_split_name = self.dataset_path / dataset_split_name
        self.batch_size = args.batch_size

    @property
    @abstractmethod
    def num_samples(self):
        ...

    @abstractmethod
    def next_batch(self):
        """-> (wavs f32 [N, L, 1] in [-1,1], one-hot f32 [N, num_labels])"""

    def get_all_dataset_paths(self):
        if self.args.has_sub_dataset:
            return sorted(p for p in self.dataset_path_with_split_name.glob("*/") if p.is_dir())
        return [self.dataset_path_with_split_name]

    def get_label_names(self, dataset_paths):
        """__null__ (silence) = 0, then sorted directory names not starting with '_' (:114-145)."""
        per_path = []
        for p in dataset_paths:
            names = [const.NULL_CLASS_LABEL] if self.args.add_null_class else []
            names += [n for n in sorted(c.name for c in p.glob("*")) if not n.startswith("_")]
            per_path.append(tuple(names))
        assert len(set(per_path)) == 1, "Different labels for each sub-dataset directory"
        assert len(per_path[0]) > 0, f"There're no label directories in {dataset_paths}"
        return list(per_path[0]), len(per_path[0])

    def get_filenames_labels(self, dataset_paths):
        filenames, labels = [], []
        for idx, cls in enumerate(self.label_names):
            for p in dataset_paths:
                for f in sorted(p.joinpath(cls).glob("*")):
                    filenames.append(str(f))
                    labels.append(idx)
        assert filenames, f"no input files under {dataset_paths}"
        return filenames, labels

    @staticmethod
    def do_shuffle(*lists):
        packed = list(zip(*lists))
        random.shuffle(packed)
        return tuple(list(x) for x in zip(*packed))

    @staticmethod
    def add_arguments(parser):
        g = parser.add_argument_group("(DataWrapperBase) Common Arguments for all data wrapper.")
        g.add_argument("--dataset_path", required=True, type=str)
        g.add_argument("--dataset_split_name", required=True, type=str, nargs="*")
        for name, default in _BOOL_FLAGS:
            g.add_argument(f"--{name}", dest=name, action="store_true")
            g.add_argument(f"--no-{name}", dest=name, action="store_false")
            g.set_defaults(**{name: default})
        g.add_argument("--batch_size", default=32, type=utils.positive_int)
        g.add_argument("--cache_dataset_path", default=None, type=lambda p: Path(p))
        g.add_argument("--width", type=int, default=-1)
        g.add_argument("--height", type=int, default=-1)
        g.add_argument("--augmentation_method", type=str, required=True, choices=_available_augmentation_methods)
        g.add_argument("--num_threads", default=8, type=int)
        g.add_argument("--buffer_size", default=1000, type=int)
        g.add_argument("--prefetch_factor", default=100, type=int)
