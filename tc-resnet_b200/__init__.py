"""tc-resnet_b200 — H100-native hot path of hyperconnect/TC-ResNet (import name: ``tcresnet_b200``).

MFCC front-end + TCResNet8/14 forward / backward / SGD-momentum as hand-written sm_90a CUDA behind a
C ABI (include/tcr_b200.h), with the reference's Python surface (factory/, datasets/, helper/,
train_audio.py, evaluate_audio.py) on top.  PyTorch tensors are only the buffer carrier.
"""
from ._lib import TcrError, LIB_PATH  # noqa: F401

__all__ = ["TcrError", "LIB_PATH"]
