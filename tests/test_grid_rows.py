"""Batches past CUDA's 65,535-row grid bound.  The front-end, the input stage (tcr_augment_pcm16, tcr_dataset_batch), the FMA DS-CNN
block and the listener's stage and reset kernels take one utterance or stream per blockIdx.y; the library launches them in slices
of at most 65,535 rows (kMaxGridRows), so a handle of any max_batch runs every batch it accepts.  At n = 65,537 the rows on both
sides of the slice boundary, and the last row, are checked against the same rows computed at a small batch or against the
oracles.  The emulator refuses a grid CUDA would refuse (tests/emu/cuda_emu.cpp), so the front-end and input-stage cases run
there too; the network-sized cases run with -m gpu.  Tiny geometries keep the device memory in the low hundreds of MB."""
import ctypes as C

import numpy as np
import pytest

import dataset_oracle as D
from oracle import augment_oracle as A
from oracle import dscnn_oracle as DS
from oracle import tcr_oracle as O
from parity_cases import TOL_LOGITS, perturbed_variables, reference_features
from tcr_harness import Engine, NumpyBackend, rel_err
from test_geometry import FRONT_END, engine_cfg, ref_args

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L

N = 65537
# the first rows of the first slice, the last rows of the first slice and the two rows of the second
EDGE = np.r_[0:8, 65528:N]
G = dict(FRONT_END["fft128-32-12"], clip=128)            # FFT 128, 12 MFCCs from 32 mel bins, clip = window: T = 1
TINY = engine_cfg(G)


@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


def clips(n, samples=128, seed=0):
    return np.random.default_rng(seed).uniform(-1.0, 1.0, (n, samples)).astype(np.float32)


def check_front_end(backend, every_row):
    wav = clips(N)
    eng = Engine(backend, max_batch=N, **TINY)
    small = Engine(backend, max_batch=512, **TINY)
    try:
        got = eng.mfcc(wav)
        assert got.shape == (N, 1, 12) and np.isfinite(got).all()          # every row written (outputs start as NaN)
        assert np.array_equal(got[EDGE], small.mfcc(wav[EDGE]))
        if every_row:
            for i in range(0, N, 512):
                assert np.array_equal(got[i:i + 512], small.mfcc(wav[i:i + 512])), i
    finally:
        eng.close()
        small.close()


def test_emulated_front_end_past_the_grid_bound(emu, monkeypatch):
    monkeypatch.setenv("TCR_MFCC_PAIR", "0")
    check_front_end(emu, every_row=False)


@pytest.mark.gpu
def test_front_end_past_the_grid_bound(cuda, monkeypatch):
    monkeypatch.setenv("TCR_MFCC_PAIR", "0")
    check_front_end(cuda, every_row=True)


def check_augment(backend):
    rng = np.random.RandomState(3)
    pcm = rng.randint(-32768, 32768, size=(N, 160)).astype(np.int16)
    bg_lengths = [128, 300, 1000]
    background = rng.uniform(-1, 1, size=sum(bg_lengths)).astype(np.float32)
    draws = A.random_clips(rng, N, 128, 160, bg_lengths)
    eng = Engine(backend, max_batch=N, **TINY)
    try:
        got = eng.augment(pcm, draws, background)
        assert np.isfinite(got).all()
        assert np.array_equal(got[EDGE], A.augment(pcm[EDGE], draws[EDGE], background, 128))
    finally:
        eng.close()


def test_emulated_augment_past_the_grid_bound(emu):
    check_augment(emu)


@pytest.mark.gpu
def test_augment_past_the_grid_bound(cuda):
    check_augment(cuda)


def check_dataset_batch(backend):
    from test_device_dataset import _desc, _padded_background, _synthetic_bank
    rng = np.random.RandomState(5)
    bank, table = _synthetic_bank(rng, 40)
    background, bg_lengths = _padded_background([rng.uniform(-1, 1, k).astype(np.float32) for k in (400, 1200, 7000)], clip=128)
    order = rng.randint(0, 40, N + 100).astype(np.int32)
    position, epoch, seed = 77, 3, 5
    eng = Engine(backend, max_batch=N, **TINY)
    try:
        desc, keep = _desc(backend, bank, table, order, background, bg_lengths, True, True, True, 0.8, 1.0)
        b = eng.b
        wav, hot = b.empty(N, 128), b.empty(N, 12)
        L.check(eng.lib, eng.lib.tcr_dataset_batch(eng.h, C.byref(desc), position, epoch, seed, N, b.ptr(wav), b.ptr(hot), b.stream),
                "tcr_dataset_batch")
        b.sync()
        wav, hot = b.download(wav), b.download(hot)
        assert np.isfinite(wav).all() and np.isfinite(hot).all()
        for lo, hi in ((0, 8), (65528, N)):
            ref, ref_hot = D.batch(bank, table, order, position + lo, hi - lo, seed, epoch, 128, 12, background, bg_lengths,
                                   background_frequency=0.8, background_max_volume=1.0)
            assert np.array_equal(wav[lo:hi], ref), (lo, np.abs(wav[lo:hi] - ref).max())
            assert np.array_equal(hot[lo:hi], ref_hot), lo
    finally:
        eng.close()


def test_emulated_dataset_batch_past_the_grid_bound(emu):
    check_dataset_batch(emu)


@pytest.mark.gpu
def test_dataset_batch_past_the_grid_bound(cuda):
    check_dataset_batch(cuda)


@pytest.mark.gpu
def test_forward_past_the_grid_bound(cuda):
    """tcr_forward at n = 65,537 from wav (the front-end runs in two slices): edge rows against the fp64 oracle."""
    spec = O.build_spec("TCResNet8", 1.0, 1, 12)
    params, moving = perturbed_variables(spec, 0)
    wav = clips(N, seed=1)
    eng = Engine(cuda, max_batch=N, dropout_keep_prob=1.0, **TINY)
    try:
        got = eng.forward(wav, O.flatten_vars(spec, params), O.flatten_moving(spec, moving))["logits"]
        assert np.isfinite(got).all()
        ref, _ = O.forward(spec, params, moving, reference_features(wav[EDGE].astype(np.float64), *ref_args(G)), False)
        err = rel_err(got[EDGE], ref)
        print("tcr_forward n=65537 edge rows vs fp64:", err)
        assert err <= TOL_LOGITS, err
    finally:
        eng.close()


@pytest.mark.gpu
def test_dscnn_fma_blocks_past_the_grid_bound(cuda, monkeypatch):
    """DS-CNN-S on 1 x 10 features with the FMA kernels (TCR_DSCNN_TC=0): dscnn_dsblock takes one utterance per blockIdx.y."""
    from test_dscnn import DsNet
    monkeypatch.setenv("TCR_DSCNN_TC", "0")
    spec = DS.build_spec("S", 1, 10)
    p = DS.init_variables(spec, 0)
    net = DsNet(cuda, "S", 1, 10, N, p)
    try:
        feat = np.random.RandomState(2).randn(N, 1, 10).astype(np.float32)
        logits, probs = net.forward(feat)
        assert np.isfinite(logits).all() and np.isfinite(probs).all()
        err = rel_err(logits[EDGE], DS.forward(spec, p, feat[EDGE].astype(np.float64)))
        print("DS-CNN-S n=65537 edge rows vs fp64:", err)
        assert err <= TOL_LOGITS, err
    finally:
        net.close()


@pytest.mark.gpu
@pytest.mark.parametrize("frames", [1, 2, 3])
def test_listener_past_the_grid_bound(cuda, frames):
    """65,537 streams, one window per push: the stage kernel and, at T = 3, the reset kernel run in two slices; at T >= 2 the
    reset at create time runs the front-end over every stream.  All streams are reset halfway."""
    from test_listener_geometry import run_listener
    cfg = dict(TINY, clip_samples=128 + 64 * (frames - 1))
    T, hop = run_listener(cuda, cfg, N, 1, 1, resets=((2, -1),))
    assert (T, hop) == (frames, 1)
