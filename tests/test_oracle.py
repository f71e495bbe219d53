"""Self-checks of the CPU oracle (oracle/tcr_oracle.py).

The reference has no tests or golden vectors (parity unpinned, SURVEY.md 8c), so the oracle is
pinned by: analytic counts from the paper/SURVEY, scipy's DCT, an independent NumPy port of the
mel matrix that ships with `transformers`, finite differences in fp64 and an independent
PyTorch-autograd restatement of the same TF-1.13 semantics.
"""
import math

import numpy as np
import pytest
import scipy.fft
import torch
import torch.nn.functional as F

from oracle import tcr_oracle as O


@pytest.mark.parametrize("model,wm,t,params,flops", [
    ("TCResNet8", 1.0, 49, 65264, 1585344),
    ("TCResNet14", 1.5, 49, 303144, 6975936),
    ("TCResNet8", 1.0, 98, 65264, 3045312),
    ("TCResNet14", 1.5, 98, 303144, 13354560),
])
def test_counts_match_survey(model, wm, t, params, flops):
    spec = O.build_spec(model, wm, t)
    assert O.count_trainable(spec) == params
    assert O.forward_flops(spec) == flops


def test_same_padding_asymmetry():
    # stride-2 9x1 conv at even T pads (3,4); at odd T (4,4)  (SURVEY.md 7, hard part 6)
    assert O.same_padding(98, 9, 2) == (49, 3, 4)
    assert O.same_padding(49, 9, 2) == (25, 4, 4)
    assert O.same_padding(49, 1, 2) == (25, 0, 0)
    assert O.same_padding(98, 1, 2) == (49, 0, 0)
    assert O.same_padding(49, 3, 1) == (49, 1, 1)


def test_frames_and_fft_sizes():
    assert O.num_frames(16000, 640, 320) == 49 and O.next_pow2(640) == 1024
    assert O.num_frames(16000, 480, 160) == 98 and O.next_pow2(480) == 512


def test_dct_matches_scipy():
    x = np.random.RandomState(0).randn(5, 64)
    ref = scipy.fft.dct(x, type=2, norm=None, axis=-1)[:, :40] / math.sqrt(2 * 64)
    np.testing.assert_allclose(x @ O.dct2_matrix(64, 40), ref, rtol=1e-12, atol=1e-12)


def test_mel_matrix_structure_and_independent_port():
    for bins, nnz in ((513, 942), (257, 471)):
        w = O.linear_to_mel_weight_matrix(64, bins, 16000, 80.0, 7600.0)
        assert w.shape == (bins, 64)
        assert int((w > 0).sum()) == nnz
        assert int((w > 0).sum(axis=1).max()) <= 2          # banded: <= 2 mel bins per fft bin
        assert np.all(w[0] == 0)                             # DC bin zeroed
    # independent NumPy port of the same TF routine that ships with transformers
    try:
        from transformers.models.lasr.feature_extraction_lasr import linear_to_mel_weight_matrix as port
    except Exception:
        pytest.skip("transformers LASR feature extractor not importable")
    ref = port(num_mel_bins=64, num_spectrogram_bins=513, sample_rate=16000,
               lower_edge_hertz=80.0, upper_edge_hertz=7600.0, dtype=np.float64)
    np.testing.assert_allclose(O.linear_to_mel_weight_matrix(64, 513), ref, rtol=1e-9, atol=1e-12)


def test_stft_against_direct_dft():
    wav, _ = O.synthetic_batch(1)
    w, s = 640, 320
    spec = O.power_spectrogram(wav, w, s)
    frame = wav[0, 3 * s:3 * s + w].astype(np.float64) * O.hann_window_periodic(w)
    n = np.arange(w)
    for k in (0, 1, 17, 400, 512):
        x = np.sum(frame * np.exp(-2j * np.pi * k * n / 1024))
        assert abs(spec[0, 3, k] - abs(x) ** 2) <= 1e-9 * max(1.0, abs(x) ** 2)


@pytest.mark.parametrize("window,stride,clip", [(128, 64, 16000), (256, 128, 16000), (1600, 640, 16000), (240, 80, 8000)])
def test_stft_against_direct_dft_at_every_fft_length(window, stride, clip):
    """FFT 128, 256 and 2048 (and 256 from a 240-sample window): every bin of two frames, DC and Nyquist included."""
    wav, _ = O.synthetic_batch(2, num_samples=clip, adversarial=True)
    fft = O.next_pow2(window)
    spec = O.power_spectrogram(wav, window, stride)
    mag = O.power_spectrogram(wav, window, stride, magnitude_squared=False)
    t = O.num_frames(clip, window, stride)
    assert spec.shape == (2, t, fft // 2 + 1)
    n, k = np.arange(window), np.arange(fft // 2 + 1)
    basis = np.exp(-2j * np.pi * np.outer(n, k) / fft)
    for c, f in ((0, 0), (1, t // 2), (1, t - 1)):
        frame = wav[c, f * stride:f * stride + window].astype(np.float64) * O.hann_window_periodic(window)
        x = frame @ basis
        np.testing.assert_allclose(spec[c, f], np.abs(x) ** 2, rtol=1e-9, atol=1e-9)
        np.testing.assert_allclose(mag[c, f], np.abs(x), rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("bins,sample_rate,lower,upper,fft", [
    (32, 16000, 80.0, 7600.0, 128), (64, 16000, 80.0, 7600.0, 128), (40, 16000, 20.0, 8000.0, 256), (41, 16000, 80.0, 7600.0, 1024),
    (80, 16000, 80.0, 7600.0, 1024), (128, 16000, 20.0, 7600.0, 1024), (96, 16000, 80.0, 7600.0, 1024),
    (64, 16000, 80.0, 7600.0, 2048), (40, 8000, 80.0, 7600.0, 256)])
def test_mel_matrix_against_the_independent_port_at_every_geometry(bins, sample_rate, lower, upper, fft):
    try:
        from transformers.models.lasr.feature_extraction_lasr import linear_to_mel_weight_matrix as port
    except Exception:
        pytest.skip("transformers LASR feature extractor not importable")
    w = O.linear_to_mel_weight_matrix(bins, fft // 2 + 1, sample_rate, lower, upper)
    ref = port(num_mel_bins=bins, num_spectrogram_bins=fft // 2 + 1, sample_rate=sample_rate, lower_edge_hertz=lower,
               upper_edge_hertz=upper, dtype=np.float64)
    np.testing.assert_allclose(w, ref, rtol=1e-9, atol=1e-12)
    assert np.all(w[0] == 0) and int((w > 0).sum(axis=1).max()) <= 2


def test_bands_above_nyquist_and_between_bins_are_exactly_the_log_offset():
    """8 kHz with the default 7600 Hz upper edge: the bands above 4 kHz cover no FFT bin, so they are log(1e-6) for any input.
    FFT 128 at 64 bands: narrow low bands fall between two bins and are empty too."""
    wav, _ = O.synthetic_batch(3, num_samples=8000, adversarial=True)
    w = O.linear_to_mel_weight_matrix(40, 129, 8000, 80.0, 7600.0)
    empty = np.flatnonzero(w.sum(axis=0) == 0)
    assert list(empty) == list(range(32, 40))
    lm = O.log_mel_spectrogram(wav, 240, 80, num_mel_bins=40, sample_rate=8000)
    assert np.all(lm[..., empty] == math.log(1e-6)) and np.all(lm[1:, :, :32] > math.log(1e-6))
    wav, _ = O.synthetic_batch(3, adversarial=True)
    empty = np.flatnonzero(O.linear_to_mel_weight_matrix(64, 65, 16000, 80.0, 7600.0).sum(axis=0) == 0)
    assert list(empty) == [2, 3, 6, 9, 12, 15]
    lm = O.log_mel_spectrogram(wav, 128, 64)
    assert np.all(lm[..., empty] == math.log(1e-6))


@pytest.mark.parametrize("mel,mfccs", [(64, 12), (40, 20), (80, 32), (128, 64), (41, 40), (41, 12), (64, 64)])
def test_dct_matches_scipy_at_every_coefficient_count(mel, mfccs):
    x = np.random.RandomState(mel + mfccs).randn(5, mel)
    ref = scipy.fft.dct(x, type=2, norm=None, axis=-1)[:, :mfccs] / math.sqrt(2 * mel)
    np.testing.assert_allclose(x @ O.dct2_matrix(mel, mfccs), ref, rtol=1e-12, atol=1e-12)


def test_silence_gives_log_offset():
    wav = np.zeros((1, 16000), np.float32)
    lm = O.log_mel_spectrogram(wav, 640, 320)
    np.testing.assert_allclose(lm, math.log(1e-6), rtol=0, atol=1e-12)


def _tiny_problem(model="TCResNet8", wm=1.0, t=25, n=3, seed=0):
    spec = O.build_spec(model, wm, t)
    params, moving = O.init_variables(spec, seed)
    rng = np.random.RandomState(seed + 1)
    for k in params:                                       # non-trivial gamma/beta
        if k.endswith("gamma"):
            params[k] = 1.0 + 0.2 * rng.randn(*params[k].shape)
        if k.endswith("beta"):
            params[k] = 0.1 * rng.randn(*params[k].shape)
    feat = rng.randn(n, t, 40)
    lab = rng.randint(0, 12, size=n)
    onehot = np.eye(12)[lab]
    mask = (rng.rand(n, spec.c_last) < 0.5).astype(np.float64)
    return spec, params, moving, feat, onehot, mask


@pytest.mark.parametrize("model,wm,t", [("TCResNet8", 1.0, 25), ("TCResNet14", 1.0, 18)])
def test_gradients_against_finite_differences(model, wm, t):
    spec, params, moving, feat, onehot, mask = _tiny_problem(model, wm, t)
    wd, keep = 1e-3, 0.5

    def total(p):
        logits, _ = O.forward(spec, p, moving, feat, True, keep, mask)
        return O.losses(spec, p, logits, onehot, wd)[0]

    logits, cache = O.forward(spec, params, moving, feat, True, keep, mask)
    grads = O.backward(spec, params, cache, logits, onehot, wd)
    rng = np.random.RandomState(3)
    eps = 1e-6
    for name in spec.var_names:
        flat = params[name].ravel()
        for idx in rng.choice(flat.size, size=min(3, flat.size), replace=False):
            p2 = {k: v.copy() for k, v in params.items()}
            p2[name].ravel()[idx] += eps
            up = total(p2)
            p2[name].ravel()[idx] -= 2 * eps
            dn = total(p2)
            fd = (up - dn) / (2 * eps)
            an = grads[name].ravel()[idx]
            assert abs(fd - an) <= 1e-6 * max(1.0, abs(an)) + 2e-8, (name, idx, fd, an)


def _torch_reference(spec, params, feat, onehot, mask, keep, wd):
    """Independent restatement with torch ops + autograd (NCW conv1d, explicit SAME padding)."""
    tp = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in params.items()}
    x = torch.tensor(feat, dtype=torch.float64).permute(0, 2, 1)           # [N, C, T]

    def conv_bn(x, cv, relu):
        p = f"{spec.scope}/{cv.name}"
        w = tp[p + "/weights"][:, 0].permute(2, 1, 0)                       # [Cout, Cin, K]
        y = F.conv1d(F.pad(x, (cv.pad_left, cv.pad_right)), w, stride=cv.stride)
        z = F.batch_norm(y, None, None, tp[p + "/BatchNorm/gamma"], tp[p + "/BatchNorm/beta"],
                         training=True, eps=1e-3)
        return F.relu(z) if relu else z

    net = conv_bn(x, spec.conv0, True)
    for b in spec.blocks:
        short = conv_bn(net, b.down, True) if b.down is not None else net
        h = conv_bn(net, b.conv_a, True)
        h = conv_bn(h, b.conv_b, False)
        net = F.relu(h + short)
    pooled = net.mean(dim=2)
    dropped = pooled / keep * torch.tensor(mask)
    logits = dropped @ tp[f"{spec.scope}/fc/weights"].reshape(spec.c_last, spec.num_classes)
    ce = -(torch.tensor(onehot) * F.log_softmax(logits, dim=1)).sum(dim=1).mean()
    l2 = sum((v ** 2).sum() / 2 for k, v in tp.items() if "BatchNorm" not in k)
    total = ce + wd * l2
    total.backward()
    return logits.detach().numpy(), float(total), {k: v.grad.numpy() for k, v in tp.items()}


@pytest.mark.parametrize("model,wm,t", [("TCResNet8", 1.0, 49), ("TCResNet14", 1.5, 49), ("TCResNet8", 1.5, 98)])
def test_against_independent_torch_autograd(model, wm, t):
    spec, params, moving, feat, onehot, mask = _tiny_problem(model, wm, t, n=4)
    wd, keep = 1e-3, 0.5
    logits, cache = O.forward(spec, params, moving, feat, True, keep, mask)
    total, _ = O.losses(spec, params, logits, onehot, wd)
    grads = O.backward(spec, params, cache, logits, onehot, wd)
    t_logits, t_total, t_grads = _torch_reference(spec, params, feat, onehot, mask, keep, wd)
    np.testing.assert_allclose(logits, t_logits, rtol=1e-9, atol=1e-11)
    assert abs(total - t_total) < 1e-10
    for name in spec.var_names:
        np.testing.assert_allclose(grads[name], t_grads[name], rtol=1e-7, atol=1e-10, err_msg=name)


def test_eval_mode_uses_moving_stats_and_no_dropout():
    spec, params, moving, feat, onehot, mask = _tiny_problem()
    rng = np.random.RandomState(5)
    for k in moving:
        moving[k] = (rng.rand(*moving[k].shape) + 0.5) if k.endswith("variance") else 0.1 * rng.randn(*moving[k].shape)
    a, _ = O.forward(spec, params, moving, feat, False, 0.5, None)
    b, _ = O.forward(spec, params, moving, feat[:1], False, 0.5, None)
    np.testing.assert_allclose(a[:1], b, rtol=1e-12, atol=1e-12)       # no cross-utterance coupling in eval


def test_train_step_semantics():
    spec, params, moving, feat, onehot, mask = _tiny_problem()
    slots = O.zeros_like_vars(spec)
    lr, mom, wd = 0.1, 0.9, 1e-3
    p1, mv1, s1, out = O.train_step(spec, params, moving, slots, feat, onehot, lr, mom, wd)
    name = f"{spec.scope}/conv0/weights"
    np.testing.assert_allclose(s1[name], out["grads"][name])
    np.testing.assert_allclose(p1[name], params[name] - lr * out["grads"][name])
    p2, mv2, s2, out2 = O.train_step(spec, p1, mv1, s1, feat, onehot, lr, mom, wd)
    np.testing.assert_allclose(s2[name], mom * s1[name] + out2["grads"][name])
    # dead fc2 head: only weight decay moves it
    fc2 = f"{spec.scope}/fc2/weights"
    np.testing.assert_allclose(out["grads"][fc2], wd * params[fc2])
    # moving variance uses the UNBIASED batch variance, decay 0.997, no zero-debias
    y = out["cache"]["conv0"]["y"]
    m = y.shape[0] * y.shape[1]
    key = f"{spec.scope}/conv0/BatchNorm/moving_variance"
    np.testing.assert_allclose(mv1[key], 1.0 - (1.0 - y.var(axis=(0, 1)) * m / (m - 1)) * (1 - 0.997))
    assert out["total_loss"] > out["model_loss"] > 0


def test_piecewise_constant():
    b, v = [10000, 20000], [0.1, 0.01, 0.001]
    assert O.piecewise_constant(0, b, v) == 0.1
    assert O.piecewise_constant(10000, b, v) == 0.1
    assert O.piecewise_constant(10001, b, v) == 0.01
    assert O.piecewise_constant(20001, b, v) == 0.001


def test_flat_roundtrip():
    spec = O.build_spec("TCResNet8", 1.0, 49)
    params, moving = O.init_variables(spec, 0, np.float32)
    flat = O.flatten_vars(spec, params)
    assert flat.shape == (65264,)
    back = O.unflatten_vars(spec, flat, np.float32)
    for k in params:
        np.testing.assert_array_equal(params[k], back[k])
    fm = O.flatten_moving(spec, moving)
    assert fm.shape == (2 * 328,)
    back = O.unflatten_moving(spec, fm, np.float32)
    for k in moving:
        np.testing.assert_array_equal(moving[k], back[k])


def test_torch_cpu_port_matches_numpy_oracle():
    """The PyTorch-CPU port bench.py times as the CPU baseline is the same arithmetic as the NumPy oracle."""
    from oracle.torch_port import TorchPort
    spec = O.build_spec("TCResNet8", 1.0, 49)
    params, moving = O.init_variables(spec, 0)
    wav, onehot = O.synthetic_batch(6)
    rng = np.random.RandomState(2)
    mask = (rng.rand(6, spec.c_last) < 0.5).astype(np.float64)
    port = TorchPort(spec, params, moving, 640, 320, keep_prob=0.5, dtype=torch.float64)
    feat = O.mfcc(wav, 640, 320)
    np.testing.assert_allclose(port.mfcc(torch.tensor(wav, dtype=torch.float64)).numpy(), feat, rtol=1e-7, atol=1e-7)
    slots = O.zeros_like_vars(spec)
    p1, mv1, s1, ref = O.train_step(spec, params, moving, slots, feat, onehot, 0.1, 0.9, 1e-3, 0.5, mask)
    total, ce, logits = port.train_step(torch.tensor(wav, dtype=torch.float64), torch.tensor(onehot, dtype=torch.float64),
                                        0.1, 0.9, 1e-3, torch.tensor(mask))
    assert abs(total - ref["total_loss"]) < 1e-9 and abs(ce - ref["model_loss"]) < 1e-9
    for k in p1:
        np.testing.assert_allclose(port.p[k].detach().numpy(), p1[k], rtol=1e-7, atol=1e-9, err_msg=k)
    for k in mv1:
        np.testing.assert_allclose(port.mv[k].numpy(), mv1[k], rtol=1e-7, atol=1e-9, err_msg=k)
