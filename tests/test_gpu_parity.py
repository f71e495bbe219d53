"""Parity tests proper: the sm_90a CUDA path through the C ABI vs the fp64 oracle, on a real H100."""
import numpy as np
import pytest

from parity_cases import run_case, perturbed_variables
from tcr_harness import Engine, launched, rel_err
from oracle import tcr_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def backend():
    from tcr_harness import TorchBackend
    return TorchBackend()


@pytest.mark.parametrize("kw", [
    dict(model="TCResNet8", wm=1.0, window=640, stride=320, n=1),                      # config 1 (plumbing)
    dict(model="TCResNet8", wm=1.0, window=640, stride=320, n=3, keep=0.5),            # eval-script batch size
    dict(model="TCResNet8", wm=1.0, window=640, stride=320, n=39, keep=0.5, steps=2, force_masks=True),  # test-script batch size
    dict(model="TCResNet8", wm=1.0, window=480, stride=160, n=37, keep=0.5, ls=0.1),   # script shape T=98, pad (3,4)
    dict(model="TCResNet14", wm=1.5, window=640, stride=320, n=21, keep=0.5),
    dict(model="TCResNet14", wm=1.0, window=480, stride=160, n=16, use_wav=False, steps=3, force_masks=True),
    dict(model="TCResNet8", wm=1.5, window=640, stride=320, n=150, check_f32_floor=True),
], ids=["r8-n1", "r8-n3", "r8-n39-2steps", "r8-T98-n37", "r14x1.5-n21", "r14-T98-3steps", "r8x1.5-n150"])
def test_cuda_path_matches_oracle(backend, kw):
    run_case(backend, **kw)


def step_launches(backend, model, n):
    """Kernel names of one training step on a handle sized for n utterances (each handle picks its resident mode)."""
    spec = O.build_spec(model, 1.0, 49)
    pv, mv = O.init_variables(spec, 0)
    pf, mf = O.flatten_vars(spec, pv).astype(np.float32), O.flatten_moving(spec, mv).astype(np.float32)
    wav, onehot = O.synthetic_batch(n)
    eng = Engine(backend, model=int(model[len("TCResNet"):]), max_batch=n, dropout_keep_prob=0.5)
    try:
        return set(launched(backend.lib, lambda: eng.train_step(wav, onehot, pf, np.zeros_like(pf), mf)))
    finally:
        eng.close()


@pytest.mark.parametrize("mode", ["0", "1", "3"])
def test_resident_kernels_match_oracle(backend, monkeypatch, mode):
    """TCR_RESIDENT = 0: per-layer kernels; 1: resident forward kernel, per-layer backward-data kernels; 3 (the default): resident
    forward and backward-data kernels (csrc/tcr_resident.cu).  Every mode meets the same bounds, including the headline shape
    (4 utterances per SM), and the launch profiler shows that each shape ran the kernels of the mode asked for."""
    monkeypatch.setenv("TCR_RESIDENT", mode)
    run_case(backend, model="TCResNet8", wm=1.0, window=640, stride=320, n=64, keep=0.5, steps=2)
    run_case(backend, model="TCResNet8", wm=1.0, window=640, stride=320, n=512, keep=0.5, force_masks=True)
    run_case(backend, model="TCResNet14", wm=1.0, window=640, stride=320, n=33, keep=1.0)
    for model, n in (("TCResNet8", 64), ("TCResNet8", 512), ("TCResNet14", 33)):
        names = step_launches(backend, model, n)
        fwd, dx = any(k.startswith("fwd:") for k in names), any(k.startswith("dx:") for k in names)
        if mode == "0":
            assert {"weight_transpose", "dw_grouped", "grad_finalize", "update"} <= names and fwd and dx, (model, n, names)
            assert not {"resident_fwd", "resident_bwd_data"} & names, (model, n, names)
        elif mode == "1":
            assert {"resident_fwd", "dw_grouped", "grad_finalize", "update"} <= names and dx and not fwd, (model, n, names)
            assert "resident_bwd_data" not in names, (model, n, names)
        else:
            assert {"resident_fwd", "resident_bwd_data", "dw_grouped", "grad_finalize", "update"} <= names, (model, n, names)
            assert not fwd and not dx, (model, n, names)


def test_log_mel_front_end_on_sm100a(backend):
    """TCR_FEATURE_LOG_MEL (LogMelSpectrogramPreprocessor._preprocess, datasets/preprocessors.py:162-170: magnitude spectrogram,
    no DCT): T=49 and T=98, silence and a full-scale square wave included, and a network step on the 64-bin features."""
    wav, onehot = O.synthetic_batch(6, adversarial=True)
    for window, stride in ((640, 320), (480, 160)):
        eng = Engine(backend, feature_kind=1, max_batch=8, window_size_samples=window, window_stride_samples=stride)
        got = eng.mfcc(wav)
        ref = O.log_mel_spectrogram(wav, window, stride, magnitude_squared=False)
        assert got.shape == ref.shape == (6, O.num_frames(16000, window, stride), 64)
        assert rel_err(got, ref) < 2e-5
        eng.close()
    # the network on log-mel features (F = 64): evaluation forward against the oracle
    eng = Engine(backend, feature_kind=1, max_batch=8)
    spec = O.build_spec("TCResNet8", 1.0, 49, f_in=64)
    params, moving = perturbed_variables(spec)
    feat = O.log_mel_spectrogram(wav, 640, 320, magnitude_squared=False)
    ev = eng.forward(wav, O.flatten_vars(spec, params), O.flatten_moving(spec, moving))
    ref_logits, _ = O.forward(spec, params, moving, feat, False)
    assert rel_err(ev["logits"], ref_logits) < 1e-4
    eng.close()


def test_unsupported_width_is_reported_through_the_model_class(backend):
    """width_multiplier 0.75 gives 12 / 18 / 24 / 36 channels; 18 is not a multiple of 4: the documented TCR_ERR_UNSUPPORTED
    (status 3) surfaces as TcrError from the reference-named model class, not as a wrong result."""
    import argparse
    from tcresnet_b200._lib import TcrError
    from tcresnet_b200.factory import audio_nets
    from tcresnet_b200.runtime import Node
    args = argparse.Namespace(width_multiplier=0.75, num_classes=12, sample_rate=16000, clip_duration_ms=1000, window_size_ms=40.0,
                              window_stride_ms=20.0, num_mel_bins=64, num_mfccs=40, lower_edge_hertz=80.0, upper_edge_hertz=7600.0,
                              preprocess_method="mfcc", batch_size=8, dropout_keep_prob=0.5, output_name="output/softmax", weight_decay=1e-3)
    model = audio_nets.TCResNet8Model(args, None)
    with pytest.raises(TcrError, match="not a positive multiple of 4"):
        model.build(Node("wavs", [None, 16000, 1]), Node("labels", [None, 12]), True)


def test_pcm16_input_matches_decoded_samples_bitwise(backend):
    """TCR_INPUT_WAV_PCM16 == decode_wav (x / 32768) followed by the fp32 path, bit for bit, front-end and full step."""
    eng = Engine(backend, max_batch=64)
    rng = np.random.default_rng(11)
    pcm = rng.integers(-32768, 32768, size=(64, 16000), dtype=np.int16)
    dec = pcm.astype(np.float32) / 32768.0
    got, ref = eng.mfcc(pcm), eng.mfcc(dec)
    assert np.array_equal(got, ref)
    assert rel_err(got, O.mfcc(pcm.astype(np.float64) / 32768.0, 640, 320)) < 1e-6
    spec = O.build_spec("TCResNet8", 1.0, 49)
    pv, mv = O.init_variables(spec, 3)
    params, moving = O.flatten_vars(spec, pv).astype(np.float32), O.flatten_moving(spec, mv).astype(np.float32)
    onehot = np.eye(12, dtype=np.float32)[rng.integers(0, 12, 64)]
    a = eng.train_step(pcm, onehot, params, np.zeros_like(params), moving, seed=4)
    b = eng.train_step(dec, onehot, params, np.zeros_like(params), moving, seed=4)
    assert np.array_equal(a["params"], b["params"]) and np.array_equal(a["losses"], b["losses"])
    eng.close()


def test_host_feed_pipeline_matches_device_steps(backend):
    """tcr_train_step_host through tcresnet_b200.engine.HostFeed: 6 pipelined steps from pinned host buffers (fp32 and int16)
    leave exactly the parameters that 6 device-buffer steps leave, and every step's loss comes back once, in order."""
    import torch
    from tcresnet_b200.engine import Engine as PublicEngine, HostFeed
    eng = PublicEngine(max_batch=32)
    gen = torch.Generator().manual_seed(3)
    pcm = [torch.randint(-30000, 30000, (32, 16000), generator=gen, dtype=torch.int16).pin_memory() for _ in range(3)]
    dec = [(p.float() / 32768.0).pin_memory() for p in pcm]
    hot = [torch.nn.functional.one_hot(torch.randint(0, 12, (32,), generator=gen), 12).float().pin_memory() for _ in range(3)]
    results = {}
    for kind, bufs in (("device", dec), ("host_f32", dec), ("host_pcm16", pcm)):
        params, slots, moving = eng.new_variables(seed=1)
        losses = []
        if kind == "device":
            for i in range(6):
                out = eng.train_step(bufs[i % 3].cuda(), hot[i % 3].cuda(), params, slots, moving, 0.05, 0.9, 1e-3, dropout_seed=i)
                losses.append(tuple(out["losses"].tolist()))
        else:
            feed = HostFeed(eng, lag=2)
            got = [feed.submit(bufs[i % 3], hot[i % 3], params, slots, moving, 0.05, 0.9, 1e-3, dropout_seed=i) for i in range(6)]
            rest = feed.flush()
            idx = [g[0] for g in got[2:] + rest]             # the step counter is per handle: consecutive, each step once
            assert got[0] is None and got[1] is None and idx == list(range(idx[0], idx[0] + 6))
            losses = [(g[1], g[2]) for g in got[2:] + rest]
        torch.cuda.synchronize()
        results[kind] = (params.cpu().numpy(), np.array(losses, np.float32))
    for kind in ("host_f32", "host_pcm16"):
        assert np.array_equal(results[kind][0], results["device"][0]), kind
        assert np.array_equal(results[kind][1], results["device"][1]), kind
    eng.close()


def test_without_thread_block_clusters(backend, monkeypatch):
    """TCR_CLUSTER=1: one statistics record per CTA instead of one per 8-CTA cluster; same results within tolerance."""
    monkeypatch.setenv("TCR_CLUSTER", "1")
    run_case(backend, model="TCResNet8", wm=1.0, window=640, stride=320, n=70, keep=0.5, steps=2, force_masks=True)
    monkeypatch.setenv("TCR_CLUSTER", "4")
    run_case(backend, model="TCResNet14", wm=1.0, window=640, stride=320, n=19, keep=1.0)


def test_full_size_config2_tcresnet8_n512(backend):
    # gradients / post-step state at the plain 1e-4 bound: the oracle takes the CUDA path's ReLU decisions (parity_cases.py)
    report = run_case(backend, model="TCResNet8", wm=1.0, n=512, keep=0.5, max_batch=512, force_masks=True)
    print(report)


def test_full_size_config3_tcresnet14x15_n1024(backend):
    report = run_case(backend, model="TCResNet14", wm=1.5, n=1024, keep=0.5, max_batch=1024, force_masks=True)
    print(report)


def test_launch_counter_proves_the_cuda_path_ran(backend):
    import ctypes as C
    before, after = C.c_uint64(), C.c_uint64()
    backend.lib.tcr_launch_count(C.byref(before))
    run_case(backend, n=4)
    backend.lib.tcr_launch_count(C.byref(after))
    assert after.value - before.value >= 10      # mfcc (1) + eval forward (11) + one training step


def test_training_step_is_bitwise_deterministic(backend):
    spec = O.build_spec("TCResNet8", 1.0, 49)
    params, moving = perturbed_variables(spec)
    wav, onehot = O.synthetic_batch(300)
    eng = Engine(backend, max_batch=300, dropout_keep_prob=0.5)
    pf, mf = O.flatten_vars(spec, params), O.flatten_moving(spec, moving)
    sf = np.zeros_like(pf)
    a = eng.train_step(wav, onehot, pf, sf, mf, seed=11)
    b = eng.train_step(wav, onehot, pf, sf, mf, seed=11)
    for k in ("logits", "grads", "params", "moving", "losses"):
        assert np.array_equal(a[k], b[k]), k
    c = eng.train_step(wav, onehot, pf, sf, mf, seed=12)     # a different dropout seed changes the step
    assert not np.array_equal(a["grads"], c["grads"])
    eng.close()


def test_eval_forward_is_per_utterance(backend):
    """No cross-utterance coupling in the evaluate_audio.py path: permuting / slicing the batch permutes logits."""
    spec = O.build_spec("TCResNet14", 1.0, 49)
    params, moving = perturbed_variables(spec)
    wav, _ = O.synthetic_batch(64, adversarial=True)
    eng = Engine(backend, model=14, max_batch=64)
    pf, mf = O.flatten_vars(spec, params), O.flatten_moving(spec, moving)
    full = eng.forward(wav, pf, mf)["logits"]
    perm = np.random.RandomState(0).permutation(64)
    np.testing.assert_array_equal(eng.forward(wav[perm], pf, mf)["logits"], full[perm])
    np.testing.assert_array_equal(eng.forward(wav[5:8], pf, mf)["logits"], full[5:8])
    eng.close()


def test_gradient_is_linear_in_the_shards(backend):
    """Data-parallel identity used by the multi-GPU path: with BN statistics computed per shard, the mean of the
    per-shard gradients of (CE) equals what N ranks all-reduce; checked against the oracle shard-wise."""
    spec = O.build_spec("TCResNet8", 1.0, 49)
    params, moving = perturbed_variables(spec)
    wav, onehot = O.synthetic_batch(64)
    feat = O.mfcc(wav, 640, 320)
    eng = Engine(backend, max_batch=64, dropout_keep_prob=1.0)
    pf, mf = O.flatten_vars(spec, params), O.flatten_moving(spec, moving)
    sf = np.zeros_like(pf)
    acc = np.zeros_like(pf, dtype=np.float64)
    ref = np.zeros_like(pf, dtype=np.float64)
    for r in range(2):
        sl = slice(32 * r, 32 * (r + 1))
        acc += eng.train_step(wav[sl], onehot[sl], pf, sf, mf, apply_update=False)["grads"]
        logits, cache = O.forward(spec, params, moving, feat[sl], True)
        ref += O.flatten_vars(spec, O.backward(spec, params, cache, logits, onehot[sl], 1e-3), np.float64)
    assert rel_err(acc / 2, ref / 2) < 1e-4
    eng.close()


def test_silent_batch_and_full_scale(backend):
    """Adversarial inputs of SURVEY 8(d): an all-silent clip gives log(1e-6) in every mel bin; +-1 square wave."""
    eng = Engine(backend, max_batch=4)
    wav = np.zeros((2, 16000), np.float32)
    wav[1] = np.where((np.arange(16000) // 40) % 2 == 0, 1.0, -1.0)
    got = eng.mfcc(wav)
    ref = O.mfcc(wav, 640, 320)
    assert np.isfinite(got).all()
    assert rel_err(got, ref) < 2e-5
    eng.close()


def test_handles_of_different_size_share_the_resident_kernels(backend):
    """The shared-memory opt-in of the resident kernels is a per-FUNCTION attribute: a second, smaller handle created later must
    not lower it under the first handle (bench.py's dp_check does exactly this: a 16-utterance handle next to the 512 one)."""
    import torch
    from tcresnet_b200.engine import Engine
    big = Engine(max_batch=512)
    p, s, m = big.new_variables(seed=0)
    gen = torch.Generator(device="cuda").manual_seed(3)
    wav = torch.rand(512, 16000, device="cuda", generator=gen) * 2 - 1
    hot = torch.nn.functional.one_hot(torch.randint(0, 12, (512,), device="cuda", generator=gen), 12).float()
    l0 = float(big.train_step(wav, hot, p.clone(), s.clone(), m.clone(), 0.1)["losses"][0])
    small = Engine(max_batch=16)
    ps, ss, ms = small.new_variables(seed=0)
    small.train_step(wav[:16], hot[:16], ps, ss, ms, 0.1)
    l1 = float(big.train_step(wav, hot, p.clone(), s.clone(), m.clone(), 0.1)["losses"][0])             # launch still fits
    assert l0 == l1
    small.close(); big.close()


def test_frontend_running_ahead_is_bitwise_equal(backend):
    """tcr_step_args::input_resident lets the front-end of a step run on the library's own stream, ahead of the previous step's tail.
    Same inputs, same seeds -> the same bits as the fully ordered steps, over rotating input buffers and both feature buffers."""
    import torch
    from tcresnet_b200.engine import Engine
    gen = torch.Generator(device="cuda").manual_seed(11)
    wavs = [torch.rand(96, 16000, device="cuda", generator=gen) * 2 - 1 for _ in range(3)]
    hots = [torch.nn.functional.one_hot(torch.randint(0, 12, (96,), device="cuda", generator=gen), 12).float() for _ in range(3)]
    results = []
    for ahead in (False, True):
        eng = Engine(max_batch=96, dropout_keep_prob=0.5)
        p, s, m = eng.new_variables(seed=0)
        losses = []
        for i in range(7):
            out = eng.train_step(wavs[i % 3], hots[i % 3], p, s, m, 0.05, dropout_seed=i, input_resident=ahead)
            losses.append(out["losses"].clone())
        torch.cuda.synchronize()
        results.append((p.clone(), s.clone(), m.clone(), torch.stack(losses)))
        eng.close()
    for x, y in zip(*results):
        assert torch.equal(x, y)


@pytest.mark.parametrize("pair", ["1", "6", "0"], ids=["pairs-10-per-item", "pairs-6-per-item", "one-frame-per-warp"])
def test_both_front_end_kernels_on_sm100a(backend, monkeypatch, pair):
    """TCR_MFCC_PAIR on the GPU: frame-pair kernel (default) and one-frame-per-warp kernel against the fp64 oracle, MFCC and
    log-mel, noise + silence + full-scale square wave, n not a multiple of anything; int16 input bit-identical to the decoded
    samples."""
    monkeypatch.setenv("TCR_MFCC_PAIR", pair)
    wav, _ = O.synthetic_batch(37, adversarial=True)
    for kind, ref in ((0, O.mfcc(wav, 640, 320)), (1, O.log_mel_spectrogram(wav, 640, 320, magnitude_squared=False))):
        eng = Engine(backend, feature_kind=kind, max_batch=64)
        got = eng.mfcc(wav)
        assert rel_err(got, ref) < (2e-6 if kind == 0 else 2e-5)
        pcm = np.clip(np.round(wav * 32768.0), -32768, 32767).astype(np.int16)
        assert np.array_equal(eng.mfcc(pcm), eng.mfcc(pcm.astype(np.float32) / 32768.0))
        eng.close()


def test_spectral_lines_through_the_run_based_mel_stage_on_sm100a(backend, monkeypatch):
    """Strong spectral lines over a -60 dB floor (see tests/test_emu_parity.py): the frame-pair kernel's run-based mel stage must
    not add to the fp32 FFT round-off that both kernels show under a line."""
    from parity_cases import spectral_lines
    tones = spectral_lines()
    err = {}
    for pair in ("1", "0"):
        monkeypatch.setenv("TCR_MFCC_PAIR", pair)
        for kind, ref in ((0, O.mfcc(tones, 640, 320)), (1, O.log_mel_spectrogram(tones, 640, 320, magnitude_squared=False))):
            eng = Engine(backend, feature_kind=kind, max_batch=8)
            err[pair, kind] = rel_err(eng.mfcc(tones), ref)
            eng.close()
    assert err["1", 0] < 2e-5 and err["1", 0] < 2.0 * err["0", 0] + 1e-6
    assert err["1", 1] < 1e-3 and err["1", 1] < 2.0 * err["0", 1] + 1e-6
