"""Parity cases shared by the emulator (CPU) and GPU tests: CUDA path through the C ABI vs the fp64 oracle.

Tolerance (BASELINE.json north_star, SURVEY.md 8c): max_i |x_cuda - x_ref| / max_i |x_ref| <= 1e-4 for logits
against the fp64 oracle, arg-max class identical on every row whose top-2 margin exceeds that error; the same
rule for gradients / post-step state, floored by the fp32 oracle's own distance to fp64.
"""
from __future__ import annotations

import numpy as np

from oracle import tcr_oracle as O
from tcr_harness import Engine, rel_err

TOL_FEATURES = 2e-5
TOL_LOGITS = 1e-4
TOL_STATE = 1e-4


def perturbed_variables(spec, seed=0):
    """Xavier weights (NumPy seed 0, SURVEY 8d) with non-trivial gamma/beta/moving stats so BN paths are exercised."""
    params, moving = O.init_variables(spec, seed)
    rng = np.random.RandomState(seed + 1)
    for k in params:
        if k.endswith("gamma"):
            params[k] = 1.0 + 0.2 * rng.randn(*params[k].shape)
        if k.endswith("beta"):
            params[k] = 0.1 * rng.randn(*params[k].shape)
    for k in moving:
        moving[k] = (rng.rand(*moving[k].shape) + 0.5) if k.endswith("variance") else 0.1 * rng.randn(*moving[k].shape)
    return params, moving


def cuda_relu_masks(eng, spec, n):
    """The ReLU decisions the CUDA path took in its last training step, rebuilt from its workspace (pre-BN outputs `y:<conv>`,
    the BN tables `bnf:<conv>` and the block outputs `out:<block>`): bn(y) = fma(y - mean, scale, beta) > 0.  Forcing them on the
    oracle removes mask flips of activations within round-off of zero from the gradient comparison (they dominate it at
    batch 512 / 1024: a flipped unit changes its whole fan-in's gradient), so the bound on gradients can be the plain 1e-4."""
    masks = {}
    for cv in spec.convs():
        if not cv.relu:
            continue
        y = eng.workspace(f"y:{cv.name}").reshape(-1, cv.t_out, cv.cout)[:n]
        t = eng.workspace(f"bnf:{cv.name}").reshape(4, cv.cout)
        d = (y - t[0]).astype(np.float32).astype(np.float64)            # the subtraction rounds to fp32, the fma does not
        masks[cv.name] = (d * t[2].astype(np.float64) + t[3].astype(np.float64)) > 0
    for b in spec.blocks:
        masks[f"block{b.index}"] = eng.workspace(f"out:block{b.index}").reshape(-1, b.conv_b.t_out, b.conv_b.cout)[:n] > 0
    return masks


def check_argmax(logits, ref_logits, err_abs):
    ref_sorted = np.sort(ref_logits, axis=1)
    margin = ref_sorted[:, -1] - ref_sorted[:, -2]
    decided = margin > 2 * err_abs
    assert np.array_equal(np.argmax(logits, 1)[decided], np.argmax(ref_logits, 1)[decided])
    return int((~decided).sum())


def reference_features(wav, window, stride, sample_rate=16000, mel=64, mfcc=40, lower=80.0, upper=7600.0, feature_kind=0,
                       dtype=np.float64):
    """The oracle front-end of a handle's configuration: MFCCs (feature_kind 0) or the magnitude log-mel spectrogram (1)."""
    if feature_kind == 0:
        return O.mfcc(wav, window, stride, mel, mfcc, sample_rate, lower, upper, dtype)
    return O.log_mel_spectrogram(wav, window, stride, False, mel, sample_rate, lower, upper, dtype)


def check_eval(eng, spec, inp, feat, onehot, params, moving, wd, ls, report, tag="eval", is_features=False):
    """evaluate_audio.py path (moving statistics, dropout identity) against the oracle; the CUDA path gets the variables in fp32."""
    ev = eng.forward(inp, O.flatten_vars(spec, params), O.flatten_moving(spec, moving), is_features=is_features, onehot_np=onehot, weight_decay=wd)
    ref_logits, _ = O.forward(spec, params, moving, feat, False)
    ref_total, ref_model = O.losses(spec, params, ref_logits, onehot, wd, ls)
    report[f"{tag}_logits"] = rel_err(ev["logits"], ref_logits)
    assert report[f"{tag}_logits"] <= TOL_LOGITS, report
    check_argmax(ev["logits"], ref_logits, report[f"{tag}_logits"] * np.abs(ref_logits).max())
    np.testing.assert_allclose(ev["probs"], O.softmax(ref_logits), rtol=0, atol=2e-5)
    assert abs(ev["losses"][0] - ref_total) <= 1e-4 * abs(ref_total) + 1e-6
    assert abs(ev["losses"][1] - ref_model) <= 1e-4 * abs(ref_model) + 1e-6


def check_step(eng, spec, inp, feat, onehot, state, lr, mom, wd, keep, mask, ls, report, tag, seed=0, is_features=False,
               check_f32_floor=False, force_masks=False, feat_f32=None):
    """One training step of the CUDA path from the flat state (params, moving, slots) against the oracle step started from the
    same state; returns the CUDA path's post-step state.  feat_f32: the features the fp32 restatement of the oracle starts
    from (default: the fp64 features rounded to fp32)."""
    pf_c, mf_c, sf_c = state
    n = inp.shape[0]
    p = O.unflatten_vars(spec, pf_c)
    mv = O.unflatten_moving(spec, mf_c)
    sl = O.unflatten_vars(spec, sf_c)
    ts = eng.train_step(inp, onehot, pf_c, sf_c, mf_c, lr, mom, wd, is_features=is_features, mask_np=mask, seed=seed)
    forced = cuda_relu_masks(eng, spec, n) if force_masks else None
    p1, mv1, sl1, ref = O.train_step(spec, p, mv, sl, feat, onehot, lr, mom, wd, keep, mask, ls, forced_masks=forced)
    report[f"train_logits{tag}"] = rel_err(ts["logits"], ref["logits"])
    report[f"grads{tag}"] = rel_err(ts["grads"], O.flatten_vars(spec, ref["grads"], np.float64))
    report[f"params{tag}"] = rel_err(ts["params"], O.flatten_vars(spec, p1, np.float64))
    report[f"slots{tag}"] = rel_err(ts["slots"], O.flatten_vars(spec, sl1, np.float64))
    report[f"moving{tag}"] = rel_err(ts["moving"], O.flatten_moving(spec, mv1, np.float64))
    floor = 0.0
    if check_f32_floor:                      # every step: the fp32 NumPy oracle's own distance to fp64 on this input
        p32, mv32, sl32 = (O.cast_vars(d, np.float32) for d in (p, mv, sl))
        f32 = feat.astype(np.float32) if feat_f32 is None else feat_f32
        _, _, _, r32 = O.train_step(spec, p32, mv32, sl32, f32, onehot, lr, mom, wd, keep, mask, ls)
        floor = 4 * rel_err(O.flatten_vars(spec, r32["grads"], np.float64), O.flatten_vars(spec, ref["grads"], np.float64))
        report[f"grads_f32_oracle_floor{tag}"] = floor / 4
    assert report[f"train_logits{tag}"] <= TOL_LOGITS, report
    assert report[f"grads{tag}"] <= max(TOL_STATE, floor), report
    assert report[f"params{tag}"] <= max(TOL_STATE, floor), report
    assert report[f"slots{tag}"] <= max(TOL_STATE, floor), report
    assert report[f"moving{tag}"] <= TOL_STATE, report
    assert abs(ts["losses"][0] - ref["total_loss"]) <= 1e-4 * abs(ref["total_loss"]) + 1e-6
    assert abs(ts["losses"][1] - ref["model_loss"]) <= 1e-4 * abs(ref["model_loss"]) + 1e-6
    return ts["params"], ts["moving"], ts["slots"]


def run_case(backend, model="TCResNet8", wm=1.0, window=640, stride=320, n=4, keep=1.0, ls=0.0, use_wav=True,
             steps=1, adversarial=True, max_batch=None, check_f32_floor=False, force_masks=False, sample_rate=16000, clip=16000,
             mel=64, mfcc=40, lower=80.0, upper=7600.0, num_classes=12, feature_kind=0, f32_front_end=False):
    """f32_front_end: with check_f32_floor, the fp32 restatement of the oracle also computes its features in fp32, so the floor
    includes the front-end's round-off as the gradient amplifies it (log-mel features keep ~1e-5 of it in their quiet bands)."""
    t = O.num_frames(clip, window, stride)
    f_in = mfcc if feature_kind == 0 else mel
    spec = O.build_spec(model, wm, t, f_in=f_in, num_classes=num_classes)
    eng = Engine(backend, model=int(model[len("TCResNet"):]), width_multiplier=wm, max_batch=max_batch or max(n, 8),
                 dropout_keep_prob=keep, window_size_samples=window, window_stride_samples=stride, label_smoothing=ls,
                 sample_rate=sample_rate, clip_samples=clip, num_mel_bins=mel, num_mfccs=mfcc, lower_edge_hertz=lower,
                 upper_edge_hertz=upper, num_classes=num_classes, feature_kind=feature_kind)
    try:
        assert eng.info.frames == t and eng.info.features == f_in and eng.info.num_trainable == O.count_trainable(spec)
        assert eng.info.forward_flops_per_utt == O.forward_flops(spec)
        tab = eng.param_table()
        assert [d["name"] for d in tab if d["kind"] < 3] == spec.var_names
        assert [d["name"] for d in tab if d["kind"] >= 3] == O.moving_names(spec)
        params, moving = perturbed_variables(spec)
        rng = np.random.RandomState(7)
        slots = {k: 0.01 * rng.randn(*v.shape) for k, v in params.items()}
        wav, onehot = O.synthetic_batch(n, num_samples=clip, num_classes=num_classes, adversarial=adversarial)
        feat = reference_features(wav, window, stride, sample_rate, mel, mfcc, lower, upper, feature_kind)
        mask = (rng.rand(n, spec.c_last) < keep).astype(np.float32) if keep < 1 else None
        lr, mom, wd = 0.1, 0.9, 1e-3
        report = {}

        # front-end
        f_cuda = eng.mfcc(wav)
        report["features"] = rel_err(f_cuda, feat)
        assert report["features"] <= TOL_FEATURES, report

        inp = wav if use_wav else feat.astype(np.float32)
        feat_f32 = reference_features(wav, window, stride, sample_rate, mel, mfcc, lower, upper, feature_kind, np.float32) \
            if f32_front_end and use_wav else None
        check_eval(eng, spec, inp, feat, onehot, params, moving, wd, ls, report, is_features=not use_wav)

        # training steps.  Each step is compared against the oracle started from the CUDA path's OWN previous state
        # (re-synchronised), so the check is per-step parity + correct carrying of state between calls, not the
        # divergence of two chaotic lr=0.1 trajectories (ReLU masks flip under 1e-6 perturbations).
        state = O.flatten_vars(spec, params), O.flatten_moving(spec, moving), O.flatten_vars(spec, slots)
        for step in range(steps):
            state = check_step(eng, spec, inp, feat, onehot, state, lr, mom, wd, keep, mask, ls, report, step, seed=step,
                               is_features=not use_wav, check_f32_floor=check_f32_floor, force_masks=force_masks, feat_f32=feat_f32)
        return report
    finally:
        eng.close()


def spectral_lines():
    """Seven full-scale sines (on and between bin centres; 2296.875 Hz = bin 147 has the smallest falling mel weight) over a
    -60 dB noise floor: the worst case of the frame-pair front-end kernel's run-based mel stage."""
    t = np.arange(16000) / 16000.0
    rng = np.random.default_rng(3)
    return np.stack([np.sin(2 * np.pi * f * t) for f in (100.0, 437.3, 2296.875, 2345.6, 3999.0, 6999.9, 7590.0)]) \
        + 1e-3 * rng.uniform(-1, 1, (7, 16000))
