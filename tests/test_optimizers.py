"""Adam and RMSProp in the fused update kernel (tcr_step_args::optimizer) against their fp64 restatements in the oracle.

The update is compared on the CUDA path's OWN gradient: per step the `grads` output (the gradient the kernel applied) goes
into optim_oracle.adam_update / rmsprop_update in fp64, starting from the CUDA path's pre-step parameters and slots, and the
parameters, both slots and Adam's powers must match to 1e-6.  The gradient itself is held to the usual 1e-4 bound against the
oracle with the CUDA path's ReLU decisions forced.  (At Adam's first step the update is lr * sign(g) for every |g| >> eps, so a
gradient element at fp32 round-off whose sign differs from the fp64 oracle's would move a weight by 2 lr: comparing the
arithmetic on the same gradient keeps such tie-breaks out of the parameter check.)
"""
import ctypes as C
import shlex

import numpy as np
import pytest

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L
import optim_oracle as OO
from oracle import tcr_oracle as O
from parity_cases import cuda_relu_masks, perturbed_variables
from tcr_harness import Engine, NumpyBackend, rel_err

ADAM = dict(kind="adam", beta1=0.9, beta2=0.999, epsilon=1e-8)
RMSPROP = dict(kind="rmsprop", decay=0.9, momentum=0.0, epsilon=1e-10)
RMSPROP_MOM = dict(kind="rmsprop", decay=0.9, momentum=0.5, epsilon=1e-10)
TOL_UPDATE = 1e-6
TOL_GRADS = 1e-4


# ---------------------------------------------------------------------------------------------------- C-ABI step
def _fill_optimizer(a, opt, slots2_ptr, beta1_power=None, beta2_power=None):
    a.slots2, a.epsilon = slots2_ptr, opt["epsilon"]
    if opt["kind"] == "adam":
        a.optimizer, a.beta1, a.beta2 = L.TCR_OPT_ADAM, opt["beta1"], opt["beta2"]
        a.beta1_power, a.beta2_power = beta1_power, beta2_power
    else:
        a.optimizer, a.rho, a.momentum = L.TCR_OPT_RMSPROP, opt["decay"], opt["momentum"]


def opt_step(eng, inp, onehot, params, slots, slots2, moving, opt, powers=(None, None), lr=1e-3, wd=1e-3, seed=0, mask=None,
             apply_update=True, is_features=False):
    """One tcr_train_step with the optimizer fields set (the test harness's own TcrStepArgs)."""
    b = eng.b
    n = inp.shape[0]
    d_inp, d_hot = b.upload(inp), b.upload(onehot)
    d_p, d_s, d_s2, d_m = (b.upload(x) for x in (params, slots, slots2, moving))
    d_mask = b.upload(mask) if mask is not None else None
    losses, grads = b.empty(2), b.empty(eng.info.num_trainable)
    a = L.TcrStepArgs()
    a.input, a.input_is_features, a.onehot, a.n = b.ptr(d_inp), int(is_features), b.ptr(d_hot), n
    a.params, a.slots, a.moving = b.ptr(d_p), b.ptr(d_s), b.ptr(d_m)
    a.learning_rate, a.weight_decay = lr, wd
    a.dropout_seed, a.dropout_mask = seed, b.ptr(d_mask)
    a.losses, a.grads = b.ptr(losses), b.ptr(grads)
    a.apply_update = int(apply_update)
    _fill_optimizer(a, opt, b.ptr(d_s2), *powers)
    L.check(eng.lib, eng.lib.tcr_train_step(eng.h, C.byref(a), b.stream), "tcr_train_step")
    b.sync()
    return dict(grads=b.download(grads), params=b.download(d_p), slots=b.download(d_s), slots2=b.download(d_s2),
                moving=b.download(d_m), losses=b.download(losses))


def initial_state(opt, num):
    """TF's slot initialisers: Adam m, v = 0; RMSProp ms = 1 (TF 1.x), mom = 0.  Adam's powers start at beta1, beta2."""
    s1 = np.ones(num, np.float32) if opt["kind"] == "rmsprop" else np.zeros(num, np.float32)
    powers = (np.float32(opt["beta1"]), np.float32(opt["beta2"])) if opt["kind"] == "adam" else (None, None)
    return s1, np.zeros(num, np.float32), powers


def run_optimizer_case(backend, opt, model="TCResNet8", wm=1.0, n=8, steps=3, keep=0.5, lr=1e-3, wd=1e-3, max_batch=None):
    """`steps` teacher-forced steps (see the module docstring); returns the worst errors."""
    spec = O.build_spec(model, wm, 49)
    eng = Engine(backend, model=int(model[len("TCResNet"):]), width_multiplier=wm, max_batch=max_batch or max(n, 8),
                 dropout_keep_prob=keep)
    try:
        params, moving = perturbed_variables(spec)
        pf, mf = O.flatten_vars(spec, params), O.flatten_moving(spec, moving)
        s1, s2, powers = initial_state(opt, pf.size)
        wav, onehot = O.synthetic_batch(n, adversarial=True)
        feat = O.mfcc(wav, 640, 320)
        rng = np.random.RandomState(7)
        mask = (rng.rand(n, spec.c_last) < keep).astype(np.float32) if keep < 1 else None
        worst = {}
        for step in range(steps):
            ts = opt_step(eng, wav, onehot, pf, s1, s2, mf, opt, powers, lr=lr, wd=wd, seed=step, mask=mask)
            # the gradient and the BN moving averages against the oracle, with the CUDA path's ReLU decisions
            forced = cuda_relu_masks(eng, spec, n)
            _, mv1, _, ref = O.train_step(spec, O.unflatten_vars(spec, pf), O.unflatten_moving(spec, mf),
                                          O.zeros_like_vars(spec), feat, onehot, lr, 0.9, wd, keep, mask, forced_masks=forced)
            err = dict(grads=rel_err(ts["grads"], O.flatten_vars(spec, ref["grads"], np.float64)),
                       moving=rel_err(ts["moving"], O.flatten_moving(spec, mv1, np.float64)))
            # the update on the gradient the kernel applied, with the hyper-parameters the kernel was given (fp32: 1 - 0.999f is
            # 1.3e-5 away from 0.001, which is a property of the inputs, not of the arithmetic)
            g = ts["grads"]
            hp = {k: np.float32(v) for k, v in opt.items() if k != "kind"}
            if opt["kind"] == "adam":
                w, r1, r2, b1p, b2p = OO.adam_update(pf, s1, s2, g, np.float32(lr), powers[0], powers[1], hp["beta1"], hp["beta2"],
                                                    hp["epsilon"])
                powers = (np.float32(powers[0] * hp["beta1"]), np.float32(powers[1] * hp["beta2"]))
                err["powers"] = max(rel_err(powers[0], b1p), rel_err(powers[1], b2p))
            else:
                w, r1, r2 = OO.rmsprop_update(pf, s1, s2, g, np.float32(lr), hp["decay"], hp["momentum"], hp["epsilon"])
            err.update(params=rel_err(ts["params"], w), slots=rel_err(ts["slots"], r1), slots2=rel_err(ts["slots2"], r2))
            assert err["grads"] <= TOL_GRADS and err["moving"] <= TOL_GRADS, (step, err)
            assert all(err[k] <= TOL_UPDATE for k in ("params", "slots", "slots2", "powers") if k in err), (step, err)
            assert np.all(np.isfinite(ts["params"]))
            assert not np.array_equal(ts["params"], pf)
            for k, v in err.items():
                worst[k] = max(worst.get(k, 0.0), v)
            pf, s1, s2, mf = ts["params"], ts["slots"], ts["slots2"], ts["moving"]
        return worst
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------- oracle pins (CPU)
def test_adam_first_step_is_lr_times_sign_of_the_gradient():
    rng = np.random.default_rng(0)
    g = rng.standard_normal(1000) * np.logspace(-4, 1, 1000)
    w = rng.standard_normal(1000)
    lr, eps = 1e-3, 1e-8
    w1, m, v, b1p, b2p = OO.adam_update(w, np.zeros(1000), np.zeros(1000), g, lr, 0.9, 0.999, epsilon=eps)
    # m = 0.1 g, v = 0.001 g^2, alpha = lr sqrt(0.001) / 0.1: the step is lr g / (|g| + eps / sqrt(0.001)) = lr sign(g) (1 - O(eps/|g|))
    assert np.all(np.abs((w - w1) - lr * np.sign(g)) <= lr * (eps / np.sqrt(1e-3)) / np.abs(g) + 1e-15)
    assert np.allclose(m, 0.1 * g, rtol=1e-15) and np.allclose(v, 1e-3 * g * g, rtol=1e-14)
    assert b1p == 0.9 * 0.9 and b2p == 0.999 * 0.999


def test_rmsprop_first_step_closed_form():
    rng = np.random.default_rng(1)
    g = rng.standard_normal(500) * 3.0
    w = rng.standard_normal(500)
    lr, rho, eps = 1e-2, 0.9, 1e-10
    w1, ms, mom = OO.rmsprop_update(w, np.ones(500), np.zeros(500), g, lr, rho, 0.0, eps)
    expect = lr * g / np.sqrt(rho + (1 - rho) * g * g + eps)
    np.testing.assert_allclose(mom, expect, rtol=1e-13, atol=0)
    np.testing.assert_allclose(w - w1, expect, rtol=0, atol=1e-15)          # w -= mom (up to the rounding of w)
    np.testing.assert_allclose(ms, rho + (1 - rho) * g * g, rtol=1e-15)
    # with momentum the accumulator carries over
    _, _, mom2 = OO.rmsprop_update(w1, ms, mom, g, lr, rho, 0.5, eps)
    np.testing.assert_allclose(mom2, 0.5 * mom + lr * g / np.sqrt(ms + (1 - rho) * (g * g - ms) + eps), rtol=1e-13)


def test_adam_powers_advance_by_one_fp32_multiply_per_submitted_step():
    """AudioNetModel keeps beta1_power / beta2_power as np.float32 and multiplies once per submitted step (TF's in-graph
    assign(beta1_power * beta1)); no engine is needed for the bookkeeping."""
    import argparse
    from tcresnet_b200.factory import audio_nets
    model = audio_nets.TCResNet8Model(argparse.Namespace(learning_rate=1e-3), None)
    model.set_optimizer(dict(ADAM))
    b1, b2 = np.float32(0.9), np.float32(0.999)
    assert model.beta1_power == b1 and model.beta2_power == b2
    e1, e2 = b1, b2
    for k in range(1, 40):
        model._advance_optimizer()
        e1, e2 = np.float32(e1 * b1), np.float32(e2 * b2)
        assert model.beta1_power.dtype == np.float32 and model.beta1_power == e1 and model.beta2_power == e2, k
        assert model._step_optimizer()["beta1_power"] == e1
    model.set_optimizer(dict(RMSPROP))
    assert model.beta1_power is None and "beta1_power" not in model._step_optimizer()


# ---------------------------------------------------------------------------------------------------- emulator (CPU)
@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


@pytest.mark.parametrize("opt", [ADAM, RMSPROP, RMSPROP_MOM], ids=["adam", "rmsprop", "rmsprop-momentum"])
def test_emulated_update_matches_oracle_on_the_applied_gradient(emu, opt):
    worst = run_optimizer_case(emu, opt, n=8, steps=3)
    print(opt["kind"], worst)


@pytest.mark.parametrize("mode", ["0", "1", "3"])
def test_emulated_resident_modes_and_gradient_only_steps(emu, monkeypatch, mode):
    """TCR_RESIDENT = 0, 1 and 3 (the default) all end in the same update launch: one Adam and one RMSProp step meet the bounds, and apply_update = 0
    computes the gradient but leaves the parameters, both slots and the moving statistics untouched, bit for bit."""
    monkeypatch.setenv("TCR_RESIDENT", mode)
    for opt in (ADAM, RMSPROP):
        run_optimizer_case(emu, opt, n=7, steps=1)
    spec = O.build_spec("TCResNet8", 1.0, 49)
    eng = Engine(emu, max_batch=8)
    try:
        params, moving = perturbed_variables(spec)
        pf, mf = O.flatten_vars(spec, params), O.flatten_moving(spec, moving)
        wav, onehot = O.synthetic_batch(7)
        rng = np.random.RandomState(2)
        s1, s2 = rng.rand(pf.size).astype(np.float32) + 0.5, 0.01 * rng.randn(pf.size).astype(np.float32)
        for opt, powers in ((ADAM, (np.float32(0.729), np.float32(0.997))), (RMSPROP, (None, None))):
            ts = opt_step(eng, wav, onehot, pf, s1, s2, mf, opt, powers, apply_update=False)
            for k, before in (("params", pf), ("slots", s1), ("slots2", s2), ("moving", mf)):
                assert np.array_equal(ts[k], before), (opt["kind"], k)
            assert np.all(np.isfinite(ts["grads"])) and np.abs(ts["grads"]).max() > 0
    finally:
        eng.close()


def test_step_args_rejections(emu):
    """TCR_ERR_INVALID for an unknown optimizer kind, Adam / RMSProp with apply_update and no slots2, and beta1_power == 1."""
    eng = Engine(emu, max_batch=4)
    try:
        b = emu
        num = eng.info.num_trainable
        spec = O.build_spec("TCResNet8", 1.0, 49)
        pv, mv = O.init_variables(spec, 0)
        wav, onehot = O.synthetic_batch(2)
        bufs = [b.upload(x) for x in (wav, onehot, O.flatten_vars(spec, pv), np.zeros(num), np.zeros(num), O.flatten_moving(spec, mv))]

        def call(**kw):
            a = L.TcrStepArgs()
            a.input, a.onehot, a.n = b.ptr(bufs[0]), b.ptr(bufs[1]), 2
            a.params, a.slots, a.slots2, a.moving = b.ptr(bufs[2]), b.ptr(bufs[3]), b.ptr(bufs[4]), b.ptr(bufs[5])
            a.learning_rate, a.apply_update = 1e-3, 1
            a.optimizer, a.beta1, a.beta2, a.epsilon, a.beta1_power, a.beta2_power = L.TCR_OPT_ADAM, 0.9, 0.999, 1e-8, 0.9, 0.999
            for k, v in kw.items():
                setattr(a, k, v)
            return eng.lib.tcr_train_step(eng.h, C.byref(a), None), eng.lib.tcr_last_error().decode()

        assert call()[0] == 0                                    # a valid Adam step: TCR_OK
        for kind in (3, -1, 99):
            rc, msg = call(optimizer=kind)
            assert rc == 1 and "unknown optimizer" in msg, (kind, rc, msg)
        for kind in (L.TCR_OPT_ADAM, L.TCR_OPT_RMSPROP):
            rc, msg = call(optimizer=kind, slots2=None)
            assert rc == 1 and "slots2" in msg, (kind, rc, msg)
            assert call(optimizer=kind, slots2=None, apply_update=0)[0] == 0     # gradients only: no state needed
        rc, msg = call(beta1_power=1.0)
        assert rc == 1 and "beta1_power" in msg, msg
        assert call(optimizer=L.TCR_OPT_MOMENTUM, slots2=None, beta1_power=1.0)[0] == 0   # the momentum step ignores the new fields
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------- trainer (CPU)
def _trainer():
    from tcresnet_b200.common import utils
    from tcresnet_b200.helper.trainer import TrainerBase
    t = TrainerBase.__new__(TrainerBase)
    t.log = utils.get_logger("test_optimizers")
    return t


def test_build_optimizer_maps_the_reference_flags():
    t = _trainer()
    assert t.build_optimizer("adam", None) == dict(kind="adam", beta1=0.9, beta2=0.999, epsilon=1e-8)
    assert t.build_optimizer("adam", None, epsilon=1e-4) == dict(kind="adam", beta1=0.9, beta2=0.999, epsilon=1e-4)
    assert t.build_optimizer("adam", None, momentum=0.0, decay=0.0) == dict(kind="adam", beta1=0.9, beta2=0.999, epsilon=1e-8)
    assert t.build_optimizer("rmsprop", None) == dict(kind="rmsprop", decay=0.9, momentum=0.0, epsilon=1e-10)
    assert t.build_optimizer("rmsprop", None, momentum=0.5, decay=0.95, epsilon=1e-6) == \
        dict(kind="rmsprop", decay=0.95, momentum=0.5, epsilon=1e-6)
    assert t.build_optimizer("mom", None, momentum=0.9) == dict(kind="mom", momentum=0.9)        # unchanged
    assert t.build_optimizer("gd", None) == dict(kind="gd", momentum=0.0)
    with pytest.raises(TypeError, match="momentum"):
        t.build_optimizer("adam", None, momentum=0.9)
    with pytest.raises(TypeError, match="optimizer_decay"):
        t.build_optimizer("adam", None, decay=0.9)


def test_reference_default_optimizer_is_adam():
    from tcresnet_b200 import train_audio
    line = ("--dataset_path synthetic:64 --dataset_split_name train --output_name output/softmax --num_classes 12 --train_dir /tmp/x "
            "--augmentation_method anchored_slice_or_pad --preprocess_method mfcc --num_mfccs 40 --batch_size 8 TCResNet8Model "
            "--weight_decay 0.001")
    a = train_audio.parse_arguments(shlex.split(line))
    assert a.optimizer == "adam"
    opt = _trainer().build_optimizer(a.optimizer, None, momentum=a.momentum, decay=a.optimizer_decay, epsilon=a.optimizer_epsilon)
    assert opt["kind"] == "adam" and opt["epsilon"] == 1e-8
    bad = train_audio.parse_arguments(shlex.split(line.replace("--batch_size 8", "--batch_size 8 --momentum 0.9")))
    with pytest.raises(TypeError):
        _trainer().build_optimizer(bad.optimizer, None, momentum=bad.momentum, decay=bad.optimizer_decay, epsilon=bad.optimizer_epsilon)


# ---------------------------------------------------------------------------------------------------- checkpoints (CPU)
def _cpu_model(kind, seed):
    """AudioNetModel over CPU tensors: get_variables / set_variables need only the engine's parameter table."""
    import argparse
    import torch
    from tcresnet_b200.engine import Engine as PublicEngine
    from tcresnet_b200.factory import audio_nets
    spec = O.build_spec("TCResNet8", 1.0, 49)
    eng = PublicEngine.__new__(PublicEngine)
    table, off = [], 0
    for name in spec.var_names:
        numel = int(np.prod(spec.var_shapes[name]))
        table.append(dict(name=name, trainable=True, shape=tuple(spec.var_shapes[name]), offset=off, numel=numel))
        off += numel
    eng.num_trainable, moff = off, 0
    for name in O.moving_names(spec):
        c = int(np.prod(spec.var_shapes[name.split("/BatchNorm/")[0] + "/weights"][3:]))
        table.append(dict(name=name, trainable=False, shape=(c,), offset=moff, numel=c))
        moff += c
    eng.table, eng.num_moving, eng.device = table, moff, torch.device("cpu")
    model = audio_nets.TCResNet8Model(argparse.Namespace(), None)
    model.engine = eng
    g = torch.Generator().manual_seed(seed)
    model.params, model.moving = torch.randn(off, generator=g), torch.randn(moff, generator=g)
    model.set_optimizer(dict(ADAM) if kind == "adam" else dict(RMSPROP))
    model.slots.copy_(torch.randn(off, generator=g))
    model.slots2.copy_(torch.rand(off, generator=g))
    if kind == "adam":
        for _ in range(seed % 7 + 1):
            model._advance_optimizer()
    return model, spec


@pytest.mark.parametrize("fmt", ["tf", "npz"])
@pytest.mark.parametrize("kind", ["adam", "rmsprop"])
def test_optimizer_state_round_trips_through_checkpoints(tmp_path, kind, fmt):
    from tcresnet_b200.common import checkpoint as ckpt
    model, spec = _cpu_model(kind, 5)
    values = model.get_variables()
    first, second = ("Adam", "Adam_1") if kind == "adam" else ("RMSProp", "RMSProp_1")
    for v in spec.var_names:
        assert f"{v}/{first}" in values and f"{v}/{second}" in values and f"{v}/Momentum" not in values
    if kind == "adam":
        assert np.asarray(values["beta1_power"]).dtype == np.float32 and values["beta1_power"] == model.beta1_power
        assert np.asarray(values["beta2_power"]).dtype == np.float32 and values["beta2_power"] == model.beta2_power
    else:
        assert "beta1_power" not in values and "beta2_power" not in values
    path = ckpt.save(tmp_path, "TCResNet8Model", 17, values, fmt=fmt)
    back = ckpt.load(path)
    names = {f"{v}/{s}" for v in spec.var_names for s in (first, second)} | ({"beta1_power", "beta2_power"} if kind == "adam" else set())
    assert names <= set(back) and int(back["global_step"]) == 17
    fresh, _ = _cpu_model(kind, 11)
    fresh.set_variables(back)
    for attr in ("params", "moving", "slots", "slots2"):
        assert np.array_equal(getattr(fresh, attr).numpy(), getattr(model, attr).numpy()), attr
    if kind == "adam":
        assert fresh.beta1_power == model.beta1_power and fresh.beta2_power == model.beta2_power
        assert fresh.beta1_power.dtype == np.float32 and fresh.beta1_power != np.float32(0.9)
    # slots and powers are optional on restore: a momentum-era checkpoint leaves them as they are
    plain = {k: v for k, v in back.items() if "/" + first not in k and "/" + second not in k and "_power" not in k}
    other, _ = _cpu_model(kind, 3)
    s_before, p_before = other.slots.clone(), other.beta1_power
    other.set_variables(plain)
    assert np.array_equal(other.slots.numpy(), s_before.numpy()) and other.beta1_power == p_before
    assert np.array_equal(other.params.numpy(), model.params.numpy())


# ---------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


@pytest.mark.gpu
@pytest.mark.parametrize("opt", [ADAM, RMSPROP, RMSPROP_MOM], ids=["adam", "rmsprop", "rmsprop-momentum"])
def test_cuda_update_matches_oracle_n8(cuda, opt):
    print(run_optimizer_case(cuda, opt, n=8, steps=3))


@pytest.mark.gpu
@pytest.mark.parametrize("opt", [ADAM, RMSPROP], ids=["adam", "rmsprop"])
def test_cuda_update_matches_oracle_tcresnet8_n512(cuda, opt):
    print(run_optimizer_case(cuda, opt, n=512, steps=2, max_batch=512))


@pytest.mark.gpu
@pytest.mark.parametrize("opt", [ADAM, RMSPROP], ids=["adam", "rmsprop"])
def test_cuda_update_matches_oracle_tcresnet14x15_n1024(cuda, opt):
    print(run_optimizer_case(cuda, opt, model="TCResNet14", wm=1.5, n=1024, steps=1, max_batch=1024))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["0", "1", "3"])
def test_cuda_resident_modes(cuda, monkeypatch, mode):
    monkeypatch.setenv("TCR_RESIDENT", mode)
    run_optimizer_case(cuda, ADAM, n=64, steps=2)
    run_optimizer_case(cuda, RMSPROP, n=64, steps=1)


@pytest.mark.gpu
def test_adam_step_is_bitwise_deterministic(cuda):
    spec = O.build_spec("TCResNet8", 1.0, 49)
    params, moving = perturbed_variables(spec)
    pf, mf = O.flatten_vars(spec, params), O.flatten_moving(spec, moving)
    wav, onehot = O.synthetic_batch(300)
    eng = Engine(cuda, max_batch=300, dropout_keep_prob=0.5)
    rng = np.random.RandomState(4)
    s1, s2 = 0.01 * rng.randn(pf.size).astype(np.float32), 1e-4 * rng.rand(pf.size).astype(np.float32)
    powers = (np.float32(0.9 ** 5), np.float32(0.999 ** 5))
    a = opt_step(eng, wav, onehot, pf, s1, s2, mf, ADAM, powers, seed=11)
    b = opt_step(eng, wav, onehot, pf, s1, s2, mf, ADAM, powers, seed=11)
    for k in ("grads", "params", "slots", "slots2", "moving", "losses"):
        assert np.array_equal(a[k], b[k]), k
    eng.close()


def _model(opt, feed_lag, batches, batch=32, seed=0):
    """TCResNet8Model on the CUDA engine, driven through AudioNetModel.execute (the trainer's session.run(train_op)) over a fixed
    list of batches."""
    import argparse
    from tcresnet_b200.factory import audio_nets

    class Batches:
        def __init__(self):
            self.i = 0

        def next_batch(self):
            wav, hot = batches[self.i % len(batches)]
            self.i += 1
            return wav, hot

    args = argparse.Namespace(width_multiplier=1.0, num_classes=12, sample_rate=16000, clip_duration_ms=1000, window_size_ms=40.0,
                              window_stride_ms=20.0, num_mel_bins=64, num_mfccs=40, lower_edge_hertz=80.0, upper_edge_hertz=7600.0,
                              preprocess_method="mfcc", batch_size=batch, input_batch_size=1, dropout_keep_prob=0.5,
                              weight_decay=1e-3, learning_rate=2e-3, feed_lag=feed_lag, seed=seed)
    model = audio_nets.TCResNet8Model(args, Batches())
    model.build_inference(None, is_training=True)
    model.is_training = True
    model.set_optimizer(dict(opt))
    return model


def _state(model):
    import torch
    model.flush_feed()
    torch.cuda.synchronize()
    return dict(params=model.params.cpu().numpy(), slots=model.slots.cpu().numpy(), slots2=model.slots2.cpu().numpy(),
                moving=model.moving.cpu().numpy(), b1=model.beta1_power, b2=model.beta2_power)


def _batches(k, n=32, seed=5):
    out = []
    for i in range(k):
        wav, hot = O.synthetic_batch(n, seed_wav=seed + i, seed_label=seed + 100 + i)
        out.append((wav.reshape(n, 16000, 1), hot))
    return out


def _assert_same_state(a, b):
    for k in a:
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("opt", [ADAM, RMSPROP], ids=["adam", "rmsprop"])
def test_host_feed_lag2_equals_synchronous_steps(cuda, opt):
    """feed_lag 2 (tcr_train_step_host through HostFeed, the powers captured per submitted call) leaves the same parameters, slots,
    moving statistics and powers as the same steps through Engine.train_step, bit for bit."""
    batches = _batches(3)
    states = []
    for lag in (0, 2):
        m = _model(opt, lag, batches)
        for _ in range(7):
            m.execute({"train_op", "global_step", "total_loss", "model_loss"}, None)
        states.append(_state(m))
        m.engine.close()
    _assert_same_state(*states)
    if opt["kind"] == "adam":                         # beta1 times 7 fp32 multiplies, one per submitted step
        b1 = np.float32(0.9)
        for _ in range(7):
            b1 = np.float32(b1 * np.float32(0.9))
        assert states[0]["b1"] == b1


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["tf", "npz"])
@pytest.mark.parametrize("opt", [ADAM, RMSPROP], ids=["adam", "rmsprop"])
def test_resume_from_checkpoint_is_bitwise_uninterrupted(cuda, tmp_path, opt, fmt):
    """k steps, checkpoint, restore into a fresh model (different initial weights), one more step == k + 1 uninterrupted steps."""
    from tcresnet_b200.common import checkpoint as ckpt
    batches, k = _batches(4), 3
    fetch = {"train_op", "global_step", "total_loss", "model_loss"}
    ref = _model(opt, 2, batches)
    for _ in range(k + 1):
        ref.execute(fetch, None)
    expect = _state(ref)
    ref.engine.close()
    first = _model(opt, 2, batches)
    for _ in range(k):
        first.execute(fetch, None)
    path = ckpt.save(tmp_path, "TCResNet8Model", first.global_step, first.get_variables(), fmt=fmt)
    first.engine.close()
    values = ckpt.load(path)
    resumed = _model(opt, 2, batches, seed=9)
    resumed.dataset.i = k
    resumed.set_variables(values)
    resumed.global_step = ckpt.checkpoint_step(path)                      # what the trainer does on restore
    resumed.execute(fetch, None)
    _assert_same_state(_state(resumed), expect)
    resumed.engine.close()


@pytest.mark.gpu
@pytest.mark.parametrize("optimizer", ["adam", "rmsprop"])
def test_train_then_evaluate_with_optimizer(tmp_path, optimizer):
    from tcresnet_b200 import evaluate_audio, train_audio
    from tcresnet_b200.common import checkpoint as ckpt
    common = ("--dataset_path synthetic:96 --output_name output/softmax --num_classes 12 --preprocess_method mfcc "
              "--num_mfccs 40 --clip_duration_ms 1000 --window_size_ms 30 --window_stride_ms 10 ")
    extra = "--optimizer_epsilon 1e-6 " if optimizer == "adam" else "--optimizer_decay 0.95 --momentum 0.5 "
    train_args = train_audio.parse_arguments(shlex.split(
        common + f"--dataset_split_name train --train_dir {tmp_path} --augmentation_method anchored_slice_or_pad_with_shift "
        "--batch_size 32 --boundaries 10 20 --max_step_from_restore 12 --lr_list 0.001 0.0005 0.0001 --absolute_schedule "
        f"--no-boundaries_epoch --step_save_checkpoint 6 --step_evaluation 6 --optimizer {optimizer} {extra}"
        "TCResNet8Model --weight_decay 0.001 --width_multiplier 1.0"))
    trainer = train_audio.train(train_args)
    assert trainer.model.global_step == 12 and np.isfinite(trainer.model._feed_last[1])
    saved = ckpt.latest_checkpoint(tmp_path)
    assert saved is not None and ckpt.checkpoint_step(saved) == 12
    values = ckpt.load(saved)
    slot = "Adam" if optimizer == "adam" else "RMSProp"
    assert f"TCResNet8/fc/weights/{slot}" in values and f"TCResNet8/fc/weights/{slot}_1" in values
    assert "TCResNet8/fc/weights/Momentum" not in values
    if optimizer == "adam":
        # 12 submitted steps: beta^13 as 12 fp32 multiplies of beta
        b1 = np.float32(0.9)
        for _ in range(12):
            b1 = np.float32(b1 * np.float32(0.9))
        assert np.float32(values["beta1_power"]) == b1 and "beta2_power" in values
    else:
        assert np.abs(values[f"TCResNet8/fc/weights/{slot}_1"]).max() > 0
    eval_args = evaluate_audio.parse_arguments(shlex.split(
        common + f"--dataset_split_name valid --checkpoint_path {tmp_path} --augmentation_method anchored_slice_or_pad "
        "--batch_size 3 --no-shuffle --valid_type once TCResNet8Model --weight_decay 0.001 --width_multiplier 1.0"))
    results = evaluate_audio.main(eval_args)
    assert len(results) == 1 and 0.0 <= results[0]["accuracy"] <= 1.0 and np.isfinite(results[0]["total_loss"])
