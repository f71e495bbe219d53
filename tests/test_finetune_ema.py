"""Partial training (--trainable_scopes, tcr_set_trainable) and the weight EMA (--use_ema, tcr_step_args::ema) on the fused step.

The subset step is checked against the full step taken from the SAME pre-step state: the gradients, parameters and slots of the
trained variables, the BatchNorm moving statistics and both losses must be bit-identical (the subset step only skips work),
the frozen variables' gradients are 0 and their parameters and slots are untouched.  The shadow is compared with an fp64
restatement of s -= (s - w)(1 - d) on the step's own updated parameters.
"""
import argparse
import ctypes as C
import shlex

import numpy as np
import pytest

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L
from tcresnet_b200.common import model_loader as ML
from oracle import tcr_oracle as O
from parity_cases import cuda_relu_masks, perturbed_variables
from tcr_harness import Engine, NumpyBackend, launched, rel_err

ADAM = dict(kind="adam", beta1=0.9, beta2=0.999, epsilon=1e-8)
MOM = dict(kind="mom", momentum=0.9)
# head only (no backward-data chain), lowest trained conv = a conv_a (odd depth), conv_b / shortcut convs (even depth: the chain stops
# after phase (2) of the block above), conv0 with (bn, conv0) and without (bn) its weights, everything
SETS = {"head": "{m}/fc", "block2": "{m}/block2", "convb1": "{m}/block1/conv1_1", "down": ".*down", "bn": ".*BatchNorm",
        "conv0": "{m}/conv0", "all": ""}


@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


def trainable_names(eng):
    return [d["name"] for d in eng.param_table() if d["kind"] < 3]


def flags_for(eng, scope, model):
    names = trainable_names(eng)
    picked = set(ML.variables_to_train(scope.format(m=model), names))
    return np.array([n in picked for n in names], np.int32), names


def set_trainable(eng, flags):
    if flags is None:
        return eng.lib.tcr_set_trainable(eng.h, None, 0)
    arr = (C.c_int32 * len(flags))(*[int(x) for x in flags])
    return eng.lib.tcr_set_trainable(eng.h, arr, len(flags))


def entry_mask(eng, flags):
    """Per-parameter bool mask [num_trainable] of the trained entries."""
    m = np.zeros(eng.info.num_trainable, bool)
    for d, f in zip([d for d in eng.param_table() if d["kind"] < 3], flags):
        m[d["offset"]:d["offset"] + d["numel"]] = bool(f)
    return m


class Run:
    """Device-resident state of a training run through the C ABI (slots2 only for Adam, ema optional)."""

    def __init__(self, eng, feat, onehot, params, moving, opt, ema_decay=None, mask=None):
        b = self.b = eng.b
        self.eng, self.opt, self.ema_decay = eng, opt, ema_decay
        num = eng.info.num_trainable
        self.inp, self.hot = b.upload(feat), b.upload(onehot)
        self.mask = b.upload(mask) if mask is not None else None
        self.n = feat.shape[0]
        self.state = dict(params=b.upload(params), slots=b.upload(np.zeros(num, np.float32)), moving=b.upload(moving))
        if opt["kind"] == "adam":
            self.state["slots2"] = b.upload(np.zeros(num, np.float32))
        if ema_decay is not None:
            self.state["ema"] = b.upload(params)
        self.powers = (np.float32(0.9), np.float32(0.999))

    def snapshot(self):
        return {k: self.b.download(v) for k, v in self.state.items()}

    def step(self, seed, state=None, eng=None):
        """One step on `state` (default: the run's own buffers) with handle `eng` (default: the run's), returns the downloaded
        outputs."""
        b, eng = self.b, eng or self.eng
        st = self.state if state is None else state
        losses, grads = b.empty(2), b.empty(eng.info.num_trainable)
        a = L.TcrStepArgs()
        a.input, a.input_is_features, a.onehot, a.n = b.ptr(self.inp), L.TCR_INPUT_FEATURES, b.ptr(self.hot), self.n
        a.params, a.slots, a.moving = b.ptr(st["params"]), b.ptr(st["slots"]), b.ptr(st["moving"])
        a.learning_rate, a.weight_decay, a.dropout_seed, a.dropout_mask = 1e-2, 1e-3, seed, b.ptr(self.mask)
        a.losses, a.grads, a.apply_update = b.ptr(losses), b.ptr(grads), 1
        if self.opt["kind"] == "adam":
            a.optimizer, a.slots2, a.beta1, a.beta2, a.epsilon = L.TCR_OPT_ADAM, b.ptr(st["slots2"]), 0.9, 0.999, 1e-8
            a.beta1_power, a.beta2_power = self.powers
        else:
            a.momentum = 0.9
        if "ema" in st:
            a.ema, a.ema_decay = b.ptr(st["ema"]), self.ema_decay
        L.check(eng.lib, eng.lib.tcr_train_step(eng.h, C.byref(a), b.stream), "tcr_train_step")
        b.sync()
        out = {k: b.download(v) for k, v in st.items()}
        out.update(grads=b.download(grads), losses=b.download(losses))
        return out

    def advance(self):
        self.powers = (np.float32(self.powers[0] * np.float32(0.9)), np.float32(self.powers[1] * np.float32(0.999)))


def poison(eng, spec):
    """NaN into the backward intermediates a step may read from an earlier call of the same handle: every layer's masked gradient
    (g:<conv>, g:<block>) and published BatchNorm-backward sums (bsum:<conv>).  A step that skips work it needs then shows NaN."""
    names = [f"g:{cv.name}" for cv in spec.convs()] + [f"bsum:{cv.name}" for cv in spec.convs()]
    names += [f"g:block{b.index}" for b in spec.blocks]
    for name in names:
        p, numel = C.c_void_p(), C.c_int64()
        L.check(eng.lib, eng.lib.tcr_workspace_tensor(eng.h, name.encode(), C.byref(p), C.byref(numel)), name)
        if eng.b.name == "emu":
            C.memset(p.value, 0xFF, numel.value * 4)                     # 0xFFFFFFFF is a NaN
        else:
            rt = C.CDLL("libcudart.so.12")
            rt.cudaMemset.argtypes = [C.c_void_p, C.c_int, C.c_size_t]
            assert rt.cudaMemset(p.value, 0xFF, numel.value * 4) == 0
            eng.b.sync()


def subset_equals_full(backend, model, wm, n, opt, sets, steps=2, max_batch=None):
    """For each trainable set: `steps` subset steps; before each, the full step from the same pre-step state on a SEPARATE handle
    is the reference.  The subset handle's backward intermediates are poisoned before each of its steps, so whatever it reads
    must have been computed by that step."""
    spec = O.build_spec(model, wm, 49)
    cfg = dict(model=int(model[len("TCResNet"):]), width_multiplier=wm, max_batch=max_batch or max(n, 8), dropout_keep_prob=0.5)
    eng, ref = Engine(backend, **cfg), Engine(backend, **cfg)
    try:
        params, moving = perturbed_variables(spec)
        pf, mf = O.flatten_vars(spec, params), O.flatten_moving(spec, moving)
        wav, onehot = O.synthetic_batch(n, adversarial=True)
        feat = O.mfcc(wav, 640, 320).astype(np.float32)
        mask = (np.random.RandomState(3).rand(n, spec.c_last) < 0.5).astype(np.float32)
        for name in sets:
            flags, _ = flags_for(eng, SETS[name], model)
            tm = entry_mask(eng, flags)
            assert set_trainable(eng, flags) == 0
            run = Run(eng, feat, onehot, pf, mf, opt, mask=mask)
            for step in range(steps):
                before = run.snapshot()
                full = run.step(step, {k: backend.upload(v) for k, v in before.items()}, eng=ref)
                poison(eng, spec)
                sub = run.step(step)
                run.advance()
                for k in ("params", "slots", "slots2"):
                    if k in sub:
                        assert np.array_equal(sub[k][tm], full[k][tm]), (name, step, k)
                        assert np.array_equal(sub[k][~tm], before[k][~tm]), (name, step, k, "frozen")
                assert np.array_equal(sub["grads"][tm], full["grads"][tm]), (name, step, "grads")
                assert not np.any(sub["grads"][~tm]), (name, step, "frozen grads")
                assert np.array_equal(sub["moving"], full["moving"]), (name, step, "moving")
                assert np.array_equal(sub["losses"], full["losses"]), (name, step, "losses")
                if name != "all":
                    assert not np.array_equal(sub["params"][tm], before["params"][tm]), (name, step, "trained params moved")
    finally:
        eng.close()
        ref.close()


def oracle_case(backend, model, wm, n, scope):
    """Trained entries of one subset step on a FRESH handle against the fp64 oracle with the CUDA path's ReLU decisions forced;
    frozen entries are 0."""
    spec = O.build_spec(model, wm, 49)
    eng = Engine(backend, model=int(model[len("TCResNet"):]), width_multiplier=wm, max_batch=max(n, 8), dropout_keep_prob=0.5)
    try:
        params, moving = perturbed_variables(spec)
        pf, mf = O.flatten_vars(spec, params), O.flatten_moving(spec, moving)
        wav, onehot = O.synthetic_batch(n, adversarial=True)
        feat = O.mfcc(wav, 640, 320)
        mask = (np.random.RandomState(3).rand(n, spec.c_last) < 0.5).astype(np.float32)
        flags, _ = flags_for(eng, scope, model)
        assert set_trainable(eng, flags) == 0
        tm = entry_mask(eng, flags)
        poison(eng, spec)
        out = Run(eng, feat.astype(np.float32), onehot, pf, mf, MOM, mask=mask).step(0)
        forced = cuda_relu_masks(eng, spec, n)
        _, _, _, ref = O.train_step(spec, O.unflatten_vars(spec, pf), O.unflatten_moving(spec, mf), O.zeros_like_vars(spec), feat,
                                    onehot, 1e-2, 0.9, 1e-3, 0.5, mask, forced_masks=forced)
        g = O.flatten_vars(spec, ref["grads"], np.float64)
        assert rel_err(out["grads"][tm], g[tm]) <= 1e-4, scope
        assert not np.any(out["grads"][~tm])
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------- scopes (CPU)
def _names8():
    spec = O.build_spec("TCResNet8", 1.0, 49)
    return list(spec.var_names)


def test_trainable_scopes_are_regexes_matched_on_the_variable_name_with_its_suffix():
    names = _names8()
    fc = ML.variables_to_train("TCResNet8/fc", names)
    assert fc == ["TCResNet8/fc/weights", "TCResNet8/fc2/weights"]            # re.match: fc2 starts with "TCResNet8/fc" too
    assert ML.variables_to_train("TCResNet8/fc/", names) == ["TCResNet8/fc/weights"]
    b2 = ML.variables_to_train("TCResNet8/block2", names)
    assert b2 and all(n.startswith("TCResNet8/block2/") for n in b2) and len(b2) == 9     # conv_a, conv_b, down: weights/beta/gamma
    bn = ML.variables_to_train(".*BatchNorm", names)
    assert bn == [n for n in names if "/BatchNorm/" in n] and len(bn) == 2 * 10
    with pytest.raises(ValueError, match="selects no"):
        ML.variables_to_train("BatchNorm", names)                                          # re.match is anchored at the start
    w = ML.variables_to_train(".*weights:0$", names)
    assert len(w) == 12 and all(n.endswith("/weights") for n in w)                         # the ":0" suffix is part of the name
    assert ML.variables_to_train("", names) == names
    # a scope that matches nothing next to one that does; whitespace around scopes is stripped
    assert ML.variables_to_train(" NoSuchNet/x , TCResNet8/conv0 ", names) == [n for n in names if n.startswith("TCResNet8/conv0/")]


def test_empty_and_overlapping_selections_raise():
    names = _names8()
    with pytest.raises(ValueError, match="selects no trainable variable"):
        ML.variables_to_train("TCResNet14/fc", names)
    with pytest.raises(ValueError, match="selected by both"):
        ML.variables_to_train("TCResNet8/block2,.*BatchNorm", names)
    with pytest.raises(ValueError, match="selected by both"):
        ML.variables_to_train("TCResNet8/fc,", names)                                      # the empty scope matches everything


def test_restore_filter_is_a_prefix_rule_covering_slots_and_shadows():
    keep = ML.restore_filter("", "TCResNet8/fc")
    for name in ("TCResNet8/fc/weights", "TCResNet8/fc/weights/Adam", "TCResNet8/fc/weights/ExponentialMovingAverage",
                 "TCResNet8/fc2/weights"):
        assert not keep(name), name
    assert keep("TCResNet8/conv0/weights/Adam_1") and keep("beta1_power") and keep("global_step")
    keep = ML.restore_filter("TCResNet8/block0, TCResNet8/conv0", "TCResNet8/block0/down")
    assert keep("TCResNet8/conv0/BatchNorm/moving_mean") and keep("TCResNet8/block0/conv0_0/weights/Momentum")
    assert not keep("TCResNet8/block0/down/weights") and not keep("TCResNet8/block1/conv1_0/weights") and not keep("beta1_power")
    assert ML.restore_filter(" , ", "")("anything")


def test_ema_restore_values_map_every_trainable_variable_to_its_shadow():
    names = ["N/a/weights", "N/b/weights"]
    vals = {"N/a/weights": 1, "N/a/weights/ExponentialMovingAverage": 2, "N/b/weights": 3, "N/c/BatchNorm/moving_mean": 4}
    out = ML.ema_restore_values(vals, names)
    assert out == {"N/a/weights": 2, "N/c/BatchNorm/moving_mean": 4}                       # b has no shadow: absent


def test_evaluator_rejects_use_ema_with_restore_scopes():
    from tcresnet_b200.helper.evaluator import Evaluator
    ev = Evaluator.__new__(Evaluator)
    ev.args = argparse.Namespace(use_ema=True, checkpoint_include_scopes="", checkpoint_exclude_scopes="TCResNet8/fc")
    with pytest.raises(ValueError, match="--use_ema cannot be combined"):
        ev.restore_values({})
    ev.args = argparse.Namespace(use_ema=False, checkpoint_include_scopes="", checkpoint_exclude_scopes="TCResNet8/fc")
    values, keep = ev.restore_values({"x": 1})
    assert values == {"x": 1} and not keep("TCResNet8/fc/weights") and keep("TCResNet8/conv0/weights")


def _cpu_model(seed, trained=None, ema=True):
    """AudioNetModel over CPU tensors (get_variables / set_variables need only the parameter table)."""
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
    eng.trained = set(trained) if trained is not None else set(spec.var_names)
    model = audio_nets.TCResNet8Model(argparse.Namespace(), None)
    model.engine = eng
    g = torch.Generator().manual_seed(seed)
    model.params, model.moving = torch.randn(off, generator=g), torch.randn(moff, generator=g)
    model.set_optimizer(dict(ADAM))
    model.slots.copy_(torch.randn(off, generator=g))
    model.slots2.copy_(torch.rand(off, generator=g))
    if ema:
        model.enable_ema(0.99)
        model.ema.copy_(torch.randn(off, generator=g))
    return model, spec


@pytest.mark.parametrize("fmt", ["tf", "npz"])
def test_shadows_and_a_partial_slot_set_round_trip_through_checkpoints(tmp_path, fmt):
    from tcresnet_b200.common import checkpoint as ckpt
    names = _names8()
    trained = ML.variables_to_train("TCResNet8/block2", names)
    model, spec = _cpu_model(5, trained)
    values = model.get_variables()
    for v in names:
        has = v in trained
        for suffix in ("Adam", "Adam_1", "ExponentialMovingAverage"):
            assert (f"{v}/{suffix}" in values) == has, (v, suffix)
        assert v in values
    path = ckpt.save(tmp_path, "TCResNet8Model", 3, values, fmt=fmt)
    back = ckpt.load(path)
    assert set(back) == set(values) | {"global_step"}
    fresh, _ = _cpu_model(11, trained)
    fresh.set_variables(back)
    tm = np.zeros(model.params.numel(), bool)
    for d in model.engine.table:
        if d["trainable"] and d["name"] in trained:
            tm[d["offset"]:d["offset"] + d["numel"]] = True
    for attr in ("params", "moving"):
        assert np.array_equal(getattr(fresh, attr).numpy(), getattr(model, attr).numpy()), attr
    for attr in ("slots", "slots2", "ema"):
        assert np.array_equal(getattr(fresh, attr).numpy()[tm], getattr(model, attr).numpy()[tm]), attr
    # shadows missing: an error, unless not strict (the shadow then keeps its value)
    plain = {k: v for k, v in back.items() if not k.endswith(ML.EMA_SUFFIX)}
    other, _ = _cpu_model(7, trained)
    with pytest.raises(KeyError, match="ExponentialMovingAverage"):
        other.set_variables(plain)
    before = other.ema.clone()
    other.set_variables(plain, strict=False)
    assert np.array_equal(other.ema.numpy(), before.numpy())
    # an excluded scope is neither restored nor required
    keep = ML.restore_filter("", "TCResNet8/block2")
    third, _ = _cpu_model(9, trained)
    p0 = third.params.clone()
    third.set_variables({k: v for k, v in back.items() if not k.startswith("TCResNet8/block2")}, restore=keep)
    assert np.array_equal(third.params.numpy()[tm], p0.numpy()[tm])
    assert np.array_equal(third.params.numpy()[~tm], model.params.numpy()[~tm])


# ---------------------------------------------------------------------------------------------------- emulator (CPU)
@pytest.mark.parametrize("mode", ["0", "1", "3"])
@pytest.mark.parametrize("opt", [ADAM, MOM], ids=["adam", "mom"])
def test_emulated_subset_step_equals_full_step_bitwise(emu, monkeypatch, mode, opt):
    monkeypatch.setenv("TCR_RESIDENT", mode)
    subset_equals_full(emu, "TCResNet8", 1.0, 8, opt, list(SETS))


@pytest.mark.parametrize("mode", ["0", "3"])
@pytest.mark.parametrize("name", ["block2", "convb1", "down", "bn", "conv0"])
def test_emulated_subset_gradients_match_the_oracle(emu, monkeypatch, mode, name):
    monkeypatch.setenv("TCR_RESIDENT", mode)
    oracle_case(emu, "TCResNet8", 1.0, 8, SETS[name])


def ema_case(backend, n, scope="{m}/block2", steps=3, decay=0.9, model="TCResNet8", opt=ADAM):
    spec = O.build_spec(model, 1.0, 49)
    eng = Engine(backend, model=int(model[len("TCResNet"):]), max_batch=max(n, 8), dropout_keep_prob=0.5)
    try:
        params, moving = perturbed_variables(spec)
        pf, mf = O.flatten_vars(spec, params), O.flatten_moving(spec, moving)
        wav, onehot = O.synthetic_batch(n)
        feat = O.mfcc(wav, 640, 320).astype(np.float32)
        flags, _ = flags_for(eng, scope, model)
        assert set_trainable(eng, flags) == 0
        tm = entry_mask(eng, flags)
        run = Run(eng, feat, onehot, pf, mf, opt, ema_decay=decay)
        s = pf.astype(np.float64)
        outs = []
        for step in range(steps):
            out = run.step(step)
            run.advance()
            s = s - (s - out["params"].astype(np.float64)) * (1.0 - np.float64(np.float32(decay)))
            assert rel_err(out["ema"][tm], s[tm]) <= 1e-6, step
            assert np.array_equal(out["ema"][~tm], pf[~tm]), step
            outs.append(out)
        assert not np.array_equal(outs[-1]["ema"][tm], pf[tm])
        return outs
    finally:
        eng.close()


def test_emulated_ema_follows_the_updated_weights(emu):
    ema_case(emu, 8)


def test_step_args_and_set_trainable_rejections(emu):
    eng = Engine(emu, max_batch=4)
    try:
        spec = O.build_spec("TCResNet8", 1.0, 49)
        pv, mv = O.init_variables(spec, 0)
        pf, mf = O.flatten_vars(spec, pv), O.flatten_moving(spec, mv)
        wav, onehot = O.synthetic_batch(2)
        run = Run(eng, O.mfcc(wav, 640, 320).astype(np.float32), onehot, pf, mf, ADAM, ema_decay=0.99)
        assert run.step(0)["ema"] is not None
        for bad in (1.5, -0.1, float("nan")):
            run.ema_decay = bad
            with pytest.raises(L.TcrError, match="ema_decay"):
                run.step(0)
        run.ema_decay = 1.0
        out = run.step(0)                                        # decay 1: the shadow stays where it is
        assert np.array_equal(out["ema"], run.snapshot()["ema"])
        rows = len(trainable_names(eng))
        assert set_trainable(eng, [1] * (rows - 1)) == 1 and "flags" in eng.lib.tcr_last_error().decode()
        assert set_trainable(eng, [0] * rows) == 1 and "no variable" in eng.lib.tcr_last_error().decode()
        assert set_trainable(eng, [1] * rows) == 0 and set_trainable(eng, None) == 0
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["0", "1", "3"])
def test_cuda_subset_step_equals_full_step_tcresnet8_n512(cuda, monkeypatch, mode):
    monkeypatch.setenv("TCR_RESIDENT", mode)
    for opt in (ADAM, MOM):
        subset_equals_full(cuda, "TCResNet8", 1.0, 512, opt, list(SETS), max_batch=512)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["0", "1", "3"])
def test_cuda_subset_step_equals_full_step_tcresnet14x15_n1024(cuda, monkeypatch, mode):
    monkeypatch.setenv("TCR_RESIDENT", mode)
    subset_equals_full(cuda, "TCResNet14", 1.5, 1024, ADAM, list(SETS), max_batch=1024)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["block2", "convb1", "down", "bn", "conv0"])
@pytest.mark.parametrize("model,wm,n,mode", [("TCResNet8", 1.0, 512, "0"), ("TCResNet8", 1.0, 512, "3"), ("TCResNet14", 1.5, 1024, "3")])
def test_cuda_subset_gradients_match_the_oracle(cuda, monkeypatch, model, wm, n, mode, name):
    monkeypatch.setenv("TCR_RESIDENT", mode)
    oracle_case(cuda, model, wm, n, SETS[name])


def _launches(cuda, mode, scope, monkeypatch, n=256):
    monkeypatch.setenv("TCR_RESIDENT", mode)
    spec = O.build_spec("TCResNet8", 1.0, 49)
    eng = Engine(cuda, max_batch=n, dropout_keep_prob=0.5)
    try:
        params, moving = perturbed_variables(spec)
        pf, mf = O.flatten_vars(spec, params), O.flatten_moving(spec, moving)
        wav, onehot = O.synthetic_batch(n)
        run = Run(eng, O.mfcc(wav, 640, 320).astype(np.float32), onehot, pf, mf, ADAM)
        run.step(0)                                                     # first launches set lazy attributes
        out = {"default": launched(cuda.lib, lambda: run.step(1))}
        if scope is not None:
            flags, _ = flags_for(eng, scope, "TCResNet8")
            assert set_trainable(eng, flags) == 0
            out["subset"] = launched(cuda.lib, lambda: run.step(2))
            assert set_trainable(eng, None) == 0
            out["back"] = launched(cuda.lib, lambda: run.step(3))
        return out
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["0", "1", "3"])
def test_cuda_launch_lists_follow_the_trainable_set(cuda, monkeypatch, mode):
    head = _launches(cuda, mode, "{m}/fc", monkeypatch)
    sub = head["subset"]
    assert not [k for k in sub if k == "resident_bwd_data" or k.startswith("dx:") or k == "dw_grouped"], sub
    assert sub["update"] == 1 and sub["grad_finalize"] == 1
    assert head["back"] == head["default"], (head["back"], head["default"])      # back to all: exactly the default list
    b2 = _launches(cuda, mode, "{m}/block2", monkeypatch)
    dx = lambda c: sum(v for k, v in c.items() if k.startswith("dx:"))          # noqa: E731
    if mode in ("0", "1"):
        assert 0 < dx(b2["subset"]) < dx(b2["default"]), b2
    else:
        assert b2["subset"]["resident_bwd_data"] == 1
    assert b2["subset"]["dw_grouped"] == 1


@pytest.mark.gpu
def test_cuda_subset_ema_step_is_bitwise_deterministic(cuda):
    a = ema_case(cuda, 300, steps=2)
    b = ema_case(cuda, 300, steps=2)
    for x, y in zip(a, b):
        for k in x:
            assert np.array_equal(x[k], y[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("mode,env,port", [("dp", {}, 29631), ("dp", {"TCR_P2P": "0"}, 29632), ("syncbn", {}, 29633)],
                         ids=["peer-memory", "nccl", "syncbn"])
def test_two_rank_finetune_with_ema_keeps_replicas_identical(mode, env, port):
    """Data-parallel block-2 fine-tune + EMA (tests/dist_finetune_worker.py): parameters, slots and shadows bit-identical on both
    ranks, frozen entries untouched; with either gradient exchange, and with SyncBN over the truncated backward-data chain."""
    import os
    import subprocess
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    here = os.path.dirname(os.path.abspath(__file__))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(here, "dist_finetune_worker.py"), mode]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=dict(os.environ, **env))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert f"finetune {mode}" in r.stdout and "bit-identical" in r.stdout, r.stdout[-500:]


@pytest.mark.gpu
def test_train_with_ema_then_finetune_the_head_and_evaluate_the_shadow(tmp_path):
    """The keyword-spotting recipe: train with --use_ema, fine-tune only fc from that checkpoint (fc excluded from the restore),
    evaluate the first checkpoint from its shadows."""
    import torch
    from tcresnet_b200 import evaluate_audio, train_audio
    from tcresnet_b200.common import checkpoint as ckpt
    common = ("--dataset_path synthetic:96 --output_name output/softmax --num_classes 12 --preprocess_method mfcc "
              "--num_mfccs 40 --clip_duration_ms 1000 --window_size_ms 40 --window_stride_ms 20 ")
    train = ("--dataset_split_name train --augmentation_method anchored_slice_or_pad_with_shift --batch_size 32 --boundaries 100 "
             "--lr_list 0.001 0.0005 --absolute_schedule --no-boundaries_epoch --step_save_checkpoint 100 --step_evaluation 100 "
             "--checkpoint_format tf ")
    net = " TCResNet8Model --weight_decay 0.001 --width_multiplier 1.0"
    d1, d2 = tmp_path / "pre", tmp_path / "ft"
    t1 = train_audio.train(train_audio.parse_arguments(shlex.split(
        common + train + f"--train_dir {d1} --max_step_from_restore 6 --use_ema --ema_decay 0.9" + net)))
    first = ckpt.latest_checkpoint(d1)
    v1 = ckpt.load(first)
    names = t1.model.engine.trainable_names
    assert all(n + ML.EMA_SUFFIX in v1 for n in names)
    assert not np.array_equal(v1["TCResNet8/fc/weights"], v1["TCResNet8/fc/weights" + ML.EMA_SUFFIX])
    t1.model.engine.close()
    t2 = train_audio.train(train_audio.parse_arguments(shlex.split(
        common + train + f"--train_dir {d2} --checkpoint_path {d1} --max_step_from_restore 4 --use_ema "
        "--trainable_scopes TCResNet8/fc --checkpoint_exclude_scopes TCResNet8/fc --ignore_missing_vars" + net)))
    v2 = ckpt.load(ckpt.latest_checkpoint(d2))
    head = {"TCResNet8/fc/weights", "TCResNet8/fc2/weights"}
    for n in names:
        if n not in head:
            assert np.array_equal(v2[n], v1[n]), n                                  # frozen: the restored value, bit for bit
    assert not np.array_equal(v2["TCResNet8/fc/weights"], v1["TCResNet8/fc/weights"])
    # what TF would write: slots and shadows for var_list only, the moving statistics of every layer, Adam's powers
    expect = set(names) | set(O.moving_names(O.build_spec("TCResNet8", 1.0, 49))) | {"beta1_power", "beta2_power", "global_step"}
    expect |= {f"{h}/{s}" for h in head for s in ("Adam", "Adam_1", "ExponentialMovingAverage")}
    assert set(v2) == expect, set(v2) ^ expect
    t2.model.engine.close()
    # evaluation from the shadows of the first checkpoint == a forward pass with the shadow weights
    ev_args = evaluate_audio.parse_arguments(shlex.split(
        common + f"--dataset_split_name valid --checkpoint_path {first} --augmentation_method anchored_slice_or_pad --batch_size 3 "
        "--no-shuffle --valid_type once --use_ema" + net))
    results = evaluate_audio.main(ev_args)
    assert len(results) == 1 and np.isfinite(results[0]["total_loss"])
    from tcresnet_b200.factory import audio_nets
    m = audio_nets.TCResNet8Model(ev_args, None)
    m.build_inference(None, is_training=False)
    m.set_variables(ML.ema_restore_values(v1, names))
    shadow = {n: v1[n + ML.EMA_SUFFIX] for n in names}
    shadow.update({k: v1[k] for k in v1 if "moving_" in k})
    p2, mv2 = torch.empty_like(m.params), torch.empty_like(m.moving)
    m.engine.variables_from_dict(shadow, p2, mv2)
    x = torch.from_numpy(O.synthetic_batch(3)[0].astype(np.float32)).to(m.engine.device)
    a = m.engine.forward(x, m.params, m.moving)["logits"].cpu().numpy()
    b = m.engine.forward(x, p2, mv2)["logits"].cpu().numpy()
    assert np.array_equal(a, b)
    m.engine.close()
