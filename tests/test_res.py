"""Honk's ResNets (Res8 / Res8Narrow / Res15 / Res15Narrow, audio_nets/res.py) on the DS-CNN handle, without a GPU: the parameter
table and FLOPs, the dilation schedule, the refusals, the oracle against torch, every kernel on the CPU emulator against the oracle
layer by layer and end to end (both residual modes: a forward_partial call that stops at a block's second conv writes a distinct
`out`, every earlier one the aliased buffer), and the CLI surface."""
import ctypes as C
import os
import shlex

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import res_oracle as R
from tcr_harness import NumpyBackend, rel_err

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TCR_ERR_INVALID, TCR_ERR_UNSUPPORTED = 1, 3           # include/tcr_b200.h

# (model, T, F): odd and even T and F, Res8 at its minimum 4 x 3 (a 1 x 1 pooled map), Res15 at maps smaller than its rates (every
# off-centre tap of the dilated convs reads padding) and one 98 x 40 case
GEOMETRY = [("Res8", 4, 3), ("Res8", 9, 6), ("Res8", 49, 10), ("Res8Narrow", 8, 5), ("Res8Narrow", 98, 40),
            ("Res15", 6, 3), ("Res15", 1, 1), ("Res15", 13, 8), ("Res15", 49, 10), ("Res15Narrow", 6, 3), ("Res15Narrow", 21, 17),
            ("Res15Narrow", 49, 10)]
# per model at 98 x 40 with 12 classes: trainable / moving values, FLOPs per utterance
COUNTS = {"Res8": (110295, 540, 792_683_280), "Res8Narrow": (19893, 228, 142_087_776), "Res15": (237870, 1170, 1_860_668_280),
          "Res15Narrow": (42636, 494, 332_479_176)}


@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


def create(lib, model, h, w, max_batch=4, classes=12, wm=0.0):
    handle = C.c_void_p()
    cfg = L.TcrDscnnConfig(ord(R.CODES.get(model, model)), h, w, classes, max_batch, 0, wm)
    return lib.tcr_dscnn_create(C.byref(cfg), C.byref(handle)), handle


def table(lib, handle):
    descs, count, nparams, flops = C.POINTER(L.TcrParamDesc)(), C.c_int32(), C.c_int64(), C.c_int64()
    L.check(lib, lib.tcr_dscnn_param_table(handle, C.byref(descs), C.byref(count), C.byref(nparams), C.byref(flops)), "table")
    rows = [(descs[i].name.decode(), tuple(descs[i].shape[:descs[i].rank]), L.KIND_NAMES[descs[i].kind]) for i in range(count.value)]
    return rows, nparams.value, flops.value


def _err(lib):
    return lib.tcr_last_error().decode()


@pytest.mark.parametrize("model", R.MODELS)
def test_parameter_table_and_flops(emu, model):
    rc, h = create(emu.lib, model, 98, 40)
    assert rc == 0, _err(emu.lib)
    try:
        rows, nparams, flops = table(emu.lib, h)
        spec = R.build_spec(model, 98, 40)
        shapes = spec.var_shapes
        assert [n for n, _, _ in rows] == spec.var_names
        assert [s for n, s, _ in rows] == [shapes[n] for n in spec.var_names]
        kinds = {"weights": "weight", "moving_mean": "moving_mean", "moving_variance": "moving_variance"}
        assert [k for _, _, k in rows] == [kinds[n.rsplit("/", 1)[1]] for n in spec.var_names]
        trainable = sum(int(np.prod(s)) for n, s, k in rows if k == "weight")
        assert (trainable, nparams - trainable, flops) == COUNTS[model]
        assert flops == R.forward_flops(spec)
        c = spec.c
        assert rows[:3] == [("Res/f_conv/weights", (3, 3, 1, c), "weight"), ("Res/conv0/Conv/weights", (3, 3, c, c), "weight"),
                            ("Res/conv1/Conv/weights", (3, 3, c, c), "weight")]
        assert rows[spec.layers + 1] == ("Res/fc/weights", (1, 1, c, 12), "weight")
        assert rows[spec.layers + 2:spec.layers + 4] == [("Res/conv0_bn/moving_mean", (c,), "moving_mean"),
                                                         ("Res/conv0_bn/moving_variance", (c,), "moving_variance")]
    finally:
        emu.lib.tcr_dscnn_destroy(h)


@pytest.mark.parametrize("model,T,Fq", GEOMETRY)
def test_flops_at_every_geometry(emu, model, T, Fq):
    rc, h = create(emu.lib, model, T, Fq, classes=7)
    assert rc == 0, _err(emu.lib)
    try:
        _, _, flops = table(emu.lib, h)
        assert flops == R.forward_flops(R.build_spec(model, T, Fq, 7))
    finally:
        emu.lib.tcr_dscnn_destroy(h)


def test_flops_and_schedule_by_hand():
    """Res15 at 98 x 40: f_conv 2 * 3920 * 9 * 45, 13 convs of 2 * 3920 * 9 * 45 * 45, fc 2 * 45 * 12; Res8's blocks run on 95 x 38."""
    assert R.forward_flops(R.build_spec("Res15")) == 3175200 + 13 * 142884000 + 1080
    assert R.block_map(R.build_spec("Res8")) == (95, 38) and R.block_map(R.build_spec("Res15")) == (98, 40)
    assert [R.build_spec("Res15").rate(k) for k in range(13)] == [1, 1, 1, 2, 2, 2, 4, 4, 4, 8, 8, 8, 16]
    assert [R.build_spec("Res15Narrow").rate(k) for k in range(13)] == [2 ** (k // 3) for k in range(13)]
    assert all(R.build_spec(m).rate(k) == 1 for m in ("Res8", "Res8Narrow") for k in range(6))


def test_refusals(emu):
    lib = emu.lib
    for model in ("Res8", "Res8Narrow"):
        for T, Fq in ((3, 40), (98, 2), (1, 1)):
            rc, h = create(lib, model, T, Fq)
            assert rc == TCR_ERR_UNSUPPORTED and not h.value, (model, T, Fq)
            assert f"Res8 / Res8Narrow need height >= 4 and width >= 3 (res_fconv's 4x3 / stride 1 average pool is VALID), got {T} x {Fq}" \
                in _err(lib)
    for model in R.MODELS:
        rc, h = create(lib, model, 98, 40, wm=1.0)
        assert rc == TCR_ERR_INVALID and "width_multiplier (1) applies to ResNet2D8 / ResNet2D8Pool only" in _err(lib), _err(lib)
    rc, h = create(lib, "Res15", 98, 300)                                    # a row past the register tiles of a CTA
    assert rc == TCR_ERR_UNSUPPORTED and "res_conv tiles whole rows of at most 256 positions; the blocks' map is 300 wide" in _err(lib)
    rc, h = create(lib, "Res15Narrow", 98, 600)
    assert rc == TCR_ERR_UNSUPPORTED and "at most 512 positions" in _err(lib), _err(lib)
    rc, h = create(lib, "Res8", 40000, 40, max_batch=2 ** 30)                # 39,997 pooled rows, 8 per f_conv CTA
    assert rc == TCR_ERR_UNSUPPORTED and "res_fconv: max_batch 1073741824 x 5000 row tiles exceeds the grid's 2147483647 CTAs" \
        in _err(lib), _err(lib)
    rc, h = create(lib, "Res15", 98, 40, max_batch=2 ** 27)                  # 13 f_conv CTAs per utterance fit, 17 conv tiles do not
    assert rc == TCR_ERR_UNSUPPORTED and "res_conv: max_batch 134217728 x 17 row tiles exceeds the 2147483647 tiles a launch walks" \
        in _err(lib), _err(lib)
    rc, h = create(lib, "Res15", 98, 40, classes=33)
    assert rc == TCR_ERR_INVALID and "bad DS-CNN configuration" in _err(lib)
    rc, h = create(lib, "Q", 98, 40)
    assert rc == TCR_ERR_INVALID and "'E' (Res8), 'N' (Res8Narrow), 'D' (Res15) or 'T' (Res15Narrow)" in _err(lib)
    for model, T, Fq in (("Res8", 4, 3), ("Res8Narrow", 4, 3), ("Res15", 1, 1), ("Res15", 998, 128), ("Res15Narrow", 2, 512)):
        rc, h = create(lib, model, T, Fq)                                    # accepted edges
        assert rc == 0, (model, T, Fq, _err(lib))
        lib.tcr_dscnn_destroy(h)
    rc, h = create(lib, "Res15", 98, 40)
    try:
        lis = C.c_void_p()
        assert lib.tcr_dscnn_listener_create(h, C.byref(L.TcrListenerConfig(1, 1, 320)), C.byref(lis)) == TCR_ERR_INVALID
        assert "no front-end" in _err(lib)
    finally:
        lib.tcr_dscnn_destroy(h)


@pytest.mark.parametrize("model,T,Fq", [("Res8", 98, 40), ("Res8Narrow", 9, 6), ("Res15", 20, 11), ("Res15Narrow", 6, 3)])
def test_oracle_matches_torch(model, T, Fq):
    spec = R.build_spec(model, T, Fq)
    p = R.init_variables(spec, 0)
    t = {k: torch.tensor(v) for k, v in p.items()}
    x = np.random.RandomState(1).randn(2, T, Fq)

    def conv(name, y, d=1):
        return F.relu(F.conv2d(y, t[f"Res/{name}/weights"].permute(3, 2, 0, 1), dilation=d, padding=d))

    def bn(k, y):
        b = f"Res/conv{k}_bn/"
        return F.batch_norm(y, t[b + "moving_mean"], t[b + "moving_variance"], None, None, False, 0.0, R.EPS)

    y = conv("f_conv", torch.tensor(x)[:, None])
    if spec.pool:
        y = F.avg_pool2d(y, (4, 3), stride=1)
    acts = [y]
    for i in range(spec.layers // 2):
        a = bn(2 * i, conv(f"conv{2 * i}/Conv", y, spec.rate(2 * i)))
        acts.append(a)
        y = bn(2 * i + 1, conv(f"conv{2 * i + 1}/Conv", a, spec.rate(2 * i + 1)) + y)
        acts.append(y)
    if spec.layers % 2:
        y = bn(12, conv("conv12/Conv", y, spec.rate(12)))
        acts.append(y)
    logits = y.mean((2, 3)) @ t["Res/fc/weights"][0, 0]
    got = R.forward_layers(spec, p, x)
    assert len(got) == len(acts) == spec.layers + 1
    for l, (a, r) in enumerate(zip(got, acts)):
        assert a.shape == (2,) + R.geometry(spec)[l]
        assert rel_err(a, r.permute(0, 2, 3, 1).numpy()) <= 1e-12, l
    assert rel_err(R.head(spec, p, got[-1]), logits.numpy()) <= 1e-12
    assert R.l2_loss(spec, p, 1e-5) == pytest.approx(1e-5 * sum(0.5 * float((v ** 2).sum()) for k, v in t.items() if k.endswith("/weights")))


class ResNet:
    """One Res8 / Res15 handle with the oracle's seeded variables on a tests/tcr_harness backend."""

    def __init__(self, b, model, T, Fq, max_batch, seed=0, classes=12):
        self.b, self.lib, self.model = b, b.lib, model
        self.spec = R.build_spec(model, T, Fq, classes)
        self.p = R.init_variables(self.spec, seed)
        rc, self.h = create(self.lib, model, T, Fq, max_batch, classes)
        L.check(self.lib, rc, "tcr_dscnn_create")
        self.params = b.upload(R.flatten(self.spec, self.p))

    def close(self):
        self.lib.tcr_dscnn_destroy(self.h)

    def forward(self, feat):
        b, n, c = self.b, feat.shape[0], self.spec.num_classes
        d_feat, logits, probs = b.upload(feat), b.empty(n, c), b.empty(n, c)
        L.check(self.lib, self.lib.tcr_dscnn_forward(self.h, b.ptr(d_feat), b.ptr(self.params), n, b.ptr(logits), b.ptr(probs),
                                                     b.stream), "tcr_dscnn_forward")
        b.sync()
        return b.download(logits), b.download(probs)

    def layer_output(self, feat, k):
        """Output of layer k - 1 (tcr_dscnn_forward_partial) with one utterance of NaN padding after it."""
        b, n = self.b, feat.shape[0]
        shape = R.geometry(self.spec)[k - 1]
        d_feat, out = b.upload(feat), b.empty(n + 1, *shape)
        L.check(self.lib, self.lib.tcr_dscnn_forward_partial(self.h, b.ptr(d_feat), b.ptr(self.params), n, k, b.ptr(out), b.stream),
                "tcr_dscnn_forward_partial")
        b.sync()
        got = b.download(out)
        assert np.isnan(got[n]).all(), f"layer {k - 1} stored past the last utterance"
        assert np.isfinite(got[:n]).all(), f"layer {k - 1} left positions unwritten"
        return got[:n]


def check_net(net, feat, layers=None, rows=None):
    """Layers (1-based counts of forward_partial, all by default) on the path's own input to them, and for a block's second conv the
    path's own block input, against res_oracle.layer within 1e-5 of the layer's maximum; then logits against the fp64 oracle within
    1e-4 and the softmax, with the arg-max equal wherever the oracle's top-2 margin exceeds the error.  rows: the utterances the
    oracle checks (all by default; the NaN canary and the finiteness check cover the whole batch).  Returns the relative error of
    each layer, and of the logits under "logits", and the logits of the whole batch."""
    spec, p = net.spec, net.p
    layers = range(1, spec.layers + 2) if layers is None else layers
    rows = slice(None) if rows is None else rows
    outs = {0: feat[rows].astype(np.float64)}
    for k in sorted({j for k in layers for j in (k, k - 1, k - 2) if j >= 1}):
        outs[k] = net.layer_output(feat, k)[rows].astype(np.float64)
    errs = {k: rel_err(outs[k], R.layer(spec, p, k - 1, outs[k - 1], outs.get(k - 2) if k >= 3 else None)) for k in layers}
    assert max(errs.values()) <= 1e-5, errs
    logits, probs = net.forward(feat)
    ref = R.forward(spec, p, feat[rows].astype(np.float64))
    err = np.abs(logits[rows] - ref).max()
    assert err <= 1e-4 * np.abs(ref).max(), err / np.abs(ref).max()
    e = np.exp(ref - ref.max(1, keepdims=True))
    np.testing.assert_allclose(probs[rows], e / e.sum(1, keepdims=True), atol=max(2e-5, 2 * err))
    top2 = np.sort(ref, 1)[:, -2:]                                     # one column for a single class: no margin to check
    clear = top2[:, -1] - top2[:, 0] > 2 * err
    assert np.array_equal(logits[rows].argmax(1)[clear], ref.argmax(1)[clear])
    errs["logits"] = float(err / np.abs(ref).max())
    return errs, logits


@pytest.mark.parametrize("model,T,Fq", GEOMETRY)
def test_emulated_forward_matches_oracle(emu, model, T, Fq):
    """res_fconv (with and without the pool), res_conv in both residual modes at every dilation, and res2d_head on the CPU emulator,
    layer by layer and end to end.  Maps past 200 positions check one utterance, on f_conv, the first block and the last two convs
    (Res15: conv11 at rate 8 with its residual, conv12 at rate 16)."""
    big = T * Fq > 200
    net = ResNet(emu, model, T, Fq, 2)
    L_ = net.spec.layers
    try:
        check_net(net, np.random.RandomState(T + Fq).randn(1 if big else 2, T, Fq).astype(np.float32),
                  [1, 2, 3, L_, L_ + 1] if big else None)
    finally:
        net.close()


def test_emulated_residual_layer_equals_the_full_forward(emu):
    """The aliased residual (out == block input, full forward) and the distinct `out` of forward_partial give the same bits: the
    logits of the full forward equal the head of the partial forward's last layer, recomputed from it in fp64 within 1e-6."""
    net = ResNet(emu, "Res15Narrow", 13, 8, 3, seed=2)
    try:
        feat = np.random.RandomState(4).randn(3, 13, 8).astype(np.float32)
        last = net.layer_output(feat, net.spec.layers + 1)
        logits, _ = net.forward(feat)
        ref = R.head(net.spec, net.p, last.astype(np.float64))
        assert np.abs(logits - ref).max() <= 1e-6 * np.abs(ref).max()
    finally:
        net.close()


def _recipe_lines(model):
    return [x for x in open(os.path.join(ROOT, "tests", "golden", "reference_recipes.txt")) if f" {model} " in x + " "]


@pytest.mark.parametrize("model", ["Res8Model", "Res8NarrowModel", "Res15Model", "Res15NarrowModel"])
def test_recipe_lines_parse_and_training_raises(model):
    from tcresnet_b200 import evaluate_audio, train_audio
    from tcresnet_b200.factory import audio_nets
    from tcresnet_b200.runtime import Node
    lines = _recipe_lines(model)
    assert len(lines) == 3
    for line in lines:
        mod = train_audio if line.startswith("python train_audio.py") else evaluate_audio
        args = mod.parse_arguments(shlex.split(line)[2:])
        assert args.model == model and args.weight_decay == 1e-5 and args.num_mfccs == 40
    cls = getattr(audio_nets, model)
    assert issubclass(cls, audio_nets.DsCnnModel) and cls.__module__ == audio_nets.__name__
    assert not hasattr(audio_nets, "_baseline")
    tr = train_audio.parse_arguments(shlex.split(lines[0])[2:])
    with pytest.raises(NotImplementedError, match="training Res8 / Res15 is out of scope.*evaluation"):
        cls(tr, None).build(Node("wav", [None, 16000, 1]), Node("labels", [None, 12]), is_training=True)
    ev = evaluate_audio.parse_arguments(shlex.split(lines[1])[2:])
    assert (ev.batch_size, ev.valid_type) == (3, "loop")
    ev.device_dataset = True
    with pytest.raises(NotImplementedError, match="--device_dataset serves the TC-ResNet models only"):
        cls(ev, None).build(Node("wav", [None, 16000, 1]), Node("labels", [None, 12]), is_training=False)
    default = evaluate_audio.parse_arguments(shlex.split(lines[1].replace("--weight_decay 0.00001", ""))[2:])
    assert default.weight_decay == 1e-5
