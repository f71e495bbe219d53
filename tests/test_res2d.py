"""The 2-D ablations of TC-ResNet8 (ResNet2D8 / ResNet2D8Pool, audio_nets/tc_resnet.py) on the DS-CNN handle, without a GPU: the
parameter table and FLOPs, the channel formula, the refusals, the oracle against torch, every kernel on the CPU emulator against
the oracle at geometries that hit both SAME-padding parities on every stage, and the CLI surface."""
import ctypes as C
import os
import shlex

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import res2d_oracle as R
from tcr_harness import NumpyBackend, rel_err

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TCR_ERR_INVALID, TCR_ERR_UNSUPPORTED = 1, 3           # include/tcr_b200.h

# (model, T, F): both parities of every stage's input in both axes across the rows, the pool variant's smallest map, and 1-wide maps
GEOMETRY = [("ResNet2D8", 98, 40), ("ResNet2D8", 97, 39), ("ResNet2D8", 99, 41), ("ResNet2D8", 49, 10), ("ResNet2D8", 6, 3),
            ("ResNet2D8", 1, 1), ("ResNet2D8", 1, 7), ("ResNet2D8", 5, 1), ("ResNet2D8", 49, 46),
            ("ResNet2D8Pool", 98, 40), ("ResNet2D8Pool", 4, 4), ("ResNet2D8Pool", 7, 9), ("ResNet2D8Pool", 61, 23)]


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


def test_stage_parities_are_covered():
    """Across GEOMETRY every strided stage sees an even and an odd input in each axis, so a leading pad of 0 and of 1."""
    seen = set()
    for model, T, Fq in GEOMETRY:
        spec = R.build_spec(model, T, Fq)
        geo = R.geometry(spec)
        for i, b in enumerate(spec.blocks):
            if b["stride"] == 2:
                seen |= {(i, "h", geo[i][0] % 2), (i, "w", geo[i][1] % 2)}
    assert seen == {(i, a, p) for i in range(3) for a in "hw" for p in (0, 1)}, sorted(seen)
    assert any(not R.build_spec(m, T, Fq).blocks[0]["down"] for m, T, Fq in GEOMETRY)      # a stride-1 identity shortcut (c0 == c1)


@pytest.mark.parametrize("model,T,Fq", GEOMETRY)
def test_parameter_table_and_flops(emu, model, T, Fq):
    rc, h = create(emu.lib, model, T, Fq)
    assert rc == 0, _err(emu.lib)
    try:
        rows, nparams, flops = table(emu.lib, h)
        spec = R.build_spec(model, T, Fq)
        shapes = spec.var_shapes
        assert [n for n, _, _ in rows] == spec.var_names
        assert [s for n, s, _ in rows] == [shapes[n] for n in spec.var_names]
        kinds = {"weights": "weight", "beta": "beta", "gamma": "gamma", "moving_mean": "moving_mean",
                 "moving_variance": "moving_variance"}
        assert [k for _, _, k in rows] == [kinds[n.rsplit("/", 1)[1]] for n in spec.var_names]
        assert nparams == sum(int(np.prod(s)) for s in shapes.values())
        assert flops == R.forward_flops(spec)
        if (T, Fq) == (98, 40):
            assert flops == {"ResNet2D8": 35744352, "ResNet2D8Pool": 3949920}[model]
            assert rows[0] == (f"{model}/conv0/weights", (3, 3, 1, 23), "weight")
            assert [n for n, _, _ in rows[3:6]] == [f"{model}/block0/down/weights", f"{model}/block0/down/BatchNorm/beta",
                                                    f"{model}/block0/down/BatchNorm/gamma"]
    finally:
        emu.lib.tcr_dscnn_destroy(h)


def test_flops_formula_by_hand():
    """ResNet2D8 at 98 x 40: conv0 1,622,880; block0 9,737,280 + 10,160,640 + down 1,081,920; block1 3,456,000 + 4,608,000 + 384,000;
    block2 1,797,120 + 2,695,680 + 199,680; fc 1,152.  The pool variant's blocks run on 24 x 10."""
    assert R.forward_flops(R.build_spec("ResNet2D8", 98, 40)) == 1622880 + 9737280 + 10160640 + 1081920 + 3456000 + 4608000 + \
        384000 + 1797120 + 2695680 + 199680 + 1152
    assert R.geometry(R.build_spec("ResNet2D8Pool", 98, 40))[0] == (24, 10, 23)


@pytest.mark.parametrize("wm", [0.5, 0.75, 1.0, 1.3, 1.5, 2.0, 2.5])
@pytest.mark.parametrize("Fq", [10, 40, 64, 128])
def test_channels_match_the_python_formula(emu, wm, Fq):
    rc, h = create(emu.lib, "ResNet2D8", 20, Fq, wm=wm)
    assert rc == 0, _err(emu.lib)
    try:
        rows, _, _ = table(emu.lib, h)
        conv = {n: s for n, s, _ in rows if n.endswith("/weights")}
        got = [conv["ResNet2D8/conv0/weights"][3]] + [conv[f"ResNet2D8/block{i}/conv{i}_1/weights"][3] for i in range(3)]
        n = [int(x * wm) for x in [16, 24, 32, 48]]
        assert got == [int((3 * Fq * n[0] + 10 * n[0] * n[1]) / (9 + 10 * n[1]))] + n[1:] == R.channels(Fq, wm)
    finally:
        emu.lib.tcr_dscnn_destroy(h)
    assert R.channels(40) == [23, 24, 32, 48] and R.channels(10) == [17, 24, 32, 48]


def test_refusals(emu):
    lib = emu.lib
    for T, Fq in ((3, 40), (98, 3), (1, 1)):
        rc, h = create(lib, "ResNet2D8Pool", T, Fq)
        assert rc == TCR_ERR_UNSUPPORTED and "height >= 4 and width >= 4" in _err(lib) and not h.value, (T, Fq, _err(lib))
    rc, h = create(lib, "ResNet2D8", 98, 40, wm=2.7)                       # c3 = int(48 * 2.7) = 129
    assert rc == TCR_ERR_UNSUPPORTED and "needs 129 channels in a block; res2d_block takes 1 to 128" in _err(lib), _err(lib)
    rc, h = create(lib, "ResNet2D8", 98, 40, wm=0.05)                      # c1 = int(16 * 0.05) = 0
    assert rc == TCR_ERR_UNSUPPORTED and "needs 0 channels" in _err(lib), _err(lib)
    for size in ("S", "P", "F"):
        rc, h = create(lib, size, 49, 40, wm=1.0)
        assert rc == TCR_ERR_INVALID and "width_multiplier (1) applies to ResNet2D8 / ResNet2D8Pool only" in _err(lib), _err(lib)
    rc, h = create(lib, "ResNet2D8", 98, 40, wm=-1.0)
    assert rc == TCR_ERR_INVALID and "bad width_multiplier" in _err(lib)
    rc, h = create(lib, "ResNet2D8", 98, 40, classes=33)                   # the shared head's class bound
    assert rc == TCR_ERR_INVALID and "bad DS-CNN configuration" in _err(lib)
    rc, h = create(lib, "Q", 98, 40)
    assert rc == TCR_ERR_INVALID and "'R' (ResNet2D8) or 'A' (ResNet2D8Pool)" in _err(lib)
    for model, T, Fq, wm in (("ResNet2D8Pool", 4, 4, 0.0), ("ResNet2D8", 1, 1, 2.5), ("ResNet2D8", 998, 128, 2.5)):   # accepted edges
        rc, h = create(lib, model, T, Fq, wm=wm)
        assert rc == 0, (model, T, Fq, _err(lib))
        lib.tcr_dscnn_destroy(h)
    rc, h = create(lib, "ResNet2D8", 98, 40)
    try:
        lis = C.c_void_p()
        assert lib.tcr_dscnn_listener_create(h, C.byref(L.TcrListenerConfig(1, 1, 320)), C.byref(lis)) == TCR_ERR_INVALID
        assert "no front-end" in _err(lib)
    finally:
        lib.tcr_dscnn_destroy(h)


def _torch_same(x, w, s):
    """conv2d with TF SAME's asymmetric pads given explicitly (F.pad takes (left, right, top, bottom))."""
    k, (H, W) = w.shape[0], x.shape[2:]
    ph = max((-(-H // s) - 1) * s + k - H, 0)
    pw = max((-(-W // s) - 1) * s + k - W, 0)
    return F.conv2d(F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2)), w.permute(3, 2, 0, 1), stride=s)


@pytest.mark.parametrize("model,T,Fq,wm", [("ResNet2D8", 98, 40, 1.0), ("ResNet2D8", 97, 39, 0.5), ("ResNet2D8", 6, 3, 1.0),
                                           ("ResNet2D8", 49, 46, 1.0), ("ResNet2D8Pool", 7, 9, 2.5)])
def test_oracle_matches_torch_with_explicit_pads(model, T, Fq, wm):
    spec = R.build_spec(model, T, Fq, width_multiplier=wm)
    p = R.init_variables(spec, 0)
    t = {k: torch.tensor(v) for k, v in p.items()}
    x = np.random.RandomState(1).randn(2, T, Fq)
    s = model + "/"

    def cbn(name, y, stride):
        b = s + name + "/BatchNorm/"
        y = _torch_same(y, t[s + name + "/weights"], stride)
        return F.batch_norm(y, t[b + "moving_mean"], t[b + "moving_variance"], t[b + "gamma"], t[b + "beta"], False, 0.0, R.EPS)

    y = F.relu(cbn("conv0", torch.tensor(x)[:, None], 1))
    if model == "ResNet2D8Pool":
        y = F.avg_pool2d(y, 4, 4)
    acts = [y]
    for i, b in enumerate(spec.blocks):
        sc = F.relu(cbn(f"block{i}/down", y, 2)) if b["down"] else y
        y = F.relu(cbn(b["conv1"], F.relu(cbn(b["conv0"], y, b["stride"])), 1) + sc)
        acts.append(y)
    logits = y.mean((2, 3)) @ t[s + "fc/weights"][0, 0]
    got = R.forward_layers(spec, p, x)
    for l, (a, r) in enumerate(zip(got, acts)):
        assert a.shape == (2,) + R.geometry(spec)[l]
        assert rel_err(a, r.permute(0, 2, 3, 1).numpy()) <= 1e-12, l
    assert rel_err(R.head(spec, p, got[-1]), logits.numpy()) <= 1e-12


def test_same_padding_parity():
    """The leading pad at stride 2 is 0 for an even input and 1 for an odd one; at 98 x 40 block0 pads (0, 1) in time, block1 (1, 1)."""
    assert R.same(98, 3, 2) == (49, 0) and R.same(49, 3, 2) == (25, 1) and R.same(40, 3, 2) == (20, 0) and R.same(1, 3, 2) == (1, 1)
    assert R.same(98, 1, 2) == (49, 0) and R.same(49, 1, 2) == (25, 0)          # down never pads
    x = np.zeros((1, 4, 4, 1))
    x[0, 0, 0, 0] = 1.0                                                          # pad 0 before: output (0, 0) sees x[0, 0] at tap (0, 0)
    w = np.zeros((3, 3, 1, 1))
    w[0, 0, 0, 0] = 1.0
    assert R.conv_same(x, w, 2)[0, 0, 0, 0] == 1.0


class Res2dNet:
    """One 2-D ablation handle with the oracle's seeded variables on a tests/tcr_harness backend."""

    def __init__(self, b, model, T, Fq, max_batch, seed=0, classes=12, wm=1.0):
        self.b, self.lib, self.model = b, b.lib, model
        self.spec = R.build_spec(model, T, Fq, classes, wm)
        self.p = R.init_variables(self.spec, seed)
        rc, self.h = create(self.lib, model, T, Fq, max_batch, classes, wm)
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


def check_net(net, feat, rows=None):
    """Each layer on the path's own input to it against res2d_oracle.layer, within 1e-5 of the layer's maximum, then logits against
    the fp64 oracle within 1e-4 and the softmax, with the arg-max equal wherever the oracle's top-2 margin exceeds the error.  rows:
    the utterances the oracle checks (all by default; the NaN canary and the finiteness check cover the whole batch).  Returns the
    relative error of each layer (1-based, as forward_partial counts them) and of the logits under "logits", and the logits of the
    whole batch."""
    spec, p = net.spec, net.p
    rows = slice(None) if rows is None else rows
    errs, x = {}, feat[rows].astype(np.float64)
    for k in range(1, 5):
        out = net.layer_output(feat, k)[rows]
        errs[k] = rel_err(out, R.layer(spec, p, k - 1, x))
        x = out.astype(np.float64)
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
    """res2d_conv0, res2d_block (both shortcuts, both pad parities, channel counts that are not multiples of 4) and res2d_head on
    the CPU emulator, layer by layer and end to end."""
    net = Res2dNet(emu, model, T, Fq, 2)
    try:
        check_net(net, np.random.RandomState(T + Fq).randn(2, T, Fq).astype(np.float32))
    finally:
        net.close()


def test_emulated_forward_sliced_filters(emu):
    """Width 2.5 at 98 x 40 (up to 120 channels): the block kernel's filter slices (COT below the channel count) and its smaller
    tiles, on one utterance."""
    net = Res2dNet(emu, "ResNet2D8Pool", 98, 40, 1, wm=2.5)
    try:
        check_net(net, np.random.RandomState(5).randn(1, 98, 40).astype(np.float32))
    finally:
        net.close()


def _recipe_lines(model):
    return [x for x in open(os.path.join(ROOT, "tests", "golden", "reference_recipes.txt")) if f" {model} " in x + " "]


@pytest.mark.parametrize("model", ["ResNet2D8Model", "ResNet2D8PoolModel"])
def test_recipe_lines_parse_and_training_raises(model):
    from tcresnet_b200 import evaluate_audio, train_audio
    from tcresnet_b200.factory import audio_nets
    from tcresnet_b200.runtime import Node
    lines = _recipe_lines(model)
    assert len(lines) == 3
    for line in lines:
        mod = train_audio if line.startswith("python train_audio.py") else evaluate_audio
        args = mod.parse_arguments(shlex.split(line)[2:])
        assert args.model == model and args.weight_decay == 1e-3 and args.width_multiplier == 1.0 and args.num_mfccs == 40
        assert args.dropout_keep_prob == 0.5
    cls = getattr(audio_nets, model)
    assert issubclass(cls, audio_nets.DsCnnModel)
    tr = train_audio.parse_arguments(shlex.split(lines[0])[2:])
    with pytest.raises(NotImplementedError, match="training the 2-D ablations is out of scope.*evaluation"):
        cls(tr, None).build(Node("wav", [None, 16000, 1]), Node("labels", [None, 12]), is_training=True)
    ev = evaluate_audio.parse_arguments(shlex.split(lines[1])[2:])
    ev.device_dataset = True
    with pytest.raises(NotImplementedError, match="--device_dataset serves the TC-ResNet models only"):
        cls(ev, None).build(Node("wav", [None, 16000, 1]), Node("labels", [None, 12]), is_training=False)
