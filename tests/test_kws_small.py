"""KWSModel's speech_commands nets (--architecture low_latency_conv / tiny_conv, audio_nets/kws.py) on the DS-CNN handle, without a
GPU: the parameter table and FLOPs, the oracle against an independent torch restatement, the refusals, the conv and dense kernels
on the CPU emulator against the oracle (tiny_conv's SAME padding at odd and even sizes), and the Python surface."""
import ctypes as C
import shlex

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import kws_small_oracle as S
from tcr_harness import NumpyBackend, rel_err
from test_kws import _recipe_lines, table

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L

TCR_ERR_INVALID, TCR_ERR_UNSUPPORTED = 1, 3           # include/tcr_b200.h
ARCHS = ["low_latency_conv", "tiny_conv"]


@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


def create(lib, arch, h, w, max_batch=4, classes=12):
    handle = C.c_void_p()
    rc = lib.tcr_dscnn_create(C.byref(L.TcrDscnnConfig(ord(S.CODES.get(arch, arch)), h, w, classes, max_batch, 0)), C.byref(handle))
    return rc, handle


def expected_table(arch, T, Fq, classes=12):
    """The formulas: W = F - 7 (low_latency_conv); H = ceil(T / 2), W = ceil(F / 2) (tiny_conv)."""
    if arch == "low_latency_conv":
        W = Fq - 7
        k = W * 186
        rows = [("first_weights", (T, 8, 1, 186)), ("first_bias", (186,)), ("first_fc_weights", (k, 128)), ("first_fc_bias", (128,)),
                ("second_fc_weights", (128, 128)), ("second_fc_bias", (128,)), ("final_fc_weights", (128, classes)),
                ("final_fc_bias", (classes,))]
        flops = 2 * W * T * 8 * 186 + 2 * k * 128 + 2 * 128 * 128 + 2 * 128 * classes
    else:
        H, W = -(-T // 2), -(-Fq // 2)
        k = H * W * 8
        rows = [("first_weights", (10, 8, 1, 8)), ("first_bias", (8,)), ("final_fc_weights", (k, classes)), ("final_fc_bias", (classes,))]
        flops = 2 * H * W * 80 * 8 + 2 * k * classes
    return rows, sum(int(np.prod(s)) for _, s in rows), flops


@pytest.mark.parametrize("arch", ARCHS)
@pytest.mark.parametrize("T,Fq", [(49, 40), (98, 40), (49, 64)])
def test_parameter_table_and_flops(emu, arch, T, Fq):
    rc, h = create(emu.lib, arch, T, Fq)
    assert rc == 0
    try:
        rows, nparams, flops = table(emu.lib, h)
        exp_rows, exp_params, exp_flops = expected_table(arch, T, Fq)
        assert [(n, s) for n, s, _ in rows] == exp_rows
        assert all(L.KIND_NAMES[kind] == ("beta" if len(s) == 1 else "weight") for _, s, kind in rows)
        assert (nparams, flops) == (exp_params, exp_flops)
        spec = S.build_spec(arch, T, Fq)
        assert spec.var_names == [n for n, _ in exp_rows] and S.forward_flops(spec) == flops
        if (T, Fq) == (49, 40):
            assert (nparams, flops) == {"low_latency_conv": (876950, 6419360), "tiny_conv": (48660, 736000)}[arch]
    finally:
        emu.lib.tcr_dscnn_destroy(h)


def test_tiny_conv_same_padding():
    """pad_total = max((out - 1) * 2 + k - in, 0), the smaller half first: 4 rows above and 5 below at T = 49, 4 and 4 at 98."""
    assert S.same_pad(49, 10, 2) == (25, 4, 5) and S.same_pad(98, 10, 2) == (49, 4, 4)
    assert S.same_pad(40, 8, 2) == (20, 3, 3) and S.same_pad(1, 10, 2) == (1, 4, 5) and S.same_pad(1, 8, 2) == (1, 3, 4)


def torch_forward(spec, p, x):
    """Independent restatement: F.pad (TF SAME) + F.conv2d + bias + ReLU, flatten NHWC, F.linear per dense layer."""
    t = torch.tensor(x)[:, None]                                        # NCHW
    w, b, stride = spec.convs[0]
    if spec.arch == "tiny_conv":
        T, Fq = x.shape[1:]
        ph, pw = max((-(-T // 2) - 1) * 2 + 10 - T, 0), max((-(-Fq // 2) - 1) * 2 + 8 - Fq, 0)
        t = F.pad(t, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2))
    t = F.relu(F.conv2d(t, torch.tensor(p[w]).permute(3, 2, 0, 1), torch.tensor(p[b]), stride=stride))
    act = t.permute(0, 2, 3, 1)
    y = act.reshape(x.shape[0], -1)
    for wm, bm in spec.mats:
        y = F.linear(y, torch.tensor(p[wm]).T, torch.tensor(p[bm]))
    return act.numpy(), y.numpy()


@pytest.mark.parametrize("arch,T,Fq", [("low_latency_conv", 49, 40), ("low_latency_conv", 7, 8), ("tiny_conv", 49, 40),
                                       ("tiny_conv", 98, 41), ("tiny_conv", 1, 1), ("tiny_conv", 5, 7)])
def test_oracle_matches_independent_torch_restatement(arch, T, Fq):
    spec = S.build_spec(arch, T, Fq)
    p = S.init_variables(spec, 0)
    x = np.random.RandomState(1).randn(3, T, Fq)
    act, ref = torch_forward(spec, p, x)
    assert act.shape == (3,) + S.conv_geometry(arch, T, Fq)[0]
    assert rel_err(S.layer(spec, p, 0, x), act) <= 1e-12
    assert rel_err(S.forward(spec, p, x), ref) <= 1e-12


def _err(lib):
    return lib.tcr_last_error().decode()


def test_refusals(emu):
    """Each bound just past its limit, then at it.  The grid and K bounds are refused before anything is allocated."""
    lib = emu.lib
    big = 2**31 // 33 + 1                                               # max_batch x 33 columns past 2^31 - 1
    for arch, T, Fq, mb, bound in (("low_latency_conv", 49, 7, 4, "width >= 8"),
                                   ("low_latency_conv", 49, 40, big, "kws_llconv: max_batch"),
                                   ("tiny_conv", 49, 2389, 4, "kws_tinyconv needs 232608 bytes of shared memory at width 2389, "
                                                               "the limit is 232448"),
                                   ("tiny_conv", 2**24, 40, 2**11, "kws_tinyconv: max_batch 2048 x 1048576 row tiles"),
                                   ("tiny_conv", 2**30, 40, 4, "kws_fcs: K = 85899345920")):
        rc, h = create(lib, arch, T, Fq, mb)
        assert rc == TCR_ERR_UNSUPPORTED and bound in _err(lib) and not h.value, (arch, T, Fq, _err(lib))
    for arch, T, Fq in (("low_latency_conv", 1, 8), ("low_latency_conv", 49, 8), ("tiny_conv", 49, 2388), ("tiny_conv", 1, 1)):
        rc, h = create(lib, arch, T, Fq)
        assert rc == 0, _err(lib)
        lib.tcr_dscnn_destroy(h)
    rc, h = create(lib, "Z", 49, 40)
    assert rc == TCR_ERR_INVALID and "'C' (low_latency_conv) or 'Y' (tiny_conv)" in _err(lib)


class SmallNet:
    """One low_latency_conv / tiny_conv handle with the oracle's seeded variables on a tests/tcr_harness backend."""

    def __init__(self, b, arch, T, Fq, max_batch, seed=0, classes=12):
        self.b, self.lib, self.arch = b, b.lib, arch
        self.spec = S.build_spec(arch, T, Fq, classes)
        self.p = S.init_variables(self.spec, seed)
        rc, self.h = create(self.lib, arch, T, Fq, max_batch, classes)
        L.check(self.lib, rc, "tcr_dscnn_create")
        self.params = b.upload(S.flatten(self.spec, self.p))

    def close(self):
        self.lib.tcr_dscnn_destroy(self.h)

    def forward(self, feat, logits=True, probs=True):
        b, n, c = self.b, feat.shape[0], self.spec.num_classes
        d_feat, lg, pr = b.upload(feat), b.empty(n, c), b.empty(n, c)
        L.check(self.lib, self.lib.tcr_dscnn_forward(self.h, b.ptr(d_feat), b.ptr(self.params), n, b.ptr(lg) if logits else None,
                                                     b.ptr(pr) if probs else None, b.stream), "tcr_dscnn_forward")
        b.sync()
        return b.download(lg), b.download(pr)

    def layer_output(self, feat):
        """Output of the conv (tcr_dscnn_forward_partial) with one utterance of NaN padding after it."""
        b, n = self.b, feat.shape[0]
        shape = S.conv_geometry(self.arch, self.spec.h, self.spec.w)[0]
        d_feat, out = b.upload(feat), b.empty(n + 1, *shape)
        L.check(self.lib, self.lib.tcr_dscnn_forward_partial(self.h, b.ptr(d_feat), b.ptr(self.params), n, 1, b.ptr(out), b.stream),
                "tcr_dscnn_forward_partial")
        b.sync()
        got = b.download(out)
        assert np.isnan(got[n]).all(), "the conv stored past the last utterance"
        assert np.isfinite(got[:n]).all(), "the conv left positions unwritten"
        return got[:n]


def check_small(net, feat, layer_output=None, rows=None):
    """The conv on the path's input against kws_small_oracle.layer, within 1e-5 of the layer's maximum (layer_output(): the path's
    conv output, net.layer_output by default), then the head on that output and the logits and softmax end to end against the
    fp64 oracle within 1e-4, with the arg-max equal wherever the oracle's top-2 margin exceeds the error.  The path runs the whole
    batch; rows: the utterances the oracle checks (all by default).  Returns the layer error and the logits error."""
    spec, p = net.spec, net.p
    out = (layer_output or (lambda: net.layer_output(feat)))()
    logits, probs = net.forward(feat)
    if rows is not None:
        feat, out, logits, probs = feat[rows], out[rows], logits[rows], probs[rows]
    act = S.layer(spec, p, 0, feat.astype(np.float64))
    lerr = rel_err(out, act)
    assert lerr <= 1e-5, lerr
    ref = S.head(spec, p, act)                                          # = S.forward: the oracle's conv computed once
    scale = np.abs(ref).max()
    err = np.abs(logits - ref).max()
    assert err <= 1e-4 * scale, err / scale
    head_err = np.abs(logits - S.head(spec, p, out.astype(np.float64))).max()
    assert head_err <= 1e-4 * scale, head_err / scale
    e = np.exp(ref - ref.max(1, keepdims=True))
    np.testing.assert_allclose(probs, e / e.sum(1, keepdims=True), atol=max(2e-5, 2 * err))
    top2 = np.sort(ref, 1)[:, -2:]
    clear = top2[:, -1] - top2[:, 0] > 2 * err
    assert np.array_equal(logits.argmax(1)[clear], ref.argmax(1)[clear])
    return lerr, err / scale


@pytest.mark.parametrize("arch,T,Fq,n", [("low_latency_conv", 49, 40, 3), ("low_latency_conv", 98, 40, 2), ("low_latency_conv", 49, 8, 5),
                                         ("tiny_conv", 49, 40, 3), ("tiny_conv", 98, 40, 2), ("tiny_conv", 49, 64, 2)])
def test_emulated_forward_matches_oracle(emu, arch, T, Fq, n):
    """kws_llconv / kws_tinyconv, kws_fcs (K = 6,138 in 48 chunks of 128, the last of 122, for low_latency_conv at 49 x 40; 4,000
    in 16 chunks of 256 for tiny_conv) and kws_fcb_head on the CPU emulator, layer and logits."""
    net = SmallNet(emu, arch, T, Fq, n)
    try:
        check_small(net, np.random.RandomState(n).randn(n, T, Fq).astype(np.float32))
    finally:
        net.close()


@pytest.mark.parametrize("T,Fq", [(1, 1), (2, 3), (5, 7), (9, 10), (10, 8), (16, 9), (49, 40), (98, 41), (17, 128)])
def test_emulated_tiny_conv_padding(emu, T, Fq):
    """tiny_conv at odd and even T and F, below the 10 x 8 kernel (the window mostly padding) and past one 8-row tile (17 x 128:
    9 rows in tiles of 8 and 1); the positive inputs make every dropped or misplaced zero of the padding show."""
    net = SmallNet(emu, "tiny_conv", T, Fq, 2, seed=T + Fq)
    try:
        rng = np.random.RandomState(T * Fq)
        check_small(net, (rng.rand(2, T, Fq) + 0.5).astype(np.float32))
        check_small(net, rng.randn(2, T, Fq).astype(np.float32))
    finally:
        net.close()


def test_emulated_batch_invariance(emu):
    """An utterance's logits are the same bits alone and in a batch that spans more than one 128-row conv tile and one 64-utterance
    head group (low_latency_conv at 49 x 9: two columns per utterance, n = 65)."""
    for arch, T, Fq in (("low_latency_conv", 6, 9), ("tiny_conv", 3, 4)):
        net = SmallNet(emu, arch, T, Fq, 65)
        try:
            feat = np.random.RandomState(0).randn(65, T, Fq).astype(np.float32)
            full = net.forward(feat)[0]
            for u in (0, 63, 64):
                assert np.array_equal(net.forward(feat[u:u + 1])[0], full[u:u + 1]), (arch, u)
            assert np.array_equal(net.forward(feat, probs=False)[0], full)
            assert np.isnan(net.forward(feat, logits=False)[0]).all()
        finally:
            net.close()


def _args(arch, train=False):
    from tcresnet_b200 import evaluate_audio, train_audio
    lines = _recipe_lines()
    if train:
        tr = [x for x in lines if x.startswith("python train_audio.py")][0]
        return train_audio.parse_arguments(shlex.split(tr)[2:-1] + [arch])
    ev = [x for x in lines if x.startswith("python evaluate_audio.py")][0]
    return evaluate_audio.parse_arguments(shlex.split(ev)[2:-1] + [arch])


@pytest.mark.parametrize("arch", ARCHS)
def test_kws_model_parses_and_refuses_training(arch):
    from tcresnet_b200.factory import audio_nets
    from tcresnet_b200.runtime import Node
    args = _args(arch)
    assert args.model == "KWSModel" and args.architecture == arch and args.weight_decay == 1e-4
    assert audio_nets.KWSModel(args, None).dscnn_size == S.CODES[arch]
    with pytest.raises(NotImplementedError, match="training the KWS baselines is out of scope.*evaluation"):
        audio_nets.KWSModel(_args(arch, train=True), None).build(Node("wav", [None, 16000, 1]), Node("labels", [None, 12]),
                                                                  is_training=True)


@pytest.mark.parametrize("arch", ["conv", "single_fc", "low_latency_svdf"])
def test_other_architectures_still_raise(arch):
    from tcresnet_b200.factory import audio_nets
    from tcresnet_b200.runtime import Node
    with pytest.raises(NotImplementedError, match=f"{arch} is not on the CUDA path; supported: trad_fpool3, one_fstride4, "
                                                  "low_latency_conv, tiny_conv"):
        audio_nets.KWSModel(_args(arch), None).build(Node("wav", [None, 16000, 1]), Node("labels", [None, 12]), is_training=False)


@pytest.mark.parametrize("arch", ARCHS)
def test_l2_term_includes_the_biases(emu, arch):
    """total_loss's L2 term is weight_decay * sum(l2_loss(v)) over every variable of the table, the biases included
    (factory/audio_nets.py build_loss excludes only BatchNorm, and these nets have none)."""
    from tcresnet_b200.factory import audio_nets
    spec = S.build_spec(arch, 49, 40)
    p = S.init_variables(spec, 3)
    rc, h = create(emu.lib, arch, 49, 40)
    assert rc == 0
    try:
        rows = table(emu.lib, h)[0]
    finally:
        emu.lib.tcr_dscnn_destroy(h)
    biases = [n for n, s, kind in rows if L.KIND_NAMES[kind] == "beta"]
    assert biases == [n for n in spec.var_names if n.endswith("_bias")] and biases
    m = object.__new__(audio_nets.KWSModel)
    m.args = _args(arch)
    m.params = torch.from_numpy(S.flatten(spec, p, np.float64))
    got = m._regularization()
    assert got == pytest.approx(1e-4 * S.l2_loss(p), rel=1e-12)
    without = 1e-4 * S.l2_loss({k: v for k, v in p.items() if k not in biases})
    assert abs(got - without) > 1e-3 * got
