"""The KWS baselines at the edges of every geometry, batch and class count their DS-CNN handle accepts, against the fp64 oracle
(kws_oracle): the parameter table, each conv layer and the logits at each row of GEOMETRIES, the persistent wgmma kernels' tile
walk against the SM count, 1 to 32 classes with the logits-only / probs-only calls and the evaluation counts, the listener at
more front-ends, and the refusals.  The FMA kernels on the CPU emulator; the wgmma kernels, kws_lin / kws_head and the windowed
kernels on the GPU."""
import argparse
import ctypes as C

import numpy as np
import pytest

from oracle import kws_oracle as K
from oracle import metrics_oracle as MO
from tcr_harness import NumpyBackend, launched, rel_err
from test_dscnn import _sms, check_invariance, features, wide_range
from test_kws import TCR_ERR_INVALID, KwsNet, check_net, create, expected_table, table
from test_kws_eval import KERNELS, check_layers, run_listener

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L

C1_TILE, C2_TILE, LIN_CHUNK = 42, 128, 256      # kws_conv1_tc pooled rows, kws_conv2_tc rows per tile; kws_lin's K chunk


def reach(arch, T, Fq):
    """What a geometry exercises.  trad_fpool3: w1_mod3 = (F - 7) % 3, the pre-pool columns the 1 x 3 pool drops; conv1_rows /
    conv2_rows, the pooled outputs (kws_conv1_tc) and output positions (kws_conv2_tc) per utterance; k and chunks, the flattened
    width kws_lin splits into chunks of 256.  one_fstride4: f8_mod4 = (F - 8) % 4, the columns its stride-4 conv drops; conv_k,
    the FMAs per output of kws_conv; staged, the floats of one utterance kws_conv stages in shared memory."""
    if arch == "trad_fpool3":
        H1, W1 = T - 19, Fq - 7
        H2, W2 = H1 - 9, W1 // 3 - 3
        k = H2 * W2 * 64
        return dict(w1_mod3=W1 % 3, conv1_rows=H1 * (W1 // 3), conv2_rows=H2 * W2, k=k, chunks=-(-k // LIN_CHUNK))
    k = ((Fq - 8) // 4 + 1) * 186
    return dict(f8_mod4=(Fq - 8) % 4, conv_k=T * 8, staged=T * Fq, k=k, chunks=-(-k // LIN_CHUNK))


# (arch, T, F, what the row reaches (checked against reach()), why it is here)
GEOMETRIES = [
    ("trad_fpool3", 29, 19, dict(w1_mod3=0, conv2_rows=1, k=64), "smallest accepted; one conv2 row per utterance"),
    ("trad_fpool3", 29, 20, dict(w1_mod3=1, conv2_rows=1), "smallest height, one pre-pool column dropped"),
    ("trad_fpool3", 29, 21, dict(w1_mod3=2, conv2_rows=1), "smallest height, two pre-pool columns dropped"),
    ("trad_fpool3", 30, 22, dict(k=256, chunks=1), "exactly one full lin chunk"),
    ("trad_fpool3", 49, 23, dict(w1_mod3=1, k=2688, chunks=11), "10 full lin chunks and a half one"),
    ("trad_fpool3", 49, 41, dict(w1_mod3=1, conv1_rows=330, conv2_rows=168), "the recipe's downstream shapes; odd row stride"),
    ("trad_fpool3", 49, 42, dict(w1_mod3=2, conv1_rows=330, conv2_rows=168), "the recipe's downstream shapes"),
    ("trad_fpool3", 61, 128, dict(w1_mod3=1, k=78144, chunks=306), "widest front-end; partial last of 306 lin chunks"),
    ("trad_fpool3", 400, 128, dict(conv2_rows=13764, k=880896, chunks=3441), "large T and F: 4.5 GFLOP of conv2 per utterance"),
    ("one_fstride4", 1, 8, dict(f8_mod4=0, conv_k=8, k=186), "T = 1, one output column"),
    ("one_fstride4", 49, 11, dict(f8_mod4=3, k=186), "three columns dropped by the stride"),
    ("one_fstride4", 400, 128, dict(f8_mod4=0, staged=51200, k=5766, chunks=23), "the 200 KB staging limit, 31 columns"),
    ("one_fstride4", 6400, 8, dict(conv_k=51200, staged=51200, k=186), "the staging limit: 51,200 FMAs per output"),
]
IDS = [f"{a}-{t}x{f}" for a, t, f, _, _ in GEOMETRIES]
BIG = {("trad_fpool3", 400, 128)}               # too slow for the emulator; small n on the GPU


def _kind(T, Fq):
    """The front end's features where the oracle's front end has the shape (MFCCs up to 40, log-mel up to 64), N(0, 1) past it."""
    if T <= 98:
        return "mfcc" if Fq <= 40 else ("logmel" if Fq <= 64 else "randn")
    return "randn"


@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


@pytest.mark.parametrize("arch,T,Fq,claims,why", GEOMETRIES, ids=IDS)
def test_table_and_flops(emu, arch, T, Fq, claims, why):
    """Each row reaches what it claims; tcr_dscnn_param_table and the FLOP count against the formulas and kws_oracle."""
    got = reach(arch, T, Fq)
    assert {k: got[k] for k in claims} == claims, (why, got)
    rc, h = create(emu.lib, arch, T, Fq)
    assert rc == 0
    try:
        rows, nparams, flops = table(emu.lib, h)
        exp_rows, exp_params, exp_flops = expected_table(arch, T, Fq)
        assert [(n, s) for n, s, _ in rows] == exp_rows
        assert (nparams, flops) == (exp_params, exp_flops)
        spec = K.build_spec(arch, T, Fq)
        assert [spec.var_shapes[n] for n in spec.var_names] == [s for _, s in exp_rows] and K.forward_flops(spec) == flops
        assert int(np.prod(K.conv_geometry(arch, T, Fq)[-1])) == got["k"]
    finally:
        emu.lib.tcr_dscnn_destroy(h)


@pytest.mark.parametrize("arch,T,Fq,claims,why", [g for g in GEOMETRIES if g[:3] not in BIG],
                         ids=[i for g, i in zip(GEOMETRIES, IDS) if g[:3] not in BIG])
def test_emulated_layers_and_logits(emu, arch, T, Fq, claims, why):
    """The FMA kernels (kws_conv for every conv layer, kws_lin, kws_head) layer by layer within 1e-5 with the NaN canary after the
    last utterance, and the logits within 1e-4: n = 2 (n = 1 past 20,000 input floats)."""
    n = 1 if T * Fq > 20000 else 2
    net = KwsNet(emu, arch, T, Fq, n)
    try:
        errs = check_net(net, features(_kind(T, Fq), n, T, Fq, seed=T + Fq))
        print(f"  {arch} {T}x{Fq} n={n}: worst error per layer " + " ".join(f"{e:.1e}" for e in errs))
    finally:
        net.close()


def _forward_one(net, feat, logits_out, probs_out):
    """tcr_dscnn_forward with logits or probs NULL: the outputs it was given."""
    b, n, c = net.b, feat.shape[0], net.spec.num_classes
    d_feat, logits, probs = b.upload(feat), b.empty(n, c) if logits_out else None, b.empty(n, c) if probs_out else None
    L.check(net.lib, net.lib.tcr_dscnn_forward(net.h, b.ptr(d_feat), b.ptr(net.params), n, b.ptr(logits), b.ptr(probs), b.stream),
            "tcr_dscnn_forward")
    b.sync()
    return b.download(logits) if logits_out else None, b.download(probs) if probs_out else None


def _counts(net, scores, onehot, topk):
    """tcr_dscnn_eval_accumulate into zeroed counts."""
    b, (n, c) = net.b, scores.shape
    d_s, d_h = b.upload(scores), b.upload(onehot)
    counts = np.zeros(c * c + 2, np.int64)
    if b.name == "cuda":
        counts = b.torch.from_numpy(counts).to(b.dev)
    L.check(net.lib, net.lib.tcr_dscnn_eval_accumulate(net.h, b.ptr(d_s), b.ptr(d_h), n, topk,
                                                       counts.data_ptr() if b.name == "cuda" else counts.ctypes.data, b.stream),
            "tcr_dscnn_eval_accumulate")
    b.sync()
    return counts.cpu().numpy() if b.name == "cuda" else counts


def check_classes(b, arch, T, Fq, classes, n):
    """n utterances on a handle of `classes` classes: the logits and softmax against the oracle, the logits-only and probs-only
    calls equal to the call with both, and the evaluation counts of the logits against metrics_oracle's top-k counts."""
    net = KwsNet(b, arch, T, Fq, n, seed=classes, classes=classes)
    try:
        feat = features(_kind(T, Fq), n, T, Fq, seed=classes)
        check_net(net, feat)
        logits, probs = net.forward(feat)
        assert logits.shape == probs.shape == (n, classes)
        assert np.array_equal(_forward_one(net, feat, True, False)[0], logits), "logits-only call"
        assert np.array_equal(_forward_one(net, feat, False, True)[1], probs), "probs-only call"
        onehot = np.eye(classes, dtype=np.float32)[np.random.RandomState(classes).randint(0, classes, n)]
        for topk in (1, 5):
            got = _counts(net, logits, onehot, topk)
            assert np.array_equal(got, MO.eval_counts(logits, onehot, topk)), topk
            assert got[-1] == n
    finally:
        net.close()


CLASS_COUNTS = pytest.mark.parametrize("classes", [1, 2, 17, 32])
ARCHS = pytest.mark.parametrize("arch", ["trad_fpool3", "one_fstride4"])


@ARCHS
@CLASS_COUNTS
def test_emulated_class_counts(emu, arch, classes):
    """n = 18: kws_head's groups of 16 utterances, a full one and a partial one."""
    check_classes(emu, arch, *((29, 21) if arch == "trad_fpool3" else (49, 40)), classes, 18)


# front-ends of the listener cases (tcr_config fields): 98 x 40 MFCCs, 128 log-mel bins, 41 and 42 of 64 MFCCs (history rows of
# 41 / 42 floats: rolled in floats, W1 % 3 = 1 and 2), and a clip of one window (T = 1)
LISTENER_FRONTENDS = {
    "98x40": dict(window_size_samples=480, window_stride_samples=160),
    "49x128-logmel": dict(feature_kind=L.TCR_FEATURE_LOG_MEL, num_mel_bins=128),
    "49x41": dict(num_mfccs=41, num_mel_bins=64),
    "49x42": dict(num_mfccs=42, num_mel_bins=64),
    "1x40": dict(clip_samples=640),
}
LISTENER_CASES = [(a, c) for a in ("trad_fpool3", "one_fstride4") for c in LISTENER_FRONTENDS if c != "1x40" or a == "one_fstride4"]


def _listen(b, arch, case, S, K_, pushes):
    """pushes fp32 and int16 chunks in turn, with a reset of every stream before the second to last push and of the last stream
    before the last one."""
    fe, resets = LISTENER_FRONTENDS[case], ((pushes - 2, -1), (pushes - 1, S - 1))
    if case == "1x40":                                             # clip = window: hop = K = 1
        run_listener(b, arch, S=S, hop=1, K_=1, pushes=pushes, reset_at=resets, pcm_every=2, case=fe)
    else:
        run_listener(b, arch, S=S, hop=int(case.split("x")[0]) - 1, K_=K_, pushes=pushes, reset_at=resets, pcm_every=2, case=fe)


@pytest.mark.parametrize("arch,case", LISTENER_CASES, ids=[f"{a}-{c}" for a, c in LISTENER_CASES])
def test_emulated_listener(emu, arch, case):
    """2 streams x 1 window at hop = T - 1 (hop = 1 at T = 1), 3 pushes: each push equal bit for bit to the forward on the cut
    clips, and the carried history to the front-end's frames."""
    _listen(emu, arch, case, S=2, K_=1, pushes=3)


@ARCHS
def test_emulated_set_frontend_refuses_another_geometry(emu, arch):
    """A front-end whose (T, F) is not the handle's is refused, naming both shapes."""
    rc, h = create(emu.lib, arch, 49, 41)
    try:
        c = L.TcrConfig()
        L.check(emu.lib, emu.lib.tcr_config_default(C.byref(c)), "tcr_config_default")   # 49 x 40 MFCCs
        assert emu.lib.tcr_dscnn_set_frontend(h, C.byref(c)) == TCR_ERR_INVALID
        assert "(T, F) = (49, 40)" in emu.lib.tcr_last_error().decode() and "(49, 41)" in emu.lib.tcr_last_error().decode()
        c.num_mfccs, c.num_mel_bins = 41, 64
        L.check(emu.lib, emu.lib.tcr_dscnn_set_frontend(h, C.byref(c)), "tcr_dscnn_set_frontend")
    finally:
        emu.lib.tcr_dscnn_destroy(h)


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


def _report(net, feat):
    errs = check_layers(net, feat)
    print(f"  {net.arch} {net.spec.h}x{net.spec.w} n={feat.shape[0]}: " + " ".join(
        f"{'+'.join(k)} {e:.1e}" for k, e in zip(KERNELS[net.arch], errs)))


@pytest.mark.gpu
@pytest.mark.parametrize("arch,T,Fq,claims,why", GEOMETRIES, ids=IDS)
def test_cuda_layers_logits_and_invariance(cuda, arch, T, Fq, claims, why):
    """Each conv layer within 1e-5 with the kernels it launches named, the logits within 1e-4, at n = 1, 3, 39 and 100 (n = 1, 3
    at 400 x 128 trad_fpool3); then the logits of the largest batch are the same bits repeated, permuted, sliced and on a handle
    with another max_batch."""
    ns = (1, 3) if (arch, T, Fq) in BIG else (1, 3, 39, 100)
    net = KwsNet(cuda, arch, T, Fq, 128, seed=1)
    other = KwsNet(cuda, arch, T, Fq, ns[-1], seed=1)
    try:
        for n in ns:
            feat = features(_kind(T, Fq), n, T, Fq, seed=n)
            _report(net, feat)
        check_invariance(net, feat, other)
    finally:
        net.close()
        other.close()


def _tiles(arch, T, Fq, n):
    r = reach(arch, T, Fq)
    return -(-n * r["conv1_rows"] // C1_TILE), -(-n * r["conv2_rows"] // C2_TILE)


@pytest.mark.gpu
@pytest.mark.parametrize("T,Fq", [(29, 19), (49, 23), (49, 40)], ids=["29x19", "49x23", "49x40"])
def test_cuda_persistent_grid_sweep(cuda, T, Fq):
    """kws_conv1_tc and kws_conv2_tc walk tiles with a stride of min(tiles, SMs): for each kernel, the last batch with fewer tiles
    than SMs and the first with at least SMs, SMs + 1 and 2 x SMs + 1 tiles (exactly, where a batch lands there), layer by layer against the oracle; then the largest batch with every
    conv's output channels scaled by 10^U(-2, 2), so that conv2's K = 256 fold runs away from unit-scale weights."""
    sms, r = _sms(), reach("trad_fpool3", T, Fq)
    ns = set()
    for kernel, (rows, tile) in enumerate(((r["conv1_rows"], C1_TILE), (r["conv2_rows"], C2_TILE))):
        for target in (sms, sms + 1, 2 * sms + 1):
            n = -(-(target - 1) * tile // rows)                    # the first n with ceil(n * rows / tile) >= target
            while -(-n * rows // tile) < target:
                n += 1
            ns |= {n, n - 1} if target == sms else {n}            # n - 1: the last batch below the SM count
    ns = sorted(ns)
    print(f"  {sms} SMs, trad_fpool3 {T}x{Fq}: (n, conv1 tiles, conv2 tiles) "
          + " ".join(str((n,) + _tiles("trad_fpool3", T, Fq, n)) for n in ns))
    net = KwsNet(cuda, "trad_fpool3", T, Fq, ns[-1], seed=2)
    try:
        for n in ns:
            _report(net, features("randn", n, T, Fq, seed=n))
        net.p = wide_range(net.spec, net.p)
        net.params = cuda.upload(K.flatten(net.spec, net.p))
        _report(net, features("randn", ns[-1], T, Fq, seed=1))
    finally:
        net.close()


@pytest.mark.gpu
@ARCHS
@CLASS_COUNTS
def test_cuda_class_counts(cuda, arch, classes):
    """n = 37 at 49 x 40: kws_head's groups of 16 utterances, two full and a partial one."""
    check_classes(cuda, arch, 49, 40, classes, 37)


@pytest.mark.gpu
@pytest.mark.parametrize("arch,case", LISTENER_CASES, ids=[f"{a}-{c}" for a, c in LISTENER_CASES])
def test_cuda_listener(cuda, arch, case):
    """13 streams x 3 windows at hop = T - 1 (7 streams x 1 window at T = 1), 5 pushes: each push equal bit for bit to the forward on
    the cut clips, and the push's first layer is the windowed kernel."""
    _listen(cuda, arch, case, S=13 if case != "1x40" else 7, K_=3, pushes=5)


@pytest.mark.gpu
@pytest.mark.parametrize("arch,flags,bound", [
    ("trad_fpool3", dict(num_mfccs=10), "width >= 19"),
    ("one_fstride4", dict(preprocess_method="log_mel_spectrogram", num_mel_bins=128, window_size_ms=30.0, window_stride_ms=1.0),
     "height x width <= 51200")], ids=["trad_fpool3-10-mfccs", "one_fstride4-971x128-logmel"])
def test_cuda_refusals_through_the_model_class(cuda, arch, flags, bound):
    """KWSModel refuses a front-end its net cannot take, naming the bound (971 x 128 log-mel frames for one_fstride4)."""
    from tcresnet_b200._lib import TcrError
    from tcresnet_b200.factory import audio_nets
    from tcresnet_b200.runtime import Node
    args = dict(num_classes=12, sample_rate=16000, clip_duration_ms=1000, window_size_ms=40.0, window_stride_ms=20.0,
                num_mel_bins=64, num_mfccs=40, lower_edge_hertz=80.0, upper_edge_hertz=7600.0, preprocess_method="mfcc",
                batch_size=3, output_name="output/softmax", weight_decay=1e-4, architecture=arch)
    args.update(flags)
    model = audio_nets.KWSModel(argparse.Namespace(**args), None)
    with pytest.raises(TcrError, match=rf"status 3\): {arch} needs .*{bound}"):
        model.build(Node("wavs", [None, 16000, 1]), Node("labels", [None, 12]), False)


@pytest.mark.gpu
@ARCHS
def test_cuda_tc_mode_leaves_kws_kernels_unchanged(cuda, monkeypatch, arch):
    """TCR_DSCNN_TC selects DS-CNN's kernels only: unset, 0 and 1 launch the same KWS kernels (trad_fpool3's wgmma kernels have no
    FMA twin) and give the same logits bit for bit."""
    feat = features("mfcc", 39, 49, 40, seed=4)
    runs = []
    for mode in (None, "0", "1"):
        if mode is None:
            monkeypatch.delenv("TCR_DSCNN_TC", raising=False)
        else:
            monkeypatch.setenv("TCR_DSCNN_TC", mode)
        net = KwsNet(cuda, arch, 49, 40, 39, seed=3)
        try:
            got = {}
            counts = launched(cuda.lib, lambda: got.setdefault("out", net.forward(feat)))
            runs.append((sorted(counts), got["out"][0]))
        finally:
            net.close()
    assert runs[0][0] == sorted(sum(KERNELS[arch], []) + ["kws_lin", "kws_head"]), runs[0][0]
    for names, logits in runs[1:]:
        assert names == runs[0][0] and np.array_equal(logits, runs[0][1])
    assert rel_err(runs[0][1], K.forward(K.build_spec(arch, 49, 40), K.init_variables(K.build_spec(arch, 49, 40), 3),
                                         feat.astype(np.float64))) <= 1e-4
