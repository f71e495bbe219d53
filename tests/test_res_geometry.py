"""Honk's ResNets (Res8 / Res8Narrow / Res15 / Res15Narrow) at the edges of every geometry, batch and class count their DS-CNN handle
accepts, against the fp64 oracle (res_oracle): the row-width refusal at the register tiles' width, the parameter table and FLOPs,
each layer and the logits at each row of GEOMETRIES, res_conv's persistent tile walk against the grid, 1 to 32 classes with the
logits-only / probs-only calls and the evaluation counts, the listener at more front-ends, and TCR_DSCNN_TC.  Every kernel runs on
the CPU emulator (one CTA walks every tile there, and cp.async is a plain copy) and on the GPU."""
import numpy as np
import pytest

from oracle import metrics_oracle as MO
from oracle import res_oracle as R
from tcr_harness import NumpyBackend, launched, rel_err
from test_dscnn import _sms, check_invariance, features, wide_range
from test_kws_geometry import _counts, _forward_one
from test_res import TCR_ERR_UNSUPPORTED, ResNet, check_net, create, table
from test_res_eval import check_layers, run_listener

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L

THREADS = 256                                   # kResConvThreads, and res_fconv's block
TILE = {48: (4, 4), 20: (1, 2)}                 # ResTile<CP>: channel lanes per position (CGW), positions per thread (TM)
FCONV_TARGET, SMEM_LIMIT = 100 * 1024, 227 * 1024


def reach(model, T, Fq):
    """The handle's plan (tcr_dscnn.cu, res_create), restated.  Blocks: the H x W map the convs run on; npmax, the positions of a
    res_conv CTA's register tiles, and slots, the positions one pass of them covers (a thread's TM positions are `slots` apart);
    TR rows per tile, as many whole rows as npmax covers, then balanced over tpu tiles per utterance; last, the last tile's rows;
    busy, the position lanes a full tile fills.  f_conv: RH output rows per CTA (8, fewer while the staged rows pass 100 KB),
    f_tiles per utterance, f_smem bytes, and f_row, the padded input row its staging walk steps through."""
    r8, narrow = model.startswith("Res8"), model.endswith("Narrow")
    c, cp = (19, 20) if narrow else (45, 48)
    H, W = (T - 3, Fq - 2) if r8 else (T, Fq)
    cgw, tm = TILE[cp]
    slots = THREADS // 32 * (32 // cgw)
    npmax = slots * tm
    ph = 4 if r8 else 1

    def f_smem(rh):
        cr = rh + ph - 1
        return 4 * ((cr + 2) * (Fq + 2) + (cr * Fq * c if ph > 1 else 0) + 9 * c)
    RH = min(H, 8)
    while RH > 1 and f_smem(RH) > FCONV_TARGET:
        RH -= 1
    out = dict(H=H, W=W, npmax=npmax, slots=slots, RH=RH, f_tiles=-(-H // RH), f_smem=f_smem(RH), f_row=Fq + 2)
    if W > npmax:
        return out
    TR = min(H, npmax // W)
    tpu = -(-H // TR)
    TR = -(-H // tpu)
    xs = cp if (cp >> 2) & 1 else cp + 4
    return dict(out, TR=TR, tpu=tpu, last=H - (tpu - 1) * TR, busy=TR * W, smem=4 * (9 * cp * cp + 3 * cp + 2 * TR * W * xs))


# (model, T, F, what the row reaches (checked against reach()), why it is here)
GEOMETRIES = [
    ("Res15", 1, 256, dict(W=256, npmax=256, TR=1, tpu=1, busy=256, f_row=258),
     "W = npmax: every position lane busy; f_conv's padded row is wider than its 256 threads; every vertical tap reads padding"),
    ("Res15", 3, 256, dict(TR=1, tpu=3, busy=256), "TR = 1, three tiles: each tap row reads a neighbouring tile's row"),
    ("Res15", 3, 129, dict(W=129, TR=1, tpu=3, busy=129, slots=64),
     "W = npmax / 2 + 1: half the position lanes idle, a row spans three register slots"),
    ("Res15", 16, 16, dict(TR=16, tpu=1, busy=256), "one tile, every lane busy; rate 16's off-centre taps read only padding"),
    ("Res15", 17, 17, dict(TR=9, tpu=2, last=8), "rate 16 reaches exactly one row and column into the map; tiles of 9 + 8 rows"),
    ("Res15", 257, 1, dict(W=1, TR=129, tpu=2, last=128, RH=8, f_tiles=33), "W = 1: every column tap is padding; 129 + 128 rows"),
    ("Res15", 61, 128, dict(TR=2, tpu=31, last=1), "TR = 2 and a last tile of one row"),
    ("Res15", 998, 128, dict(TR=2, tpu=499, last=2, busy=256),
     "the largest map test_res.test_refusals accepts: 499 tiles per utterance, more than the grid at n = 1; the head averages "
     "127,744 positions"),
    ("Res15Narrow", 2, 512, dict(W=512, npmax=512, TR=1, tpu=2, busy=512, f_row=514), "W = npmax at CP = 20"),
    ("Res15Narrow", 3, 257, dict(W=257, TR=1, tpu=3, busy=257, slots=256), "W = npmax / 2 + 1 at CP = 20"),
    ("Res15Narrow", 33, 16, dict(TR=17, tpu=2, last=16), "TR = 17 (17 + 16); dilation 16 equals W"),
    ("Res15Narrow", 61, 128, dict(TR=4, tpu=16, last=1), "a last tile of one row at CP = 20"),
    ("Res8", 4, 258, dict(H=1, W=256, TR=1, RH=1, f_smem=193620, f_row=260),
     "the widest Res8: pooled W = npmax; f_conv at RH = 1 on 189 KB of shared memory (the opt-in past 100 KB), padded row 260"),
    ("Res8", 12, 131, dict(H=9, W=129, RH=1, f_tiles=9, f_smem=99132, TR=1, tpu=9),
     "f_conv's RH shrinks to 1 (97 KB), nine f_conv tiles; blocks at W = 129, TR = 1"),
    ("Res8Narrow", 4, 514, dict(W=512, TR=1, RH=1, f_smem=169324), "pooled W = npmax at CP = 20; f_conv at 165 KB"),
    ("Res8Narrow", 101, 130, dict(H=98, W=128, RH=6, f_tiles=17, TR=4, tpu=25, last=2),
     "f_conv at RH = 6 with a partial last tile (98 = 16 x 6 + 2); blocks at TR = 4 with a last tile of 2 rows"),
]
IDS = [f"{m}-{t}x{f}" for m, t, f, _, _ in GEOMETRIES]
BIG = {("Res15", 998, 128)}                     # 13 dilated convs over 127,744 positions: hours on the emulator; n = 1 and 2 on the GPU


@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


def _err(lib):
    return lib.tcr_last_error().decode()


@pytest.mark.parametrize("model,T,Fq,npmax", [("Res15", 1, 256, 256), ("Res15Narrow", 2, 512, 512), ("Res8", 4, 258, 256),
                                              ("Res8Narrow", 4, 514, 512)])
def test_row_width_refusal_sits_at_npmax(emu, model, T, Fq, npmax):
    """The widest block map the handle accepts is the register tiles' width: one column more is refused at tcr_dscnn_create,
    naming both widths, and reach() agrees on npmax."""
    assert reach(model, T, Fq)["npmax"] == npmax and reach(model, T, Fq)["W"] == npmax
    rc, h = create(emu.lib, model, T, Fq)
    assert rc == 0, _err(emu.lib)
    emu.lib.tcr_dscnn_destroy(h)
    rc, h = create(emu.lib, model, T, Fq + 1)
    assert rc == TCR_ERR_UNSUPPORTED and not h.value
    assert f"res_conv tiles whole rows of at most {npmax} positions; the blocks' map is {npmax + 1} wide" in _err(emu.lib), _err(emu.lib)


@pytest.mark.parametrize("model,T,Fq,claims,why", GEOMETRIES, ids=IDS)
def test_table_and_flops(emu, model, T, Fq, claims, why):
    """Each row reaches what it claims; tcr_dscnn_param_table and the FLOP count against res_oracle."""
    got = reach(model, T, Fq)
    assert {k: got[k] for k in claims} == claims, (why, got)
    assert got["smem"] <= SMEM_LIMIT and got["f_smem"] <= SMEM_LIMIT
    rc, h = create(emu.lib, model, T, Fq)
    assert rc == 0, _err(emu.lib)
    try:
        rows, nparams, flops = table(emu.lib, h)
        spec = R.build_spec(model, T, Fq)
        assert [(n, s) for n, s, _ in rows] == [(n, spec.var_shapes[n]) for n in spec.var_names]
        assert nparams == sum(int(np.prod(s)) for s in spec.var_shapes.values()) and flops == R.forward_flops(spec)
        assert R.block_map(spec) == (got["H"], got["W"])
    finally:
        emu.lib.tcr_dscnn_destroy(h)


@pytest.mark.parametrize("model,T,Fq,claims,why", [g for g in GEOMETRIES if g[:3] not in BIG],
                         ids=[i for g, i in zip(GEOMETRIES, IDS) if g[:3] not in BIG])
def test_emulated_layers_and_logits(emu, model, T, Fq, claims, why):
    """res_fconv, res_conv in both residual modes at every dilation, and the head, layer by layer within 1e-5 with the NaN canary
    after the last utterance, and the logits within 1e-4: n = 2 (n = 1 past 4,000 input floats)."""
    n = 1 if T * Fq > 4000 else 2
    net = ResNet(emu, model, T, Fq, n, seed=T + Fq)
    try:
        errs, _ = check_net(net, features("randn", n, T, Fq, seed=T + Fq))
        print(f"  {model} {T}x{Fq} n={n}: error per layer " + " ".join(f"{e:.1e}" for e in errs.values()))
    finally:
        net.close()


def check_classes(b, model, T, Fq, classes, n):
    """n utterances on a handle of `classes` classes: the logits and softmax against the oracle, the logits-only and probs-only
    calls equal to the call with both, and the evaluation counts of the logits against metrics_oracle's top-k counts."""
    net = ResNet(b, model, T, Fq, n, seed=classes, classes=classes)
    try:
        feat = features("randn", n, T, Fq, seed=classes)
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
NARROW = pytest.mark.parametrize("model", ["Res8Narrow", "Res15Narrow"])


@NARROW
@CLASS_COUNTS
def test_emulated_class_counts(emu, model, classes):
    """n = 5 on small maps (Res8Narrow 9 x 6, Res15Narrow 13 x 8)."""
    check_classes(emu, model, *((9, 6) if model == "Res8Narrow" else (13, 8)), classes, 5)


# front-ends of the listener cases (tcr_config fields), keyed T x F: 128 log-mel bins (Res8's windowed f_conv at RH = 1,
# Res8Narrow's at RH = 7), 41 and 42 of 64 MFCCs (odd and even history rows), and a clip of the smallest height each model takes
LISTENER_FRONTENDS = {
    "49x128-logmel": dict(feature_kind=L.TCR_FEATURE_LOG_MEL, num_mel_bins=128),
    "49x41": dict(num_mfccs=41, num_mel_bins=64),
    "49x42": dict(num_mfccs=42, num_mel_bins=64),
    "1x40": dict(clip_samples=640),
    "4x40": dict(clip_samples=1600),
}
LISTENER_CASES = [(m, c) for m in R.MODELS for c in LISTENER_FRONTENDS
                  if c not in ("1x40", "4x40") or (c == "4x40") == m.startswith("Res8")]


def _listen(b, model, case, S, K_, pushes):
    """pushes fp32 and int16 chunks in turn, with a reset of every stream before the second to last push and of the last stream
    before the last one; hop = T - 1 (hop = K = 1 at T = 1)."""
    T = int(case.split("x")[0])
    resets = ((pushes - 2, -1), (pushes - 1, S - 1))
    run_listener(b, model, S=S, hop=max(1, T - 1), K_=1 if T == 1 else K_, pushes=pushes, reset_at=resets, pcm_every=2,
                 case=LISTENER_FRONTENDS[case])


@pytest.mark.parametrize("model,case", LISTENER_CASES, ids=[f"{m}-{c}" for m, c in LISTENER_CASES])
def test_emulated_listener(emu, model, case):
    """2 streams x 1 window (1 stream at C = 45 on 49 frames: the emulator's slowest forwards), 3 pushes: each push equal bit for
    bit to the forward on the cut clips, and the carried history to the front-end's frames."""
    _listen(emu, model, case, S=1 if not model.endswith("Narrow") and case.startswith("49x") else 2, K_=1, pushes=3)


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


ORACLE_POSITIONS = 200_000     # the fp64 oracle checks every utterance up to this many input positions, a slice from both ends past it


def _rows(n, T, Fq):
    k = max(1, ORACLE_POSITIONS // (T * Fq))
    return None if k >= n else np.r_[0:k // 2, n - (k - k // 2):n]


WORST = {}


def _report(net, feat, where):
    """check_layers with the oracle on _rows, and the worst error per kernel kept for the summary."""
    n, spec = feat.shape[0], net.spec
    errs, _ = check_layers(net, feat, _rows(n, spec.h, spec.w))
    kinds = {}
    for k, e in errs.items():
        kind = "logits" if k == "logits" else "res_fconv" if k == 1 else ("res_conv_res" if (k - 2) % 2 else "res_conv")
        kinds[kind] = max(kinds.get(kind, 0.0), e)
        if e >= WORST.get(kind, (0.0,))[0]:
            WORST[kind] = (e, f"{where} n={n}")
    print(f"  {where} n={n}: " + " ".join(f"{k} {e:.1e}" for k, e in sorted(kinds.items())))


@pytest.fixture(scope="module")
def worst_errors():
    yield WORST
    print("\n  worst error per kernel: " + "; ".join(f"{k} {e:.1e} ({w})" for k, (e, w) in sorted(WORST.items())))


@pytest.mark.gpu
@pytest.mark.parametrize("model,T,Fq,claims,why", GEOMETRIES, ids=IDS)
def test_cuda_layers_logits_and_invariance(cuda, worst_errors, model, T, Fq, claims, why):
    """Each layer within 1e-5 with the kernels it launches named, the logits within 1e-4, at n = 1, 3, 39 and 100 (n = 1 and 2 at
    998 x 128); then the logits of the largest batch are the same bits repeated, permuted, sliced and on a handle with another
    max_batch."""
    ns = (1, 2) if (model, T, Fq) in BIG else (1, 3, 39, 100)
    net = ResNet(cuda, model, T, Fq, ns[-1] + 3, seed=1)
    other = ResNet(cuda, model, T, Fq, ns[-1], seed=1)
    try:
        for n in ns:
            _report(net, features("randn", n, T, Fq, seed=n), f"{model} {T}x{Fq}")
        check_invariance(net, features("randn", ns[-1], T, Fq, seed=ns[-1]), other)
    finally:
        net.close()
        other.close()


# (model, T, F) of the persistent-grid sweep: the recipe's map (17 tiles per utterance, one CTA per SM), a map small enough for
# two res_conv CTAs per SM (106 KB of shared memory, one tile per utterance), and a Narrow map of two tiles per utterance
SWEEP = [("Res15", 98, 40), ("Res15", 6, 10), ("Res15Narrow", 33, 16)]


def sweep_batches(sms, tpu):
    """For p = 1, 2, 3 CTAs per SM: the batches whose tile count n * tpu is just below, at, one past and 2x + 1 past sms * p (the
    first n with at least that many tiles, and the last n below sms * p)."""
    ns = set()
    for p in (1, 2, 3):
        for target in (sms * p, sms * p + 1, 2 * sms * p + 1):
            n = -(-target // tpu)
            ns |= {n, n - 1} if target == sms * p else {n}
    return sorted(x for x in ns if x >= 1)


@pytest.mark.gpu
@pytest.mark.parametrize("model,T,Fq", SWEEP, ids=[f"{m}-{t}x{f}" for m, t, f in SWEEP])
def test_cuda_persistent_grid_sweep(cuda, worst_errors, model, T, Fq):
    """res_conv walks n * tpu tiles with a grid of min(tiles, SMs * CTAs per SM): layer by layer against the oracle at the batches
    of sweep_batches; then the largest batch with every weight bank's output channels and every moving variance spread over four
    decades (test_dscnn.wide_range)."""
    sms, tpu = _sms(), reach(model, T, Fq)["tpu"]
    assert reach("Res15", 6, 10)["smem"] < 110 * 1024
    ns = sweep_batches(sms, tpu)
    print(f"  {sms} SMs, {model} {T}x{Fq} (tpu {tpu}): (n, tiles) " + " ".join(str((n, n * tpu)) for n in ns))
    net = ResNet(cuda, model, T, Fq, ns[-1], seed=2)
    try:
        for n in ns:
            _report(net, features("randn", n, T, Fq, seed=n), f"sweep {model} {T}x{Fq}")
        net.p = wide_range(net.spec, net.p)
        net.params = cuda.upload(R.flatten(net.spec, net.p))
        _report(net, features("randn", ns[-1], T, Fq, seed=1), f"sweep {model} {T}x{Fq} wide-range")
    finally:
        net.close()


@pytest.mark.gpu
@NARROW
@CLASS_COUNTS
def test_cuda_class_counts(cuda, model, classes):
    """n = 37 at 98 x 40."""
    check_classes(cuda, model, 98, 40, classes, 37)


@pytest.mark.gpu
@pytest.mark.parametrize("model,case", LISTENER_CASES, ids=[f"{m}-{c}" for m, c in LISTENER_CASES])
def test_cuda_listener(cuda, model, case):
    """13 streams x 3 windows at hop = T - 1 (7 streams x 1 window at T = 1), 5 pushes: each push equal bit for bit to the forward on
    the cut clips, and the push's first kernel is res_fconv:win."""
    _listen(cuda, model, case, S=13 if case != "1x40" else 7, K_=3, pushes=5)


@pytest.mark.gpu
@pytest.mark.parametrize("model", R.MODELS)
def test_cuda_tc_mode_leaves_res_kernels_unchanged(cuda, monkeypatch, model):
    """TCR_DSCNN_TC selects DS-CNN's kernels only: unset, 0 and 1 launch the same Res kernels and give the same logits bit for bit."""
    feat = features("mfcc", 39, 98, 40, seed=4)
    runs = []
    for mode in (None, "0", "1"):
        if mode is None:
            monkeypatch.delenv("TCR_DSCNN_TC", raising=False)
        else:
            monkeypatch.setenv("TCR_DSCNN_TC", mode)
        net = ResNet(cuda, model, 98, 40, 39, seed=3)
        try:
            got = {}
            counts = launched(cuda.lib, lambda: got.setdefault("out", net.forward(feat)))
            runs.append((dict(counts), got["out"][0]))
        finally:
            net.close()
    nl = R.build_spec(model).layers
    assert runs[0][0] == {"res_fconv": 1, "res_conv": (nl + 1) // 2, "res_conv_res": nl // 2, "res2d_head": 1}, runs[0][0]
    for names, logits in runs[1:]:
        assert names == runs[0][0] and np.array_equal(logits, runs[0][1])
    spec = R.build_spec(model)
    assert rel_err(runs[0][1], R.forward(spec, R.init_variables(spec, 3), feat.astype(np.float64))) <= 1e-4
