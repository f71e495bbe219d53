"""KWSModel's speech_commands nets (low_latency_conv, tiny_conv) at the edges of every geometry, batch and class count their DS-CNN
handle accepts, against the fp64 oracle (kws_small_oracle): reach() restates the handle's plan (kwsb_define) on plain integers and
is checked against the handle's width bound at every height class; the parameter table, the conv and the logits at each row of
GEOMETRIES (kws_tinyconv's shared-memory opt-in and its 227 KB limit, kws_llconv's single K step and tile edges, kws_fcs's K chunk
edges), 1 to 32 classes, weights of unequal scale held per channel, the listener at more front-ends, and the refusals.  Every kernel
on the CPU emulator; on the GPU with the launched kernels named, batch invariance and the TCR_DSCNN_TC switch."""
import argparse

import numpy as np
import pytest

import kws_small_oracle as S
from oracle import metrics_oracle as MO
from tcr_harness import NumpyBackend, launched, rel_err
from test_dscnn import check_invariance, features, wide_range
from test_kws_geometry import LISTENER_FRONTENDS, _counts, _forward_one, _kind
from test_kws_small import TCR_ERR_UNSUPPORTED, SmallNet, check_small, create, expected_table, table
from test_kws_small_eval import CONV, check_cuda, run_listener

import tcresnet_b200  # noqa: F401

LL_BM, LL_KC = 128, 128                 # kws_llconv's rows per CTA; kws_fcs's K chunk for low_latency_conv
TINY_RH, TINY_KC = 8, 256               # kws_tinyconv's output rows per CTA at most; kws_fcs's K chunk for tiny_conv
TINY_FIXED = 10 * 8 * 8 + 8             # kws_tinyconv's staged taps (10 x 8 x 8 channels) and biases, in floats
SMEM_DEFAULT, SMEM_LIMIT = 48 * 1024, 227 * 1024    # dynamic shared memory per block without the opt-in, and sm_90's opt-in limit
ARCHS = ["low_latency_conv", "tiny_conv"]


def reach(arch, T, Fq, n=1):
    """What a geometry exercises, restated from kwsb_define and the kernels.  low_latency_conv: W = F - 7 output columns, ksteps = T
    filter rows kws_llconv walks (one staged per step, the next prefetched), m_tiles, the 128-row tiles of M = n x W rows.
    tiny_conv: the SAME output (hout, wout) and pads (above, below, left, right); rh = min(hout, 8), the output rows of a CTA,
    tiles of them per utterance and the rows of the last; smem, the bytes kws_tinyconv stages ((2 rh + 8) input rows of 2 wout + 6
    columns, and the taps and biases), optin whether that passes the 48 KB a kernel gets without the opt-in, fits whether it is
    within 227 KB.  Both: k, the flattened conv output kws_fcs splits into chunks of 128 / 256, and the last chunk's k_tail (0: all
    chunks full)."""
    if arch == "low_latency_conv":
        W = Fq - 7
        k = W * 186
        return dict(W=W, ksteps=T, m_tiles=-(-n * W // LL_BM), k=k, chunks=-(-k // LL_KC), k_tail=k % LL_KC, fits=W >= 1)
    hout, pt, pb = S.same_pad(T, 10, 2)
    wout, pl, pr = S.same_pad(Fq, 8, 2)
    rh = min(hout, TINY_RH)
    tiles = -(-hout // rh)
    smem = 4 * (TINY_FIXED + (2 * rh + 8) * (2 * wout + 6))
    k = hout * wout * 8
    return dict(hout=hout, wout=wout, pads=(pt, pb, pl, pr), rh=rh, tiles=tiles, last_rows=hout - (tiles - 1) * rh, smem=smem,
                optin=smem > SMEM_DEFAULT, fits=smem <= SMEM_LIMIT, k=k, chunks=-(-k // TINY_KC), k_tail=k % TINY_KC)


def widest(T):
    """The widest F reach() accepts for tiny_conv at height T (staged bytes grow with F, so a bisection)."""
    lo, hi = 1, 1 << 16
    assert reach("tiny_conv", T, lo)["fits"] and not reach("tiny_conv", T, hi)["fits"]
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if reach("tiny_conv", T, mid)["fits"] else (lo, mid)
    return lo


BOUND_HEIGHTS = list(range(1, 18)) + [49, 98]


@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


def _err(lib):
    return lib.tcr_last_error().decode()


def _accepted(lib, arch, T, Fq):
    rc, h = create(lib, arch, T, Fq)
    assert rc == 0, (arch, T, Fq, _err(lib))
    lib.tcr_dscnn_destroy(h)


def test_reach_matches_the_handles_width_bound(emu):
    """tiny_conv: at every T from 1 to 17 (rh = 1 .. 8 and the first tiles past 8 rows) and at 49 and 98, the widest F reach()
    accepts is accepted and F + 1 is refused, the message quoting reach()'s bytes; the bound falls with rh up to T = 15 and holds
    from there on; 13 x 2606 needs exactly the 227 KB limit and is accepted.  low_latency_conv: width 8 accepted, 7 refused."""
    lib, bounds = emu.lib, {}
    for T in BOUND_HEIGHTS:
        Fw = bounds[T] = widest(T)
        _accepted(lib, "tiny_conv", T, Fw)
        rc, h = create(lib, "tiny_conv", T, Fw + 1)
        assert rc == TCR_ERR_UNSUPPORTED and not h.value
        assert _err(lib) == (f"kws_tinyconv needs {reach('tiny_conv', T, Fw + 1)['smem']} bytes of shared memory at width {Fw + 1}, "
                             f"the limit is {SMEM_LIMIT}"), (T, _err(lib))
        _accepted(lib, "low_latency_conv", T, 8)
        rc, h = create(lib, "low_latency_conv", T, 7)
        assert rc == TCR_ERR_UNSUPPORTED and "width >= 8" in _err(lib) and not h.value
    print("  widest tiny_conv width per height: " + ", ".join(f"{T}: {F}" for T, F in bounds.items()))
    assert all(bounds[T] >= bounds[T + 1] for T in range(1, 17)) and bounds[15] == bounds[16] == bounds[17] == bounds[49] == bounds[98]
    assert bounds[1] == bounds[2] > bounds[3] and bounds[13] == 2606
    assert reach("tiny_conv", 13, 2606)["smem"] == SMEM_LIMIT
    _accepted(lib, "tiny_conv", 13, 2606)


# (arch, T, F, what the row reaches (checked against reach()), why it is here)
GEOMETRIES = [
    ("tiny_conv", 1, 1, dict(hout=1, wout=1, pads=(4, 5, 3, 4), rh=1, k=8, chunks=1, k_tail=8), "one output, all but 1 of 80 taps padding"),
    ("tiny_conv", 8, 16, dict(hout=4, rh=4, tiles=1, k=256, chunks=1, k_tail=0), "K exactly one kws_fcs chunk"),
    ("tiny_conv", 6, 22, dict(hout=3, wout=11, k=264, chunks=2, k_tail=8), "K one chunk plus 8"),
    ("tiny_conv", 16, 16, dict(hout=8, rh=8, tiles=1, last_rows=8, pads=(4, 4, 3, 3)), "hout = 8: one full tile"),
    ("tiny_conv", 17, 40, dict(hout=9, tiles=2, last_rows=1, pads=(4, 5, 3, 3)), "a last tile of one row"),
    ("tiny_conv", 33, 40, dict(hout=17, tiles=3, last_rows=1), "two full tiles and a last of one row"),
    ("tiny_conv", 49, 478, dict(smem=49056, optin=False), "the widest staging without the opt-in"),
    ("tiny_conv", 49, 479, dict(smem=49248, optin=True), "the narrowest staging that needs the opt-in"),
    ("tiny_conv", 15, 2388, dict(rh=8, tiles=1, smem=232416, optin=True), "the widest F at rh = 8, one tile"),
    ("tiny_conv", 49, 2388, dict(rh=8, tiles=4, last_rows=1, k=238800), "the widest F at rh = 8, four tiles"),
    ("tiny_conv", 13, 2606, dict(hout=7, rh=7, tiles=1, smem=SMEM_LIMIT), "exactly 227 KB of shared memory"),
    ("tiny_conv", 1, 5740, dict(hout=1, rh=1, smem=232432, pads=(4, 5, 3, 3)), "rh = 1: the widest F accepted"),
    ("tiny_conv", 2, 5739, dict(hout=1, rh=1, wout=2870, pads=(4, 4, 3, 4)), "rh = 1, an even T and an odd F"),
    ("low_latency_conv", 1, 8, dict(W=1, ksteps=1, k=186, chunks=2, k_tail=58), "T = 1: a single K step, no prefetch"),
    ("low_latency_conv", 2, 8, dict(W=1, ksteps=2), "one prefetched K step"),
    ("low_latency_conv", 1, 135, dict(W=128, ksteps=1, m_tiles=1), "an utterance is exactly one 128-row tile"),
    ("low_latency_conv", 49, 134, dict(W=127, m_tiles=1), "one row short of a tile: utterances straddle tiles"),
    ("low_latency_conv", 49, 136, dict(W=129, m_tiles=2), "one row past a tile"),
    ("low_latency_conv", 49, 71, dict(W=64, k=11904, chunks=93, k_tail=0), "K = 93 full kws_fcs chunks, no tail"),
    ("low_latency_conv", 49, 1031, dict(W=1024, k=190464, chunks=1488, k_tail=0), "W = 1,024: eight tiles an utterance"),
    ("low_latency_conv", 6400, 8, dict(W=1, ksteps=6400, k=186), "6,400 K steps: 51,200 taps in one fmaf chain"),
]
IDS = [f"{'C' if a == 'low_latency_conv' else 'Y'}-{t}x{f}" for a, t, f, _, _ in GEOMETRIES]
# the slowest rows on the emulator (seconds an utterance): one utterance there, and on the GPU the oracle checks a slice of the batch
BIG = {("low_latency_conv", 49, 1031), ("low_latency_conv", 6400, 8)}
# rerun on the GPU with wide-range weights, each conv channel held to its own maximum
WIDE = {("tiny_conv", 49, 478), ("tiny_conv", 49, 479), ("tiny_conv", 13, 2606), ("tiny_conv", 1, 5740), ("low_latency_conv", 1, 135),
        ("low_latency_conv", 49, 71), ("low_latency_conv", 49, 1031)}


@pytest.mark.parametrize("arch,T,Fq,claims,why", GEOMETRIES, ids=IDS)
def test_table_and_flops(emu, arch, T, Fq, claims, why):
    """Each row is accepted and reaches what it claims; tcr_dscnn_param_table and the FLOP count against the formulas and
    kws_small_oracle."""
    got = reach(arch, T, Fq)
    assert got["fits"] and {k: got[k] for k in claims} == claims, (why, got)
    rc, h = create(emu.lib, arch, T, Fq)
    assert rc == 0, _err(emu.lib)
    try:
        rows, nparams, flops = table(emu.lib, h)
        exp_rows, exp_params, exp_flops = expected_table(arch, T, Fq)
        assert [(n, s) for n, s, _ in rows] == exp_rows
        assert (nparams, flops) == (exp_params, exp_flops)
        spec = S.build_spec(arch, T, Fq)
        assert [spec.var_shapes[n] for n in spec.var_names] == [s for _, s in exp_rows] and S.forward_flops(spec) == flops
        assert int(np.prod(S.conv_geometry(arch, T, Fq)[0])) == got["k"]
    finally:
        emu.lib.tcr_dscnn_destroy(h)


@pytest.mark.parametrize("arch,T,Fq,claims,why", GEOMETRIES, ids=IDS)
def test_emulated_conv_and_logits(emu, arch, T, Fq, claims, why):
    """The conv within 1e-5 of its maximum with the NaN canary after the last utterance, and the logits within 1e-4: n = 2 (n = 1
    at the BIG rows); tiny_conv also on positive inputs, so that every dropped or misplaced zero of the padding shows."""
    n = 1 if (arch, T, Fq) in BIG else 2
    net = SmallNet(emu, arch, T, Fq, n, seed=T + Fq)
    try:
        errs = check_small(net, features(_kind(T, Fq), n, T, Fq, seed=T + Fq))
        if arch == "tiny_conv":
            check_small(net, (np.random.RandomState(T * Fq).rand(n, T, Fq) + 0.5).astype(np.float32))
        print(f"  {arch} {T}x{Fq} n={n}: conv {errs[0]:.1e} logits {errs[1]:.1e}")
    finally:
        net.close()


WIDE_ROWS = sorted(WIDE)


@pytest.mark.parametrize("arch,T,Fq", WIDE_ROWS, ids=[f"{'C' if a == 'low_latency_conv' else 'Y'}-{t}x{f}" for a, t, f in WIDE_ROWS])
def test_emulated_wide_range_per_channel(emu, arch, T, Fq):
    """Wide-range weights (each weight bank's output channels scaled by 10^U(-2, 2)): the conv and logits as above, and each conv
    channel held to its own maximum (channel_errors); n = 2 (1 at the BIG rows)."""
    n = 1 if (arch, T, Fq) in BIG else 2
    net = SmallNet(emu, arch, T, Fq, n, seed=1)
    try:
        net.p = wide_range(net.spec, net.p)
        net.params = emu.upload(S.flatten(net.spec, net.p))
        feat = features(_kind(T, Fq), n, T, Fq, seed=5)
        check_small(net, feat)
        ratio, rel = channel_errors(net, feat, net.layer_output(feat))
        print(f"  {arch} {T}x{Fq} n={n}: worst channel {ratio.max():.2f} of its bound, {rel.max():.1e} of its maximum")
        assert ratio.max() <= 1, (ratio.max(), rel[ratio.argmax()])
    finally:
        net.close()


def check_classes(b, arch, T, Fq, classes, n):
    """n utterances on a handle of `classes` classes: the conv and logits against the oracle, the logits-only and probs-only calls
    equal to the call with both, and the evaluation counts of the logits against metrics_oracle's top-k counts."""
    net = SmallNet(b, arch, T, Fq, n, seed=classes, classes=classes)
    try:
        feat = features("randn", n, T, Fq, seed=classes)
        check_small(net, feat)
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


@pytest.mark.parametrize("arch", ARCHS)
@pytest.mark.parametrize("classes", [1, 2, 17, 32])
def test_emulated_class_counts(emu, arch, classes):
    """n = 18: kws_fcb_head's groups of 16 utterances, a full one and a partial one; tiny_conv's split matmul N = classes wide
    (padded to 32 columns), low_latency_conv's final_fc in the head kernel.  7 x 12 and 9 x 10: K = 930 (7 chunks of 128 and 34)
    and 200 (one partial chunk of 256)."""
    check_classes(emu, arch, *((7, 12) if arch == "low_latency_conv" else (9, 10)), classes, 18)


LISTENER_CASES = [(a, c) for a in ARCHS for c in LISTENER_FRONTENDS]


def _listen(b, arch, case, S_, K_, pushes):
    """fp32 and int16 chunks in turn at hop = T - 1 (hop = K = 1 at T = 1, a clip of one window), with a reset of every stream
    before the second to last push and of the last stream before the last one."""
    fe, resets = LISTENER_FRONTENDS[case], ((pushes - 2, -1), (pushes - 1, S_ - 1))
    T = int(case.split("x")[0])
    run_listener(b, arch, S_=S_, hop=max(1, T - 1), K_=1 if T == 1 else K_, pushes=pushes, reset_at=resets, pcm_every=2, case=fe)


@pytest.mark.parametrize("arch,case", LISTENER_CASES, ids=[f"{a}-{c}" for a, c in LISTENER_CASES])
def test_emulated_listener(emu, arch, case):
    """2 streams x 1 window, 3 pushes, at 98 x 40, 49 x 128 log-mel, 49 x 41 and 49 x 42 MFCCs (history rows of an odd and an even
    number of floats) and a one-window clip (tiny_conv: the window's only row between 4 zero rows above and 5 below): each push
    equal bit for bit to the forward on the cut clips."""
    _listen(emu, arch, case, S_=2, K_=1, pushes=3)


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


ORACLE_FLOPS = 5e8      # the fp64 oracle checks every utterance up to this many forward FLOPs a batch, a slice from both ends past it


def _rows(n, spec):
    k = max(2, int(ORACLE_FLOPS // S.forward_flops(spec)))
    return None if k >= n else np.r_[0:k // 2, n - (k - k // 2):n]


U = 2.0 ** -24                          # fp32's unit roundoff


def channel_errors(net, feat, out):
    """The conv held per output channel: each output's error over 1e-5 of its channel's maximum plus the fp32 chain's own rounding
    floor, sqrt(K) u (sum |w x| + |b|) (the usual probabilistic estimate for a K-term fp32 dot product: K = T x 8 taps for
    low_latency_conv, 80 for tiny_conv), the worst per channel, for channels the ReLU does not leave all zero.  The floor matters
    where a negative bias clips all but the top of a channel: its maximum can be hundreds of times below the magnitude its sums
    are accumulated at, and there a few ulps of that magnitude exceed 1e-5 of the maximum.  Returns those ratios (pass: <= 1) and,
    per channel, the error over the channel's maximum alone."""
    spec, p = net.spec, net.p
    x = feat.astype(np.float64)
    ref = S.layer(spec, p, 0, x)
    w, b = spec.convs[0][:2]
    mag = S.layer(spec, dict(p, **{w: np.abs(p[w]), b: np.abs(p[b])}), 0, np.abs(x))
    K = int(np.prod(spec.var_shapes[w][:2]))
    out, ref, mag = (a.reshape(-1, a.shape[-1]).astype(np.float64) for a in (out, ref, mag))
    scale = np.abs(ref).max(0)
    live = scale > 0
    err = np.abs(out - ref)
    ratio = (err / (1e-5 * scale + np.sqrt(K) * U * mag)).max(0)
    return ratio[live], (err.max(0) / np.maximum(scale, 1e-300))[live]


WORST = {}


def _report(net, feat, where, per_channel=False):
    """check_cuda with the oracle on _rows, the worst errors kept for the summary; per_channel: also each conv channel held to its
    own maximum (channel_errors)."""
    n = feat.shape[0]
    rows = _rows(n, net.spec)
    conv, logits = check_cuda(net, feat, rows)
    found = dict(conv=conv, logits=logits)
    if per_channel:
        sel = np.arange(n) if rows is None else rows
        ratio, rel = channel_errors(net, feat[sel], net.layer_output(feat)[sel])
        found["conv per channel / bound"], found["conv per channel / channel max"] = float(ratio.max()), float(rel.max())
        assert ratio.max() <= 1, (ratio.max(), rel[ratio.argmax()])
    for k, e in found.items():
        if e >= WORST.get(k, (0.0,))[0]:
            WORST[k] = (e, f"{where} n={n}")
    print(f"  {where} n={n}{'' if rows is None else f' (oracle on {len(rows)})'}: "
          + " ".join(f"{k} {e:.1e}" for k, e in found.items()))


@pytest.fixture(scope="module")
def worst_errors():
    yield WORST
    print("\n  worst errors: " + "; ".join(f"{k} {e:.1e} ({w})" for k, (e, w) in sorted(WORST.items())))


@pytest.mark.gpu
@pytest.mark.parametrize("arch,T,Fq,claims,why", GEOMETRIES, ids=IDS)
def test_cuda_conv_logits_and_invariance(cuda, worst_errors, arch, T, Fq, claims, why):
    """The conv within 1e-5 and the logits within 1e-4 with the kernels each call launches named, at n = 1, 3, 39 and 100; then the
    logits of the largest batch are the same bits repeated, permuted, sliced and on a handle with another max_batch; at the WIDE
    rows the largest batch once more with wide-range weights, each conv channel held to its own maximum (channel_errors)."""
    where = f"{arch} {T}x{Fq}"
    net = SmallNet(cuda, arch, T, Fq, 128, seed=1)
    other = SmallNet(cuda, arch, T, Fq, 100, seed=1)
    try:
        for n in (1, 3, 39, 100):
            _report(net, features(_kind(T, Fq), n, T, Fq, seed=n), where)
        feat = features(_kind(T, Fq), 100, T, Fq, seed=100)
        check_invariance(net, feat, other)
        if (arch, T, Fq) in WIDE:
            net.p = wide_range(net.spec, net.p)
            net.params = cuda.upload(S.flatten(net.spec, net.p))
            _report(net, feat, where + " wide-range", per_channel=True)
    finally:
        net.close()
        other.close()


@pytest.mark.gpu
@pytest.mark.parametrize("arch,case", LISTENER_CASES, ids=[f"{a}-{c}" for a, c in LISTENER_CASES])
def test_cuda_listener(cuda, arch, case):
    """13 streams x 3 windows at hop = T - 1 (7 streams x 1 window at T = 1), 5 pushes: each push equal bit for bit to the forward on
    the cut clips, and the push's conv is the windowed kernel."""
    _listen(cuda, arch, case, S_=13 if case != "1x40" else 7, K_=3, pushes=5)


@pytest.mark.gpu
def test_cuda_refusal_through_the_model_class(cuda):
    """KWSModel refuses a front-end low_latency_conv cannot take (7 MFCCs: narrower than its T x 8 conv), naming the bound."""
    from tcresnet_b200._lib import TcrError
    from tcresnet_b200.factory import audio_nets
    from tcresnet_b200.runtime import Node
    args = argparse.Namespace(num_classes=12, sample_rate=16000, clip_duration_ms=1000, window_size_ms=40.0, window_stride_ms=20.0,
                              num_mel_bins=64, num_mfccs=7, lower_edge_hertz=80.0, upper_edge_hertz=7600.0, preprocess_method="mfcc",
                              batch_size=3, output_name="output/softmax", weight_decay=1e-4, architecture="low_latency_conv")
    model = audio_nets.KWSModel(args, None)
    with pytest.raises(TcrError, match=r"status 3\): low_latency_conv needs width >= 8"):
        model.build(Node("wavs", [None, 16000, 1]), Node("labels", [None, 12]), False)


@pytest.mark.gpu
@pytest.mark.parametrize("arch", ARCHS)
def test_cuda_tc_mode_leaves_small_kernels_unchanged(cuda, monkeypatch, arch):
    """TCR_DSCNN_TC selects DS-CNN's kernels only: unset, 0 and 1 launch the same kernels and give the same logits bit for bit."""
    feat = features("mfcc", 39, 49, 40, seed=4)
    runs = []
    for mode in (None, "0", "1"):
        if mode is None:
            monkeypatch.delenv("TCR_DSCNN_TC", raising=False)
        else:
            monkeypatch.setenv("TCR_DSCNN_TC", mode)
        net = SmallNet(cuda, arch, 49, 40, 39, seed=3)
        try:
            got = {}
            counts = launched(cuda.lib, lambda: got.setdefault("out", net.forward(feat)))
            runs.append((dict(counts), got["out"][0]))
        finally:
            net.close()
    assert runs[0][0] == {CONV[arch]: 1, "kws_fcs": 1, "kws_fcb_head": 1}, runs[0][0]
    for names, logits in runs[1:]:
        assert names == runs[0][0] and np.array_equal(logits, runs[0][1])
    spec = S.build_spec(arch, 49, 40)
    assert rel_err(runs[0][1], S.forward(spec, S.init_variables(spec, 3), feat.astype(np.float64))) <= 1e-4
