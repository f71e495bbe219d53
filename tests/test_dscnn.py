"""DS-CNN forward (BASELINE.json config 5): oracle self-check against torch, emulated kernels on CPU, CUDA path on GPU."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dscnn_oracle as D
from tcr_harness import launched, rel_err
from tcresnet_b200 import _lib as L


def test_oracle_matches_independent_torch_restatement():
    spec = D.build_spec("S")
    p = D.init_variables(spec, 0)
    assert D.forward_flops(spec) == 21249536            # 21.25 MFLOP, SURVEY.md 8a (a18)
    x = np.random.RandomState(1).randn(3, 49, 40)

    def conv(t, w, stride, groups=1):                   # torch weight [Cout, Cin/groups, kh, kw]
        kh, kw = w.shape[2:]
        _, pt, pb = D.same_pad(t.shape[2], kh, stride[0])
        _, pl, pr = D.same_pad(t.shape[3], kw, stride[1])
        return F.conv2d(F.pad(t, (pl, pr, pt, pb)), w, stride=stride, groups=groups)

    def bn(t, s):
        v = lambda k: torch.tensor(p[s + "/" + k])[None, :, None, None]
        return F.relu((t - v("moving_mean")) / torch.sqrt(v("moving_variance") + 1e-3) + v("beta"))

    t, cin, acts = torch.tensor(x)[:, None], 1, []
    for typ, depth, k, stride, scope in D.NET_DEFS["S"]:
        s = f"DSCNN/{scope}"
        bias = lambda k_: torch.tensor(p[k_])[None, :, None, None]
        if typ == "conv":
            t = bn(conv(t, torch.tensor(p[s + "/weights"]).permute(3, 2, 0, 1), stride) + bias(s + "/biases"), s + "/batch_norm")
        else:
            dw = torch.tensor(p[s + "/depthwise_conv/depthwise_weights"]).permute(2, 3, 0, 1)
            t = bn(conv(t, dw, stride, groups=cin) + bias(s + "/depthwise_conv/biases"), s + "/dw_batch_norm")
            pw = torch.tensor(p[s + "/pointwise_conv/weights"]).permute(3, 2, 0, 1)
            t = bn(conv(t, pw, (1, 1)) + bias(s + "/pointwise_conv/biases"), s + "/pw_batch_norm")
        cin = depth
        acts.append(t.permute(0, 2, 3, 1).numpy())                     # NCHW -> NHWC
    ref = t.mean(dim=(2, 3)) @ torch.tensor(p["DSCNN/fc1/weights"]) + torch.tensor(p["DSCNN/fc1/biases"])
    np.testing.assert_allclose(D.forward(spec, p, x), ref.numpy(), rtol=1e-10, atol=1e-12)
    got = D.forward_layers(spec, p, x)
    assert [a.shape for a in got] == [a.shape for a in acts] == [(3, 25, 20, 64)] * 5
    for l, (a, r) in enumerate(zip(got, acts)):
        np.testing.assert_allclose(a, r, rtol=1e-10, atol=1e-12, err_msg=f"layer {l}")
        np.testing.assert_array_equal(D.layer(spec, p, l, x if l == 0 else got[l - 1]), a)


def _run(backend, size, h, w, n):
    lib = backend.lib
    spec = D.build_spec(size, h, w)
    p = D.init_variables(spec, 0)
    cfg = L.TcrDscnnConfig(ord(size), h, w, 12, max(n, 4), 0)
    handle = C.c_void_p()
    L.check(lib, lib.tcr_dscnn_create(C.byref(cfg), C.byref(handle)), "tcr_dscnn_create")
    descs, count, nparams, flops = C.POINTER(L.TcrParamDesc)(), C.c_int32(), C.c_int64(), C.c_int64()
    L.check(lib, lib.tcr_dscnn_param_table(handle, C.byref(descs), C.byref(count), C.byref(nparams), C.byref(flops)), "table")
    assert [descs[i].name.decode() for i in range(count.value)] == spec.var_names
    assert flops.value == D.forward_flops(spec)
    flat = D.flatten(spec, p)
    assert nparams.value == flat.size
    feat = np.random.RandomState(3).randn(n, h, w).astype(np.float32)
    d_feat, d_par = backend.upload(feat), backend.upload(flat)
    logits, probs = backend.empty(n, 12), backend.empty(n, 12)
    L.check(lib, lib.tcr_dscnn_forward(handle, backend.ptr(d_feat), backend.ptr(d_par), n, backend.ptr(logits),
                                       backend.ptr(probs), backend.stream), "tcr_dscnn_forward")
    backend.sync()
    ref = D.forward(spec, p, feat.astype(np.float64))
    got = backend.download(logits)
    assert rel_err(got, ref) <= 1e-4                      # north-star tolerance; measured ~1e-6
    e = np.exp(ref - ref.max(1, keepdims=True))
    np.testing.assert_allclose(backend.download(probs), e / e.sum(1, keepdims=True), atol=2e-5)
    assert np.array_equal(got.argmax(1), ref.argmax(1))
    lib.tcr_dscnn_destroy(handle)
    return rel_err(got, ref)


def test_emulated_dscnn_matches_oracle():
    from tcr_harness import NumpyBackend
    b = NumpyBackend()
    assert _run(b, "S", 49, 40, 2) < 1e-5
    assert _run(b, "S", 49, 10, 1) < 1e-5                 # the reference's DS-CNN recipes use 10 MFCCs
    assert _run(b, "M", 49, 10, 1) < 1e-5                 # 172 channels, strided depthwise
    assert _run(b, "L", 49, 10, 1) < 1e-5                 # 276 channels: the pointwise bank is walked in output-channel tiles


@pytest.mark.gpu
@pytest.mark.parametrize("size,h,w,n", [("S", 49, 40, 512), ("S", 49, 10, 39), ("M", 49, 10, 33), ("L", 49, 10, 17)])
def test_cuda_dscnn_matches_oracle(size, h, w, n):
    from tcr_harness import TorchBackend
    assert _run(TorchBackend(), size, h, w, n) < 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["0", "1"], ids=["fp32-fma", "wgmma-lockstep"])
def test_cuda_dscnn_other_kernel_paths(mode, monkeypatch):
    """TCR_DSCNN_TC picks the kernels when the net is created: 0 = register-tiled fp32 FMA, 1 = the lock-step wgmma kernels
    (dscnn_conv_tc, dscnn_dsblock_tc).  Unset, conv_1 runs on dscnn_conv_ws and the blocks on dscnn_dsblock_ws where its
    shared memory fits (49x40) and on dscnn_dsblock_tc where it does not (49x10): see test_cuda_dscnn_layers.  Every path meets
    the same bound."""
    from tcr_harness import TorchBackend
    monkeypatch.setenv("TCR_DSCNN_TC", mode)
    assert _run(TorchBackend(), "S", 49, 40, 150) < 1e-5
    assert _run(TorchBackend(), "S", 49, 10, 39) < 1e-5


# ---- layer by layer against the oracle, across the tile planner's shapes ----
# Which kernel runs each DS-CNN-S layer, per feature shape (H, W): (conv_1, the four blocks) with TCR_DSCNN_TC unset and with
# TCR_DSCNN_TC=1; TCR_DSCNN_TC=0 runs dscnn_conv + dscnn_dsblock everywhere.  The comments give conv_1's / the blocks' output
# shape and the tile planner's (tile rows, rows of the last tile): a last tile with fewer rows runs the partial-tile paths.
S_KERNELS = {
    (49, 10): (("conv_ws", "dsblock_tc"), ("conv_tc", "dsblock_tc")),   # 25x5, one tile of 25: dsblock_ws needs 267,008 B of smem
    (49, 40): (("conv_ws", "dsblock_ws"), ("conv_tc", "dsblock_tc")),   # 25x20, 5 tiles of 5
    (49, 12): (("conv_ws", "dsblock_ws"), ("conv_tc", "dsblock_tc")),   # 25x6, (13, 12)
    (13, 40): (("conv_ws", "dsblock_ws"), ("conv_tc", "dsblock_tc")),   # 7x20, (4, 3)
    (49, 18): (("conv_ws", "dsblock_tc"), ("conv_tc", "dsblock_tc")),   # 25x9, (13, 12)
    (98, 40): (("conv_ws", "dsblock_tc"), ("conv_tc", "dsblock_tc")),   # 49x20, (6, 1)
    (49, 64): (("conv_ws", "dsblock"), ("conv_tc", "dsblock")),         # 25x32, conv_1 (4, 1); the blocks do not fit wgmma
    (49, 128): (("conv_tc", "dsblock"), ("conv_tc", "dsblock")),        # 25x64 (the wgmma width limit), conv_1 (2, 1)
    (49, 130): (("conv", "dsblock"), ("conv", "dsblock")),              # 25x65: past the limit, FMA
    (9, 10): (("conv_ws", "dsblock_ws"), ("conv_tc", "dsblock_tc")),    # 5x5: the 10-row filter is taller than the input
    (1, 10): (("conv_ws", "dsblock_ws"), ("conv_tc", "dsblock_tc")),    # 1x5
}
NLAYERS = {"S": 5, "M": 5, "L": 6}


def expected_kernels(size, h, w, mode):
    """Launch names of each layer of a forward pass."""
    if size != "S" or mode == "0":
        conv, block = "conv", "dsblock"
    else:
        conv, block = S_KERNELS[h, w][mode == "1"]
    return ["dscnn_" + conv] + ["dscnn_" + block] * (NLAYERS[size] - 1)


def features(kind, n, h, w, seed=3):
    """[n, h, w] fp32 model input.  mfcc / logmel: the front end's statistics (the oracle's MFCC of synthetic clips, with silence
    in clip 0 and a full-scale square wave in clip 1), the first h frames and w coefficients; randn: N(0, 1)."""
    from oracle import tcr_oracle as O
    if kind == "randn":
        return np.random.RandomState(seed).randn(n, h, w).astype(np.float32)
    wav, _ = O.synthetic_batch(n, seed_wav=1234 + seed, adversarial=True)
    window, stride = (640, 320) if h <= 49 else (480, 160)
    f = O.mfcc(wav, window, stride) if kind == "mfcc" else O.log_mel_spectrogram(wav, window, stride, False)
    assert f.shape[1] >= h and f.shape[2] >= w
    return np.ascontiguousarray(f[:, :h, :w], np.float32)


def wide_range(spec, p, seed=7):
    """The same net with every weight bank's output channels scaled by 10^U(-2, 2) and moving variances 10^U(-2, 2): per-channel
    magnitudes four decades apart in every activation."""
    rng = np.random.RandomState(seed)
    q = dict(p)
    for k, v in p.items():
        if k.endswith("weights"):
            q[k] = v * 10.0 ** rng.uniform(-2, 2, size=v.shape[-1])
        elif k.endswith("moving_variance"):
            q[k] = 10.0 ** rng.uniform(-2, 2, size=v.shape)
    return q


class DsNet:
    """One tcr_dscnn handle with its parameters on the device."""

    def __init__(self, backend, size, h, w, max_batch, p, classes=12):
        self.b, self.lib, self.spec, self.p = backend, backend.lib, D.build_spec(size, h, w, classes), p
        cfg = L.TcrDscnnConfig(ord(size), h, w, classes, max_batch, 0)
        self.h = C.c_void_p()
        L.check(self.lib, self.lib.tcr_dscnn_create(C.byref(cfg), C.byref(self.h)), "tcr_dscnn_create")
        self.params = backend.upload(D.flatten(self.spec, p))
        self.shapes = [a.shape[1:] for a in D.forward_layers(self.spec, p, np.zeros((1, h, w)))]

    def close(self):
        self.lib.tcr_dscnn_destroy(self.h)

    def forward(self, feat):
        b, n = self.b, feat.shape[0]
        c = self.spec.num_classes
        d_feat, logits, probs = b.upload(feat), b.empty(n, c), b.empty(n, c)
        L.check(self.lib, self.lib.tcr_dscnn_forward(self.h, b.ptr(d_feat), b.ptr(self.params), n, b.ptr(logits), b.ptr(probs),
                                                     b.stream), "tcr_dscnn_forward")
        b.sync()
        return b.download(logits), b.download(probs)

    def layer_output(self, feat, k):
        """Output of layer k - 1 (tcr_dscnn_forward_partial), written into a buffer with one utterance of NaN padding after it:
        the padding must survive and every position of the n utterances must be written."""
        b, n = self.b, feat.shape[0]
        d_feat, out = b.upload(feat), b.empty(n + 1, *self.shapes[k - 1])
        L.check(self.lib, self.lib.tcr_dscnn_forward_partial(self.h, b.ptr(d_feat), b.ptr(self.params), n, k, b.ptr(out), b.stream),
                "tcr_dscnn_forward_partial")
        b.sync()
        got = b.download(out)
        assert np.isnan(got[n]).all(), f"layer {k - 1} stored past the last utterance"
        assert np.isfinite(got[:n]).all(), f"layer {k - 1} left positions unwritten"
        return got[:n]


def check_layers(net, feat, kernels=None, rows=None, logit_tol=1e-5):
    """Each layer in isolation: layer l on the CUDA path's own output of layer l - 1 (fp32 -> fp64) against oracle.layer, bound
    max|d| / max|ref| <= 1e-5; then the logits, probabilities and argmax of the whole forward pass.  kernels: the launch names
    each layer must run (checked through the launch profiler).  rows: the utterances the oracle checks (all by default); every
    layer still runs on the whole batch.  logit_tol: the logits' bound.  Returns the per-layer errors."""
    spec, p, cuda = net.spec, net.p, net.b.name == "cuda"
    rows = np.arange(feat.shape[0]) if rows is None else rows
    errs, ran, prev, x = [], [], None, feat[rows].astype(np.float64)
    for k in range(1, NLAYERS[spec.size] + 1):
        if cuda:
            got = {}
            counts = launched(net.lib, lambda: got.setdefault("a", net.layer_output(feat, k)))
            new = counts - prev if prev is not None else counts
            assert sum(new.values()) == 1 and sum(counts.values()) == k, counts
            ran.append(next(iter(new)))
            prev, out = counts, got["a"]
        else:
            out = net.layer_output(feat, k)
        errs.append(rel_err(out[rows], D.layer(spec, p, k - 1, x)))
        x = out[rows].astype(np.float64)
    print(f"  {spec.size} {spec.h}x{spec.w} n={feat.shape[0]}: {' '.join(ran) or 'emulated'}; worst error per layer "
          + " ".join(f"{e:.1e}" for e in errs))
    if kernels is not None:
        assert ran == kernels, ran
    assert max(errs) <= 1e-5, errs
    logits, probs = net.forward(feat)
    logits, probs = logits[rows], probs[rows]
    ref = D.forward(spec, p, feat[rows].astype(np.float64))
    assert rel_err(logits, ref) <= logit_tol, rel_err(logits, ref)
    e = np.exp(ref - ref.max(1, keepdims=True))
    np.testing.assert_allclose(probs, e / e.sum(1, keepdims=True), atol=2e-5)
    if ref.shape[1] > 1:
        top2 = np.sort(ref, 1)[:, -2:]
        clear = top2[:, 1] - top2[:, 0] > 1e-4 * np.abs(ref).max()     # no near-tie the bound allows to flip
        assert np.array_equal(logits.argmax(1)[clear], ref.argmax(1)[clear])
    return errs


def check_invariance(net, feat, other):
    """The logits of an utterance are the same bits whatever else is in the batch and whichever CTA runs its tiles: repeated,
    permuted, from a slice, on a handle with a different max_batch (`other`)."""
    n = feat.shape[0]
    ref, _ = net.forward(feat)
    assert np.array_equal(net.forward(feat)[0], ref), "repeated call"
    perm = np.random.RandomState(n).permutation(n)
    assert np.array_equal(net.forward(np.ascontiguousarray(feat[perm]))[0], ref[perm]), "permuted batch"
    i, j = n // 3, n // 3 + max(1, n // 2)
    assert np.array_equal(net.forward(np.ascontiguousarray(feat[i:j]))[0], ref[i:j]), "slice"
    assert np.array_equal(other.forward(feat)[0], ref), "max_batch"


def emulated_case(size, h, w, n, kind):
    from tcr_harness import NumpyBackend
    spec = D.build_spec(size, h, w)
    net = DsNet(NumpyBackend(), size, h, w, n, D.init_variables(spec, 0))
    try:
        return check_layers(net, features(kind, n, h, w))
    finally:
        net.close()


@pytest.mark.parametrize("size,h,w,n,kind", [("S", 49, 64, 2, "logmel"), ("S", 98, 40, 1, "mfcc"), ("M", 49, 40, 1, "mfcc"),
                                             ("L", 49, 10, 1, "mfcc")],
                         ids=["S-49x64-partial-tiles", "S-98x40", "M-49x40", "L-49x10"])
def test_emulated_dscnn_layers(size, h, w, n, kind):
    """The FMA kernels on the CPU emulator, layer by layer, with the NaN canary after the output (the FMA block kernel's tile of
    8 rows leaves a last tile of 1 row at 49x64 and 98x40)."""
    emulated_case(size, h, w, n, kind)


def _tf32(a):
    return (np.ascontiguousarray(a, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def _split(a):
    """The kernels' operand split: hi = x with the low 13 mantissa bits cleared, lo = x - hi (exact), each read as TF32."""
    hi = _tf32(a)
    return hi.astype(np.float64), _tf32(np.float32(a) - hi).astype(np.float64)


def test_3xtf32_split_is_what_the_gpu_bound_measures():
    """NumPy emulation of the wgmma kernels' arithmetic on this suite's own layer inputs (DS-CNN-S 49x40 on MFCCs, and a wide
    dynamic-range net): conv_1 and every pointwise conv as TF32 products of split operands, lo*hi + hi*lo + hi*hi.  Three passes
    land well inside the 1e-5 per-layer bound; one pass (hi*hi) or two (either lo term dropped) miss it by 10x or more, so the GPU
    layer checks tell a correct kernel from one that skips a pass."""
    spec = D.build_spec("S", 49, 40)
    feat = features("mfcc", 4, 49, 40).astype(np.float64)
    for p in (D.init_variables(spec, 0), wide_range(spec, D.init_variables(spec, 0))):
        x = feat[..., None]
        for l, (typ, _, _, stride, scope) in enumerate(D.NET_DEFS["S"]):
            s = f"DSCNN/{scope}"
            ref = D.layer(spec, p, l, x)
            if typ == "conv":
                a, wk, b, bn, st = x, p[s + "/weights"], p[s + "/biases"], s + "/batch_norm", stride
            else:      # the depthwise stage runs in fp32 FMAs: its output (the A operand) is rounded to fp32
                dw = D._depthwise(x, p[s + "/depthwise_conv/depthwise_weights"], stride) + p[s + "/depthwise_conv/biases"]
                a = D._bn_relu(dw, p, s + "/dw_batch_norm").astype(np.float32)
                wk, b, bn, st = p[s + "/pointwise_conv/weights"], p[s + "/pointwise_conv/biases"], s + "/pw_batch_norm", (1, 1)
            (a_hi, a_lo), (w_hi, w_lo) = _split(a), _split(wk)
            mm = {(i, j): D._conv2d(u, v, st) for i, u in enumerate((a_hi, a_lo)) for j, v in enumerate((w_hi, w_lo)) if i + j < 2}
            err = {name: rel_err(D._bn_relu(sum(mm[t] for t in terms) + b, p, bn), ref) for name, terms in
                   (("3", [(1, 0), (0, 1), (0, 0)]), ("no lo*hi", [(0, 1), (0, 0)]), ("no hi*lo", [(1, 0), (0, 0)]), ("1", [(0, 0)]))}
            assert err["3"] < 1e-6, (l, err)
            assert min(err["no lo*hi"], err["no hi*lo"], err["1"]) > 1e-4, (l, err)
            x = ref


# ---- GPU ----
def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _gpu_case(size, h, w, ns, kind, mode, monkeypatch, wide=False):
    from tcr_harness import TorchBackend
    if mode is not None:
        monkeypatch.setenv("TCR_DSCNN_TC", mode)
    else:
        monkeypatch.delenv("TCR_DSCNN_TC", raising=False)
    b = TorchBackend()
    spec = D.build_spec(size, h, w)
    p = D.init_variables(spec, 0)
    p = wide_range(spec, p) if wide else p
    big = DsNet(b, size, h, w, 512, p)                 # n < max_batch: the TMA map spans all 512 utterances
    try:
        for n in ns:
            feat = features(kind, n, h, w, seed=n)
            net = DsNet(b, size, h, w, n, p)
            try:
                check_layers(net, feat, expected_kernels(size, h, w, mode))
                check_invariance(net, feat, big)
            finally:
                net.close()
    finally:
        big.close()


MODES = pytest.mark.parametrize("mode", [None, "1", "0"], ids=["default", "TC1-lockstep", "TC0-fma"])


@pytest.mark.gpu
@MODES
@pytest.mark.parametrize("h,w", [(49, 12), (13, 40), (49, 18), (98, 40), (49, 64), (49, 128), (49, 130), (9, 10), (1, 10)])
def test_cuda_dscnn_layers(h, w, mode, monkeypatch):
    """DS-CNN-S layer by layer at the shapes that reach each kernel's partial last tile (S_KERNELS), on the front end's features
    (log-mel at 64 bins, N(0, 1) past it), n = 3 and 5."""
    kind = "mfcc" if w <= 40 else ("logmel" if w == 64 else "randn")
    _gpu_case("S", h, w, [3, 5], kind, mode, monkeypatch)


@pytest.mark.gpu
@MODES
@pytest.mark.parametrize("h,w,tiles_per_utt", [(49, 10, 1), (49, 40, 5)], ids=["49x10-recipes", "49x40-bench"])
def test_cuda_dscnn_layers_batch_sweep(h, w, tiles_per_utt, mode, monkeypatch):
    """The persistent wgmma kernels walk tiles with a stride of the grid (= min(tiles, SMs)) and prefetch the tile two ahead:
    batches whose tile count is below the SM count, equal to it (where a multiple), one more, and one more than 2 x SMs, and the
    recipes' batch sizes 3, 39, 100, on the default weights and MFCCs; then 2 x SMs + 1 tiles of N(0, 1) features with
    wide-range weights."""
    sms = _sms()
    ns = sorted({3, 39, 100} | {-(-t // tiles_per_utt) for t in (sms, sms + 1, 2 * sms + 1)})
    print(f"  {sms} SMs, {tiles_per_utt} tile(s) per utterance: n = {ns}")
    _gpu_case("S", h, w, ns, "mfcc", mode, monkeypatch)
    _gpu_case("S", h, w, [-(-(2 * sms + 1) // tiles_per_utt)], "randn", mode, monkeypatch, wide=True)


@pytest.mark.gpu
@pytest.mark.parametrize("size,h,w", [("M", 49, 40), ("M", 98, 40), ("L", 49, 40), ("L", 98, 40)])
def test_cuda_dscnn_m_l_layers(size, h, w, monkeypatch):
    """DS-CNN-M and -L (172 / 276 channels, strided first block) on the FMA kernels, L's pointwise bank in output-channel tiles."""
    _gpu_case(size, h, w, [5], "mfcc", None, monkeypatch)
