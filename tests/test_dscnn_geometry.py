"""DS-CNN S, M and L at the edges of every geometry, batch and class count their handle accepts, against the fp64 oracle
(dscnn_oracle): reach() restates the plan tcr_dscnn_create makes for each layer (ds_plan_layer) on plain integers and is checked
against the handle's width and height bounds, in each TCR_DSCNN_TC mode for S; the parameter table, every layer and the logits at
each row of GEOMETRIES (the SAME pads of M and L's stride-2 block in all four parities, the widest and tallest geometries, L's
pointwise bank in output-channel slices with a short last slice, S's wgmma tile edges), 1 to 32 classes, weights of unequal scale
held per channel, batches past the 65,535-row grid bound, the listener at new geometries, and the refusals.  The FMA kernels on the
CPU emulator; on the GPU with the launched kernels named, batch invariance and the TCR_DSCNN_TC switch."""
import argparse
import ctypes as C
import re

import numpy as np
import pytest

from oracle import dscnn_oracle as D
from oracle import metrics_oracle as MO
from tcr_harness import NumpyBackend, launched, rel_err
from test_dscnn import NLAYERS, DsNet, check_invariance, check_layers, features, wide_range
from test_dscnn_listener import run_case
from test_kws_geometry import _counts, _forward_one

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L

TCR_ERR_UNSUPPORTED = 3
CONV_LIMIT = 227 * 1024                 # dscnn_conv stages a whole utterance: sm_90's opt-in shared memory per block
BLOCK_LIMIT = 200 * 1024                # dscnn_dsblock's cap
CONV_WS_CAP, BLOCK_WS_CAP, BLOCK_TC_CAP = 220 * 1024, 226 * 1024, 200 * 1024    # where the wgmma kernels give way
TC_THREADS, WS_PRODUCERS = 512, 320     # threads of a wgmma CTA; producer threads of the warp-specialised kernels
CONV_CELLS, CONV_TASKS, DW_CELLS = 4, 4, 8    # per-thread input cells / operand tasks of the im2col walk; dsblock_tc's input cells
LBA_FULL = 128 * 4 + 4                  # K-chunk stride (floats) of a 128-row A operand


def _lbb(co):
    return co * 4 + 4


def _tile_rows(hout, wout):
    """ds_tile_rows: at most 128 accumulator rows a tile, balanced."""
    cap = max(1, min(hout, 128 // max(1, min(wout, 128))))
    tiles = -(-hout // cap)
    return -(-hout // tiles)


def reach(size, T, F, mode="0"):
    """What DS-CNN `size` runs at T x F features, restated from ds_plan_layer and the kernels.  mode: TCR_DSCNN_TC ("0" FMA
    everywhere, which is also what the emulator build runs; "1" the lock-step wgmma kernels; None the warp-specialised ones), wgmma
    for S only.  Per layer (keyed by scope): hin, win, hout, wout and the SAME pads (top, left); the kernel; rh, the tile rows
    (ds_tile_rows' RHt for wgmma, the FMA block's RH, 0 for dscnn_conv, which stages the whole utterance), tiles per utterance and
    the rows of the last; the FMA block's output-channel slice cot, its number of slices and the width of the last; smem, the
    bytes.  fits: every layer within its limit; refusal: the message tcr_dscnn_create gives at the first layer past it."""
    h, w, cin, out, refusal = T, F, 1, {}, None
    for typ, cout, (kh, kw), (sh, sw), scope in D.NET_DEFS[size]:
        hout, pt, _ = D.same_pad(h, kh, sh)
        wout, pl, _ = D.same_pad(w, kw, sw)
        in_rows = lambda rh: (rh - 1) * sh + kh              # noqa: E731
        in_cols = (wout - 1) * sw + kw
        r = dict(hin=h, win=w, hout=hout, wout=wout, pads=(pt, pl), cot=None, slices=None, last_slice=None)
        tc = mode != "0" and size == "S"
        rht = _tile_rows(hout, wout)
        if typ == "conv":
            def walk(nt, rh=rht):
                return in_rows(rh) * in_cols <= CONV_CELLS * nt and 128 * (kh * kw // 4) <= CONV_TASKS * nt and in_rows(rh) < 512
            k4 = kh * kw // 4
            tc_smem = lambda nbuf: 4 * (2 * nbuf * k4 * LBA_FULL + 2 * k4 * _lbb(64) + 2 * 64      # noqa: E731
                                        + 2 * ((in_rows(rht) * in_cols + 3) & ~3))
            if tc and cout == 64 and (kh * kw) % 8 == 0 and wout <= 64 and walk(TC_THREADS):
                if mode is None and tc_smem(2) <= CONV_WS_CAP and walk(WS_PRODUCERS) and k4 % 2 == 0:
                    r.update(kernel="dscnn_conv_ws", rh=rht, smem=tc_smem(2))
                else:
                    r.update(kernel="dscnn_conv_tc", rh=rht, smem=tc_smem(1))
            else:
                smem = 4 * (((in_rows(hout) * in_cols + 3) & ~3) + kh * kw * cout + 2 * cout)
                r.update(kernel="dscnn_conv", rh=0, smem=smem, limit=CONV_LIMIT)
        else:
            tab = 9 * cin + 2 * cin + 2 * cout
            ws_xs = (((rht + 2) * (wout + 2) * 32 * 4 + 1023) & ~1023) // 4
            ws_smem = 4 * (4 * ws_xs + 4 * 16 * (((rht * wout + 7) & ~7) * 4 + 4) + 2 * 16 * _lbb(64) + tab)
            tc_smem = 4 * (2 * 16 * ((rht + 2) * (wout + 2) * 4 + 4) + 2 * 16 * LBA_FULL + 2 * 16 * _lbb(64) + tab)
            if tc and cin == cout == 64 and (sh, sw) == (1, 1) and wout <= 64 and mode is None and ws_smem <= BLOCK_WS_CAP \
                    and 16 * wout <= WS_PRODUCERS and wout + 2 <= 256 and rht + 2 <= 256:
                r.update(kernel="dscnn_dsblock_ws", rh=rht, smem=ws_smem)
            elif tc and cin == cout == 64 and (sh, sw) == (1, 1) and wout <= 64 and tc_smem <= BLOCK_TC_CAP \
                    and (rht + 2) * (wout + 2) <= DW_CELLS * (TC_THREADS // 16):
                r.update(kernel="dscnn_dsblock_tc", rh=rht, smem=tc_smem)
            else:
                def smem(rh, cot):
                    return 4 * (in_rows(rh) * in_cols * cin + rh * wout * cin + cin * cot + tab)
                cot = cout
                while cot > 32 and smem(1, cot) > 96 * 1024:
                    cot = (cot // 2 + 3) & ~3
                rh = min(hout, 8)
                while rh > 1 and smem(rh, cot) > 100 * 1024:
                    rh -= 1
                r.update(kernel="dscnn_dsblock", rh=rh, smem=smem(rh, cot), limit=BLOCK_LIMIT, cot=cot, slices=-(-cout // cot),
                         last_slice=cout - (-(-cout // cot) - 1) * cot)
        if r["rh"]:
            r.update(tiles=-(-hout // r["rh"]), last_rows=hout - (-(-hout // r["rh"]) - 1) * r["rh"])
        else:
            r.update(tiles=1, last_rows=hout)
        if refusal is None and r["smem"] > r.get("limit", r["smem"]):
            refusal = (f"{r['kernel']} ({scope}) needs {r['smem']} bytes of shared memory at {T} x {F}, the limit is {r['limit']}")
        out[scope] = r
        h, w, cin = hout, wout, cout
    return dict(layers=out, fits=refusal is None, refusal=refusal)


def flops(size, T, F, classes=12):
    """Forward FLOPs from reach()'s shapes: 2 per multiply-add of each conv, the depthwise and pointwise stages, and fc."""
    f, cin = 0, 1
    for (typ, cout, (kh, kw), _, _), r in zip(D.NET_DEFS[size], reach(size, T, F)["layers"].values()):
        pos = r["hout"] * r["wout"]
        f += 2 * pos * kh * kw * cin * cout if typ == "conv" else 2 * pos * 9 * cin + 2 * pos * cin * cout
        cin = cout
    return f + 2 * cin * classes


def widest(size, T, mode="0"):
    """The widest F reach() accepts at height T: the first F past which it refuses, and nothing wider up to twice that fits."""
    F = 1
    while reach(size, T, F + 1, mode)["fits"]:
        F += 1
    assert reach(size, T, F, mode)["fits"] and not any(reach(size, T, g, mode)["fits"] for g in range(F + 1, 2 * F + 2, 7))
    return F


def tallest(size, F, mode="0", cap=8192):
    """The tallest T reach() accepts at width F: None where no T up to `cap` is refused (the wgmma conv tiles rows), 0 where no T
    is accepted (a block is past its limit at every height)."""
    if reach(size, cap, F, mode)["fits"]:
        return None
    if not reach(size, 1, F, mode)["fits"]:
        return 0
    lo, hi = 1, cap
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if reach(size, mid, F, mode)["fits"] else (lo, mid)
    return lo


# The envelope: the widest F at each height and the tallest T at each width (None: no height bound), per net; S per mode.
BOUND_HEIGHTS = list(range(1, 18)) + [49, 98, 1000]
BOUND_WIDTHS = [10, 40, 64]
SIZES = ["S", "M", "L"]


def _err(lib):
    return lib.tcr_last_error().decode()


def create(lib, size, T, F, classes=12, max_batch=1):
    h = C.c_void_p()
    rc = lib.tcr_dscnn_create(C.byref(L.TcrDscnnConfig(ord(size), T, F, classes, max_batch, 0)), C.byref(h))
    return rc, h


def _stale(lib):
    """Leave a different message in tcr_last_error, so that a refusal that sets none shows."""
    assert lib.tcr_dscnn_create(None, None) != 0 and _err(lib) == "NULL argument"


def check_bound(lib, size, T, F, mode):
    """T x F is accepted and reach() agrees; the next geometry past it (given by the caller) is refused with reach()'s message."""
    assert reach(size, T, F, mode)["fits"]
    rc, h = create(lib, size, T, F)
    assert rc == 0, (size, T, F, mode, _err(lib))
    lib.tcr_dscnn_destroy(h)


def check_refused(lib, size, T, F, mode):
    r = reach(size, T, F, mode)
    assert not r["fits"]
    _stale(lib)
    rc, h = create(lib, size, T, F)
    assert rc == TCR_ERR_UNSUPPORTED and not h.value, (size, T, F, mode, rc)
    assert _err(lib) == r["refusal"], (size, T, F, mode, _err(lib), r["refusal"])


def run_bounds(lib, mode, sizes):
    found = {}
    for size in sizes:
        for T in BOUND_HEIGHTS:
            F = widest(size, T, mode)
            check_bound(lib, size, T, F, mode)
            check_refused(lib, size, T, F + 1, mode)
            found[size, "T", T] = F
        for F in BOUND_WIDTHS:
            T = tallest(size, F, mode)
            if T is None:                            # no height bound: a tall clip is accepted
                check_bound(lib, size, 8192, F, mode)
            elif T == 0:                             # no height fits
                check_refused(lib, size, 1, F, mode)
            else:
                check_bound(lib, size, T, F, mode)
                check_refused(lib, size, T + 1, F, mode)
            found[size, "F", F] = T
    for size in sizes:
        print(f"  {size} mode {mode}: widest F per T " + ", ".join(f"{T}: {found[size, 'T', T]}" for T in BOUND_HEIGHTS)
              + "; tallest T per F " + ", ".join(f"{F}: {found[size, 'F', F]}" for F in BOUND_WIDTHS))
    return found


@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


def test_reach_matches_the_handles_bounds(emu):
    """The FMA plan (what the emulator build and TCR_DSCNN_TC=0 run): at T = 1 to 17, 49, 98 and 1,000 the widest F reach() accepts
    is accepted and F + 1 is refused with reach()'s message and bytes; at F = 10, 40 and 64 the same for the tallest T.  The
    envelope: M's conv_ds_1 stops at F = 72, L's at 42 and S's first block at 374 (at T = 49), M's conv_1 at T = 1,174 and L's at
    1,072 (F = 40)."""
    found = run_bounds(emu.lib, "0", SIZES)
    assert (found["S", "T", 49], found["M", "T", 49], found["L", "T", 49]) == (374, 72, 42)
    assert (found["S", "F", 40], found["M", "F", 40], found["L", "F", 40]) == (1310, 1174, 1072)
    assert reach("M", 49, 73)["refusal"].startswith("dscnn_dsblock (conv_ds_1) needs ")
    assert reach("M", 1175, 40)["refusal"] == f"dscnn_conv (conv_1) needs 232544 bytes of shared memory at 1175 x 40, the limit is {CONV_LIMIT}"


def test_reach_agrees_with_the_tile_planners_table():
    """reach() gives S_KERNELS' kernels at every one of its shapes, in the default and the lock-step mode."""
    from test_dscnn import S_KERNELS
    for (h, w), modes in S_KERNELS.items():
        for mode, (conv, block) in zip((None, "1"), modes):
            got = [r["kernel"] for r in reach("S", h, w, mode)["layers"].values()]
            assert got == ["dscnn_" + conv] + ["dscnn_" + block] * 4, (h, w, mode, got)


def test_emulated_refusals_leave_a_fresh_message(emu):
    """Each refusal replaces the last error: refused geometries of S, M and L in turn, each after a different failure."""
    lib = emu.lib
    for size, T, F in (("M", 49, 80), ("L", 49, 64), ("S", 49, 375), ("M", 1175, 40), ("L", 1073, 40), ("S", 1311, 40), ("L", 1, 64)):
        check_refused(lib, size, T, F, "0")
    rc, h = create(lib, "M", 49, 72)
    assert rc == 0
    lib.tcr_dscnn_destroy(h)


# (size, T, F, TCR_DSCNN_TC mode on the GPU, {scope: what the layer reaches (checked against reach())}, why it is here)
GEOMETRIES = [
    ("M", 47, 41, None, dict(conv_ds_1=dict(hin=24, win=41, pads=(0, 1))), "conv_ds_1: even height, odd width (pads 0, 1)"),
    ("M", 48, 40, None, dict(conv_ds_1=dict(hin=24, win=40, pads=(0, 0))), "conv_ds_1: even height, even width (pads 0, 0)"),
    ("L", 48, 41, None, dict(conv_ds_1=dict(pads=(0, 1), cot=20, slices=14, last_slice=16)), "L: even / odd into conv_ds_1"),
    ("L", 49, 39, None, dict(conv_ds_1=dict(hin=25, win=39, pads=(1, 1))), "L: odd / odd into conv_ds_1 (pads 1, 1)"),
    ("M", 1, 1, None, dict(conv_1=dict(hout=1, wout=1), conv_ds_1=dict(pads=(1, 1), cot=88, last_slice=84)), "one output position"),
    ("M", 2, 3, None, dict(conv_1=dict(hout=1, wout=3), conv_ds_1=dict(hout=1, wout=2)), "T = 2, F = 3"),
    ("L", 1, 2, None, dict(conv_ds_1=dict(win=2, pads=(1, 0), cot=36, slices=8, last_slice=24)), "T = 1, F = 2"),
    ("L", 2, 1, None, dict(conv_1=dict(hout=1, wout=1)), "T = 2, F = 1"),
    ("M", 49, 72, None, dict(conv_ds_1=dict(rh=1, cot=24, last_slice=4, smem=200896)), "M's widest F"),
    ("L", 49, 42, None, dict(conv_ds_1=dict(rh=1, cot=20, smem=202032)), "L's widest F"),
    ("M", 1174, 40, None, dict(conv_1=dict(hout=587, smem=232208), conv_ds_1=dict(tiles=294)), "M's tallest T at F = 40"),
    ("L", 1072, 40, None, dict(conv_1=dict(hout=536, smem=232128), conv_ds_1=dict(pads=(0, 0))), "L's tallest T at F = 40"),
    ("L", 49, 20, None, dict(conv_ds_1=dict(cot=20, slices=14, last_slice=16), conv_ds_2=dict(rh=1, tiles=13)), "L at 20: 14 slices"),
    ("M", 49, 10, None, dict(conv_ds_2=dict(rh=2, tiles=7, last_rows=1, cot=88, slices=2, last_slice=84)), "the recipes' M"),
    ("L", 49, 10, None, dict(conv_ds_2=dict(rh=2, tiles=7, cot=36, slices=8, last_slice=24)), "the recipes' L"),
    ("S", 49, 374, None, dict(conv_1=dict(kernel="dscnn_conv"), conv_ds_1=dict(kernel="dscnn_dsblock", cot=32, slices=2,
                                                                               smem=204544)), "S's widest F"),
    ("S", 49, 1, None, dict(conv_1=dict(kernel="dscnn_conv_ws", wout=1), conv_ds_4=dict(kernel="dscnn_dsblock_ws", rh=25)), "F = 1"),
    ("S", 49, 2, "1", dict(conv_1=dict(kernel="dscnn_conv_tc", wout=1), conv_ds_4=dict(kernel="dscnn_dsblock_tc")), "F = 2, lock-step"),
    ("S", 7, 10, None, dict(conv_1=dict(hout=4, rh=4, kernel="dscnn_conv_ws"), conv_ds_1=dict(kernel="dscnn_dsblock_ws")),
     "odd T, the 10-row filter taller than the input"),
    ("S", 1310, 40, "0", dict(conv_1=dict(kernel="dscnn_conv", smem=232176), conv_ds_1=dict(rh=6, tiles=110, last_rows=1)),
     "S's tallest T at F = 40 with TCR_DSCNN_TC=0"),
    ("S", 98, 40, None, dict(conv_1=dict(kernel="dscnn_conv_ws", rh=6, tiles=9, last_rows=1), conv_ds_1=dict(kernel="dscnn_dsblock_tc")),
     "S's persistent wgmma kernels, a last tile of one row"),
]
IDS = [f"{s}-{t}x{f}" + ("" if m is None else f"-TC{m}") for s, t, f, m, _, _ in GEOMETRIES]
ORACLE_FLOPS = 5e8      # the fp64 oracle checks every utterance up to this many forward FLOPs a batch, a slice from both ends past it
# one utterance on the emulator
BIG = {(s, t, f) for s, t, f, _, _, _ in GEOMETRIES if D.forward_flops(D.build_spec(s, t, f)) > 1e8}
# rerun with wide-range weights, each layer's channels held to their own maximum
WIDE = {("M", 47, 41), ("M", 49, 72), ("L", 48, 41), ("L", 49, 10), ("S", 49, 374), ("S", 98, 40), ("S", 49, 2), ("S", 7, 10)}


@pytest.mark.parametrize("size,T,F,mode,claims,why", GEOMETRIES, ids=IDS)
def test_table_and_flops(emu, size, T, F, mode, claims, why):
    """Each row is accepted and reaches what it claims; tcr_dscnn_param_table's names and shapes and the FLOP count against
    dscnn_oracle and the formulas on reach()'s shapes."""
    got = reach(size, T, F, mode)
    assert got["fits"], why
    for scope, c in claims.items():
        assert {k: got["layers"][scope][k] for k in c} == c, (why, scope, got["layers"][scope])
    rc, h = create(emu.lib, size, T, F)
    assert rc == 0, _err(emu.lib)
    try:
        descs, count, nparams, fl = C.POINTER(L.TcrParamDesc)(), C.c_int32(), C.c_int64(), C.c_int64()
        L.check(emu.lib, emu.lib.tcr_dscnn_param_table(h, C.byref(descs), C.byref(count), C.byref(nparams), C.byref(fl)), "table")
        spec = D.build_spec(size, T, F)
        rows = [(descs[i].name.decode(), tuple(descs[i].shape[:descs[i].rank])) for i in range(count.value)]
        assert rows == [(n, spec.var_shapes[n]) for n in spec.var_names]
        assert nparams.value == sum(int(np.prod(s)) for _, s in rows)
        assert fl.value == flops(size, T, F) == D.forward_flops(spec)
    finally:
        emu.lib.tcr_dscnn_destroy(h)


def _net(b, size, T, F, max_batch, seed=0, classes=12, wide=False):
    spec = D.build_spec(size, T, F, classes)
    p = D.init_variables(spec, seed)
    return DsNet(b, size, T, F, max_batch, wide_range(spec, p) if wide else p, classes)


def _logit_tol(size, T, F):
    """The logits' bound: 1e-5, but the library's 1e-4 where the average pool sums more than 2,048 positions a channel.
    dscnn_head sums a channel's positions in three fp32 segments for M and L: at L's 268 x 20 (1,072 x 40) a segment is 1,787 long
    and the emulator's logits land at 1.01e-5 while every layer stays within 6e-7."""
    last = list(reach(size, T, F)["layers"].values())[-1]
    return 1e-4 if last["hout"] * last["wout"] > 2048 else 1e-5


def _kind(T, F):
    """The front end's features where the oracle's front end has the shape (MFCCs up to 40, log-mel up to 64), N(0, 1) past it."""
    if T <= 49:
        return "mfcc" if F <= 40 else ("logmel" if F <= 64 else "randn")
    return "randn"


@pytest.mark.parametrize("size,T,F,mode,claims,why", GEOMETRIES, ids=IDS)
def test_emulated_layers_and_logits(emu, size, T, F, mode, claims, why):
    """The FMA plan on the emulator: every layer within 1e-5 with the NaN canary after the last utterance, and the logits; n = 2
    (n = 1 on the BIG rows)."""
    n = 1 if (size, T, F) in BIG else 2
    net = _net(emu, size, T, F, n, seed=T + F)
    try:
        check_layers(net, features(_kind(T, F), n, T, F, seed=T + F), logit_tol=_logit_tol(size, T, F))
    finally:
        net.close()


U = 2.0 ** -24                          # fp32's unit roundoff


def _magnitude(spec, p, l, x):
    """The magnitudes layer l accumulates at, per output: the layer with |x|, every weight and bias taken absolute and the BatchNorm
    shift widened to |b - mean| / std + |beta| (the separable block's depthwise stage feeds its pointwise stage the same way)."""
    typ, _, _, stride, scope = D.NET_DEFS[spec.size][l]
    s = f"DSCNN/{scope}"
    x = np.abs(x[..., None] if x.ndim == 3 else x)

    def bn(a, bnscope):
        return (a + np.abs(p[bnscope + "/moving_mean"])) / np.sqrt(p[bnscope + "/moving_variance"] + D.BN_EPS) + np.abs(p[bnscope + "/beta"])
    if typ == "conv":
        return bn(D._conv2d(x, np.abs(p[s + "/weights"]), stride) + np.abs(p[s + "/biases"]), s + "/batch_norm")
    a = bn(D._depthwise(x, np.abs(p[s + "/depthwise_conv/depthwise_weights"]), stride) + np.abs(p[s + "/depthwise_conv/biases"]),
           s + "/dw_batch_norm")
    return bn(D._conv2d(a, np.abs(p[s + "/pointwise_conv/weights"]), (1, 1)) + np.abs(p[s + "/pointwise_conv/biases"]), s + "/pw_batch_norm")


def channel_errors(net, feat, kernels):
    """Every layer held per output channel: each output's error (layer l on the kernel's own output of layer l - 1) over 1e-5 of its
    channel's maximum plus the fp32 chain's rounding at the magnitude it accumulates, sqrt(K) u (sum |w x| + |b|) (K: 40 taps for
    conv_1, 9 depthwise taps and the cin-term pointwise sum for a block), plus 12 u of that magnitude on the wgmma layers (the 3xTF32
    split truncates each operand's low part to TF32 and drops lo * lo: at most 3 * 2^-22 of each product).  The worst ratio per
    layer over the channels the ReLU does not leave all zero (pass: <= 1), and the worst error over the channel maximum alone."""
    spec, p = net.spec, net.p
    x, ratios, rels = feat.astype(np.float64), [], []
    for l, (typ, cout, (kh, kw), _, _) in enumerate(D.NET_DEFS[spec.size]):
        full = net.layer_output(feat, l + 1).astype(np.float64)
        ref, mag = D.layer(spec, p, l, x), _magnitude(spec, p, l, x)
        cin = 1 if l == 0 else D.NET_DEFS[spec.size][l - 1][1]
        K = kh * kw if typ == "conv" else 9 + cin
        floor = (np.sqrt(K) + (12 if kernels[l] != "dscnn_conv" and kernels[l] != "dscnn_dsblock" else 0)) * U
        out, ref, mag = (a.reshape(-1, cout) for a in (full, ref, mag))
        scale = np.abs(ref).max(0)
        live = scale > 0
        err = np.abs(out - ref)
        ratios.append(float((err / (1e-5 * scale + floor * mag)).max(0)[live].max()))
        rels.append(float((err.max(0) / np.maximum(scale, 1e-300))[live].max()))
        x = full
    return ratios, rels


WIDE_ROWS = sorted(WIDE)


@pytest.mark.parametrize("size,T,F", WIDE_ROWS, ids=[f"{s}-{t}x{f}" for s, t, f in WIDE_ROWS])
def test_emulated_wide_range_per_channel(emu, size, T, F):
    """Wide-range weights (each bank's output channels scaled by 10^U(-2, 2), moving variances 10^U(-2, 2)) on the FMA plan: every
    layer and the logits as above, and each layer's channels held to their own maximum (channel_errors); n = 1."""
    net = _net(emu, size, T, F, 1, seed=1, wide=True)
    try:
        feat = features("randn", 1, T, F, seed=5)
        check_layers(net, feat, logit_tol=_logit_tol(size, T, F))
        ratios, rels = channel_errors(net, feat, [r["kernel"] for r in reach(size, T, F, "0")["layers"].values()])
        print(f"  {size} {T}x{F}: worst channel per layer " + " ".join(f"{r:.2f}" for r in ratios) + " of its bound, "
              + " ".join(f"{r:.1e}" for r in rels) + " of its maximum")
        assert max(ratios) <= 1, ratios
    finally:
        net.close()


CLASS_GEOMETRY = {"S": (9, 10), "M": (9, 10), "L": (9, 10)}


def check_classes(b, size, classes, n):
    """n utterances on a handle of `classes` classes: every layer and the logits against the oracle; with one class every
    probability is exactly 1; the logits-only and probs-only calls equal to the call with both; the evaluation counts of the
    logits against metrics_oracle's top-k counts."""
    T, F = CLASS_GEOMETRY[size]
    net = _net(b, size, T, F, n, seed=classes, classes=classes)
    try:
        feat = features("randn", n, T, F, seed=classes)
        check_layers(net, feat)
        logits, probs = net.forward(feat)
        assert logits.shape == probs.shape == (n, classes)
        if classes == 1:
            assert (probs == 1).all()
        assert np.array_equal(_forward_one(net, feat, True, False)[0], logits), "logits-only call"
        assert np.array_equal(_forward_one(net, feat, False, True)[1], probs), "probs-only call"
        onehot = np.eye(classes, dtype=np.float32)[np.random.RandomState(classes).randint(0, classes, n)]
        for topk in (1, 5):
            got = _counts(net, logits, onehot, topk)
            assert np.array_equal(got, MO.eval_counts(logits, onehot, topk)), topk
            assert got[-1] == n
    finally:
        net.close()


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("classes", [1, 2, 17, 32])
def test_emulated_class_counts(emu, size, classes):
    check_classes(emu, size, classes, 3)


# M and L through the listener at geometries off the recipes' (T x F: front-end flags)
LISTENER_FRONTENDS = {
    "47x41": dict(clip_samples=640 + 46 * 320, num_mfccs=41, num_mel_bins=64),
    "48x40": dict(clip_samples=640 + 47 * 320),
}
LISTENER_CASES = [(s, c) for s in ("M", "L") for c in LISTENER_FRONTENDS]


@pytest.mark.parametrize("size,case", LISTENER_CASES, ids=[f"{s}-{c}" for s, c in LISTENER_CASES])
def test_emulated_listener(emu, size, case):
    """2 streams x 1 window, 3 pushes at hop = 2 frames: each push equal bit for bit to tcr_dscnn_forward_input on the cut clips."""
    run_case(emu, size, LISTENER_FRONTENDS[case], S=2, hop=2, K=1, pushes=3, reset_at=((2, 1),), pcm_every=2)


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


def _mode(monkeypatch, mode):
    if mode is None:
        monkeypatch.delenv("TCR_DSCNN_TC", raising=False)
    else:
        monkeypatch.setenv("TCR_DSCNN_TC", mode)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [None, "1", "0"], ids=["default", "TC1-lockstep", "TC0-fma"])
def test_cuda_reach_matches_the_handles_bounds(cuda, monkeypatch, mode):
    """The bounds of test_reach_matches_the_handles_bounds on the CUDA build, S in each TCR_DSCNN_TC mode (M and L run the FMA
    kernels in every mode): where the wgmma conv runs conv_1, no height is refused."""
    _mode(monkeypatch, mode)
    found = run_bounds(cuda.lib, mode, SIZES)
    assert found["S", "T", 49] == 374 and found["M", "T", 49] == 72 and found["L", "T", 49] == 42
    assert found["S", "F", 40] == (1310 if mode == "0" else None)


WORST = {}


@pytest.fixture(scope="module")
def worst_errors():
    yield WORST
    print("\n  worst per-layer errors: " + "; ".join(f"{k} {e:.1e} ({w})" for k, (e, w) in sorted(WORST.items())))


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _keep(where, errs, kernels):
    for k, e in zip(kernels, errs):
        if e >= WORST.get(k, (0.0,))[0]:
            WORST[k] = (e, where)


@pytest.mark.gpu
@pytest.mark.parametrize("size,T,F,mode,claims,why", GEOMETRIES, ids=IDS)
def test_cuda_layers_logits_and_invariance(cuda, monkeypatch, worst_errors, size, T, F, mode, claims, why):
    """Every layer within 1e-5 and the logits, with the kernel each layer launches named from reach(), at n = 1, 3, 39 and 100, and
    at the n that gives SM count + 1 tiles where a persistent wgmma kernel runs; the oracle checks a slice from both ends of the batch
    past ORACLE_FLOPS.  Then the logits of the largest batch are the same bits repeated, permuted, sliced and on a handle with
    another max_batch; at the WIDE rows once more with wide-range weights, each layer's channels held to their own maximum."""
    _mode(monkeypatch, mode)
    r = reach(size, T, F, mode)
    kernels = [x["kernel"] for x in r["layers"].values()]
    persistent = [x["tiles"] for x in r["layers"].values() if x["kernel"] not in ("dscnn_conv", "dscnn_dsblock")]
    ns = sorted({1, 3, 39, 100} | {-(-(_sms() + 1) // t) for t in persistent})
    per_utt = D.forward_flops(D.build_spec(size, T, F))
    net = _net(cuda, size, T, F, max(ns), seed=1)
    other = _net(cuda, size, T, F, 100, seed=1)
    try:
        for n in ns:
            k = max(2, int(ORACLE_FLOPS // per_utt))
            rows = None if k >= n else np.r_[0:k // 2, n - (k - k // 2):n]
            errs = check_layers(net, features(_kind(T, F), n, T, F, seed=n), kernels, rows, _logit_tol(size, T, F))
            _keep(f"{size} {T}x{F} n={n}", errs, kernels)
        feat = features(_kind(T, F), 100, T, F, seed=100)
        check_invariance(net, feat, other)
        if (size, T, F) in WIDE:
            wide = _net(cuda, size, T, F, 3, seed=1, wide=True)
            try:
                feat = features("randn", 3, T, F, seed=5)
                errs = check_layers(wide, feat, kernels, logit_tol=_logit_tol(size, T, F))
                _keep(f"{size} {T}x{F} wide-range n=3", errs, kernels)
                ratios, rels = channel_errors(wide, feat, kernels)
                print(f"  wide-range: worst channel per layer " + " ".join(f"{x:.2f}" for x in ratios) + " of its bound, "
                      + " ".join(f"{x:.1e}" for x in rels) + " of its maximum")
                assert max(ratios) <= 1, ratios
            finally:
                wide.close()
    finally:
        net.close()
        other.close()


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("classes", [1, 2, 17, 32])
def test_cuda_class_counts(cuda, monkeypatch, size, classes):
    monkeypatch.delenv("TCR_DSCNN_TC", raising=False)
    check_classes(cuda, size, classes, 39)


N = 65537
EDGE = np.r_[0:8, 65528:N]                # both sides of the first 65,535-row slice and the rows of the second


@pytest.mark.gpu
@pytest.mark.parametrize("size,T,F", [("M", 1, 1), ("L", 2, 1)])
def test_cuda_m_l_past_the_grid_bound(cuda, size, T, F):
    """n = 65,537 utterances: dscnn_dsblock takes one utterance per blockIdx.y and runs in two launches; the edge rows against the
    fp64 oracle, every row written."""
    net = _net(cuda, size, T, F, N, seed=2)
    try:
        feat = np.random.RandomState(2).randn(N, T, F).astype(np.float32)
        logits, probs = net.forward(feat)
        assert np.isfinite(logits).all() and np.isfinite(probs).all()
        err = rel_err(logits[EDGE], D.forward(net.spec, net.p, feat[EDGE].astype(np.float64)))
        print(f"  DS-CNN-{size} n=65537 edge rows vs fp64: {err:.1e}")
        assert err <= 1e-5, err
    finally:
        net.close()


@pytest.mark.gpu
@pytest.mark.parametrize("size,case", LISTENER_CASES, ids=[f"{s}-{c}" for s, c in LISTENER_CASES])
def test_cuda_listener(cuda, monkeypatch, size, case):
    """13 streams x 3 windows at hop = 3 frames, 5 pushes: each push equal bit for bit to tcr_dscnn_forward_input on the cut clips."""
    monkeypatch.delenv("TCR_DSCNN_TC", raising=False)
    run_case(cuda, size, LISTENER_FRONTENDS[case], S=13, hop=3, K=3, pushes=5, reset_at=((3, -1), (4, 12)))


@pytest.mark.gpu
@pytest.mark.parametrize("size,T,F", [("M", 47, 41), ("L", 48, 41), ("M", 49, 72)])
def test_cuda_tc_mode_leaves_m_and_l_unchanged(cuda, monkeypatch, size, T, F):
    """TCR_DSCNN_TC unset, 0 and 1: M and L launch the same FMA kernels and give the same logits bit for bit."""
    feat = features(_kind(T, F), 39, T, F, seed=4)
    runs = []
    for mode in (None, "0", "1"):
        _mode(monkeypatch, mode)
        net = _net(cuda, size, T, F, 39, seed=3)
        try:
            got = {}
            counts = launched(cuda.lib, lambda: got.setdefault("out", net.forward(feat)))
            runs.append((dict(counts), got["out"][0]))
        finally:
            net.close()
    assert runs[0][0] == {"dscnn_conv": 1, "dscnn_dsblock": NLAYERS[size] - 1, "dscnn_head": 1}, runs[0][0]
    for names, logits in runs[1:]:
        assert names == runs[0][0] and np.array_equal(logits, runs[0][1])


@pytest.mark.gpu
def test_cuda_refusal_through_the_model_class(cuda):
    """DSCNNMModel on an 80-bin log-mel front-end (49 x 80) raises the library's refusal when the model is built, not at the first
    batch."""
    from tcresnet_b200._lib import TcrError
    from tcresnet_b200.factory import audio_nets
    from tcresnet_b200.runtime import Node
    args = argparse.Namespace(num_classes=12, sample_rate=16000, clip_duration_ms=1000, window_size_ms=40.0, window_stride_ms=20.0,
                              num_mel_bins=80, num_mfccs=10, lower_edge_hertz=80.0, upper_edge_hertz=7600.0,
                              preprocess_method="log_mel_spectrogram", batch_size=3, output_name="output/softmax", weight_decay=0.0)
    model = audio_nets.DSCNNMModel(args, None)
    msg = reach("M", 49, 80)["refusal"]
    assert msg.startswith("dscnn_dsblock (conv_ds_1) needs 220160 bytes")
    with pytest.raises(TcrError, match=re.escape(f"status 3): {msg}")):
        model.build(Node("wavs", [None, 16000, 1]), Node("labels", [None, 12]), False)
