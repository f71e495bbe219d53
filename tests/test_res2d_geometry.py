"""The 2-D ablations (ResNet2D8 / ResNet2D8Pool) at the edges of every width, geometry, batch and class count their DS-CNN handle
accepts, against the fp64 oracle (res2d_oracle): reach(), a restatement of res2d_define's plan, checked against the handle's grid
refusals and swept over the accepted space; the refusals at the channel bounds; the parameter table, FLOPs, each layer and the
logits at each row of GEOMETRIES (channel counts that are not multiples of 4, the identity shortcut across filter slices, 1 and
128 channels, tiles shrunk to one row or column); 1 to 32 classes with the logits-only / probs-only calls and the evaluation
counts; the listener at more front-ends and widths; and TCR_DSCNN_TC.  Every kernel runs on the CPU emulator and on the GPU."""
import numpy as np
import pytest

from oracle import metrics_oracle as MO
from oracle import res2d_oracle as R
from tcr_harness import NumpyBackend, launched, rel_err
from test_dscnn import check_invariance, features, wide_range
from test_kws_geometry import _counts, _forward_one
from test_res2d import TCR_ERR_UNSUPPORTED, Res2dNet, check_net, create, table
from test_res2d_eval import check_layers, run_listener

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L

THREADS, MAX_CHANNELS = 256, 128                # res2d_conv0's block; kR2MaxChannels
COT_TARGET, SHRINK_AT, SMEM_LIMIT = 100 * 1024, 200 * 1024, 227 * 1024
GRID = 2 ** 31 - 1                              # the grid's x limit, in CTAs


def _pad4(c):
    return (c + 3) & ~3


def _cdiv(a, b):
    return -(-a // b)


def channels(Fq, wm):
    """res2d_define's channel counts (arrays broadcast): int(x * wm) of 16, 24, 32, 48 (wm = 0 means 1), then conv0's first_c, one
    rounded division of exact integers, where the first two are positive."""
    wm = np.where(np.asarray(wm) == 0, 1.0, wm)
    n = [np.floor(x * wm).astype(np.int64) for x in (16, 24, 32, 48)]
    first = np.floor((3 * np.asarray(Fq, np.int64) * n[0] + 10 * n[0] * n[1]) / (9 + 10 * n[1])).astype(np.int64)
    n[0] = np.where((n[0] >= 1) & (n[1] >= 1), first, n[0])
    return n


def _block_bytes(cip, cop, s, down, RH, WT, COT):
    """r2_block_smem: the input tile, the intermediate tile, one filter slice (conv_0's or conv_1's and down's) and six tables."""
    xr, xc = (RH + 1) * s + 3, (WT + 1) * s + 3
    return 4 * (xr * xc * cip + (RH + 2) * (WT + 2) * cop + (9 * np.maximum(cip, cop) + np.where(down, cip, 0)) * COT + 6 * cop)


def _block(cin, cout, h, w):
    """One block's plan on arrays: stride and pads, COT halved while the plan passes 100 KB and COT > 32, then RH or WT (the larger,
    RH on a tie) halved while it passes 200 KB, then both balanced over the tiles they need."""
    down = cout != cin
    s = np.where(down, 2, 1)
    hout, wout = _cdiv(h, s), _cdiv(w, s)
    pt, pl = np.maximum((hout - 1) * s + 3 - h, 0) // 2, np.maximum((wout - 1) * s + 3 - w, 0) // 2
    cip, cop = _pad4(cin), _pad4(cout)
    RH, WT, COT = np.minimum(hout, 8), np.minimum(wout, 16), cop
    while True:
        m = (_block_bytes(cip, cop, s, down, RH, WT, COT) > COT_TARGET) & (COT > 32)
        if not m.any():
            break
        COT = np.where(m, _pad4(COT // 2), COT)
    shrunk = np.zeros(np.shape(RH), bool)
    while True:
        m = (_block_bytes(cip, cop, s, down, RH, WT, COT) > SHRINK_AT) & ((RH > 1) | (WT > 1))
        if not m.any():
            break
        shrunk = shrunk | m
        wide = WT > RH
        WT, RH = np.where(m & wide, np.maximum(1, WT // 2), WT), np.where(m & ~wide, np.maximum(1, RH // 2), RH)
    RH, WT = _cdiv(hout, _cdiv(hout, RH)), _cdiv(wout, _cdiv(wout, WT))
    th, tw, slices = _cdiv(hout, RH), _cdiv(wout, WT), _cdiv(cop, COT)
    return dict(cin=cin, cout=cout, cip=cip, cop=cop, s=s, down=down, pt=pt, pl=pl, hout=hout, wout=wout, RH=RH, WT=WT,
                shrunk=shrunk, COT=COT, slices=slices, last_slice=cop - (slices - 1) * COT, tiles=th * tw,
                last_rows=hout - (th - 1) * RH, last_cols=wout - (tw - 1) * WT, smem=_block_bytes(cip, cop, s, down, RH, WT, COT))


def plan(model, T, Fq, wm):
    """res2d_define's plan on arrays of T, F and wm (broadcast): ok, the channel counts within 1 to 128; conv0 (hout, wout, RH rows
    per CTA, tiles per utterance, the last tile's rows, smem bytes, pstep positions in flight and idle threads, 256 % cout) and each
    block's _block.  Entries where ok is False are meaningless."""
    pool = model == "ResNet2D8Pool"
    ch = channels(Fq, wm)
    ok = np.logical_and.reduce([(c >= 1) & (c <= MAX_CHANNELS) for c in ch])
    ch = [np.where(ok, c, 1) for c in ch]
    T, Fq = np.asarray(T, np.int64), np.asarray(Fq, np.int64)
    ho, wo = (T // 4, Fq // 4) if pool else (T, Fq)
    RH = np.minimum(ho, 2 if pool else 8)
    tiles = _cdiv(ho, RH)
    conv0 = dict(hout=ho, wout=wo, RH=RH, tiles=tiles, last=ho - (tiles - 1) * RH, pstep=THREADS // ch[0], idle=THREADS % ch[0],
                 smem=4 * ((RH * (4 if pool else 1) + 2) * (Fq + 2) + 11 * ch[0]))
    blocks, h, w, cin = [], ho, wo, ch[0]
    for i in range(3):
        b = _block(cin, ch[i + 1], h, w)
        blocks.append(b)
        h, w, cin = b["hout"], b["wout"], b["cout"]
    return ok, ch, conv0, blocks


def reach(model, T, Fq, wm):
    """plan() at one configuration, as Python scalars: ch, the four channel counts; ok; head_scalar, the head's scalar path (the
    last block's channels not a multiple of 4); conv0 and b0, b1, b2 as plan() gives them."""
    ok, ch, conv0, blocks = plan(model, T, Fq, wm)
    scalar = lambda d: {k: (bool(v) if np.asarray(v).dtype == bool else int(v)) for k, v in d.items()}
    out = dict(ok=bool(ok), ch=tuple(int(c) for c in channels(Fq, wm)), conv0=scalar(conv0))
    out.update({f"b{i}": scalar(b) for i, b in enumerate(blocks)})
    out["head_scalar"] = out["ch"][3] % 4 != 0
    return out


def _claimed(got, claims):
    return {k: ({j: got[k][j] for j in v} if isinstance(v, dict) else got[k]) for k, v in claims.items()}


# (model, T, F, width multiplier, what the row reaches (checked against reach()), why it is here)
GEOMETRIES = [
    ("ResNet2D8", 98, 40, 1.3, dict(ch=(26, 31, 41, 62), head_scalar=True, conv0=dict(idle=22), b0=dict(cop=32),
                                    b1=dict(COT=24, slices=2, last_slice=20)),
     "every block's cout % 4 != 0 (the scalar store tail, padded intermediate channels); the head's scalar path; block 1 in "
     "slices of 24 + 20"),
    ("ResNet2D8", 98, 66, 1.3, dict(ch=(31, 31, 41, 62), b0=dict(down=False, s=1, cout=31, tiles=65, last_rows=2, last_cols=10)),
     "the identity shortcut at 31 channels on the full map, 65 tiles with partial last rows and columns"),
    ("ResNet2D8Pool", 98, 64, 1.3, dict(ch=(31, 31, 41, 62), b0=dict(down=False, hout=24, wout=16, tiles=3)),
     "the identity shortcut at 31 channels on the pooled 24 x 16 map"),
    ("ResNet2D8", 98, 107, 2.5, dict(ch=(60, 60, 80, 120), b0=dict(down=False, COT=32, slices=2, last_slice=28, tiles=91)),
     "the identity shortcut across two filter slices (32 + 28 channels)"),
    ("ResNet2D8", 98, 40, 2.6874, dict(ch=(49, 64, 85, 128), b1=dict(COT=24, slices=4, last_slice=16), b2=dict(cout=128, RH=2, WT=2)),
     "the widest width: 128 channels; cout 85 in slices of 24 ending in 16"),
    ("ResNet2D8Pool", 98, 40, 2.6874, dict(ch=(49, 64, 85, 128), b1=dict(COT=24, last_slice=16), b2=dict(RH=1, WT=2, shrunk=True)),
     "the widest width on the pool variant"),
    ("ResNet2D8", 8, 451, 2.68, dict(ch=(128, 64, 85, 128), conv0=dict(pstep=2, idle=0, tiles=1),
                                     b0=dict(cin=128, RH=1, WT=2, shrunk=True, smem=200704, tiles=452)),
     "conv0 at 128 channels; block 0 reads 128 channels, its tile shrunk to 1 x 2 at 196 KB"),
    ("ResNet2D8", 5, 813, 0.0625, dict(ch=(128, 1, 2, 3), b0=dict(cin=128, cout=1, cop=4, COT=4, tiles=51)),
     "the narrowest width at its widest F: block 0 goes from 128 channels to 1, COT = 4"),
    ("ResNet2D8", 5, 1240, 0.09, dict(ch=(128, 2, 2, 4), b1=dict(down=False, cout=2), b0=dict(cin=128, shrunk=True)),
     "the widest F the handle accepts (F = 1241 needs 129 channels in conv0); the identity shortcut at 2 channels"),
    ("ResNet2D8Pool", 4, 1240, 0.09, dict(ch=(128, 2, 2, 4), conv0=dict(hout=1, wout=310, RH=1), b1=dict(down=False)),
     "the pool variant's widest F: a 1 x 310 pooled map"),
    ("ResNet2D8", 3, 9, 0.0625, dict(ch=(1, 1, 2, 3), conv0=dict(pstep=256, idle=0), b0=dict(down=False, cout=1, cop=4)),
     "a 1-channel conv0 (every thread its own position); the identity shortcut at 1 channel"),
    ("ResNet2D8", 9, 564, 58 / 48, dict(ch=(125, 29, 38, 58), b0=dict(RH=1, WT=2, shrunk=True, tiles=705, smem=198400)),
     "the shrink drives block 0's RH to 1: 705 tiles per utterance at 194 KB"),
    ("ResNet2D8", 17, 17, 121 / 48, dict(ch=(42, 60, 80, 121), b2=dict(RH=1, WT=3, shrunk=True), b1=dict(COT=20, slices=4)),
     "the shrink drives block 2's RH to 1; block 1 in slices of 20"),
    ("ResNet2D8", 98, 17, 127.5 / 48, dict(ch=(44, 63, 85, 127), b2=dict(RH=2, WT=1, shrunk=True, tiles=21)),
     "the shrink drives block 2's WT to 1"),
    ("ResNet2D8", 17, 9, 125 / 48, dict(ch=(42, 62, 83, 125), b1=dict(COT=24, last_slice=12), b2=dict(smem=204784, shrunk=False)),
     "the largest shared-memory plan of the accepted space (test_sweep_of_the_accepted_space)"),
    ("ResNet2D8", 998, 128, 2.6874, dict(ch=(66, 64, 85, 128), b0=dict(tiles=1000, last_rows=3)),
     "the largest map at the widest width: block 0 has 1,000 tiles per utterance (GPU only)"),
    ("ResNet2D8", 998, 128, 2.5, dict(ch=(64, 60, 80, 120), b0=dict(tiles=1000), b2=dict(tiles=252)),
     "the accepted edge test_res2d.test_refusals only creates (GPU only)"),
]
IDS = [f"{'A' if m.endswith('Pool') else 'R'}-{t}x{f}-w{wm:.6g}" for m, t, f, wm, _, _ in GEOMETRIES]
BIG = {(998, 128)}                              # billions of FLOPs per utterance: minutes on the emulator
WIDE = {("ResNet2D8", 98, 40, 1.3), ("ResNet2D8", 98, 107, 2.5), ("ResNet2D8", 98, 40, 2.6874), ("ResNet2D8", 8, 451, 2.68),
        ("ResNet2D8", 17, 9, 125 / 48)}        # rows run once more with wide-range weights


@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


def _err(lib):
    return lib.tcr_last_error().decode()


@pytest.mark.parametrize("model,T,Fq,wm,claims,why", GEOMETRIES, ids=IDS)
def test_reach_matches_the_handles_grid_refusals(emu, model, T, Fq, wm, claims, why):
    """The handle reports its plan only through the grid refusals, made before anything is allocated: for conv0 and each block whose
    tile count t exceeds every earlier kernel's, max_batch = (2^31 - 1) // t + 1 is refused naming that kernel and t.  A plan that
    differs from reach() in the tile shape alone computes the same results, so only this check sees it."""
    got = reach(model, T, Fq, wm)
    assert _claimed(got, claims) == claims, (why, got)
    kernels = [("res2d_conv0", got["conv0"]["tiles"], "row tiles")] + [
        (f"res2d_block {i}", got[f"b{i}"]["tiles"], "tiles") for i in range(3)]
    checked, most = 0, 1
    for name, t, what in kernels:
        if t <= most:
            continue
        most = t
        mb = GRID // t + 1
        # a plan that accepted mb would ask for activation buffers of more than a TiB, which the allocation refuses; and t * t < 2^31
        # keeps mb x (an earlier kernel's count) under the grid's limit
        act = max(h * w * c for h, w, c in R.geometry(R.build_spec(model, T, Fq, 12, wm)))
        assert t * t < GRID and 4 * act * mb > 2 ** 40, (t, act, mb)
        rc, h = create(emu.lib, model, T, Fq, max_batch=mb, wm=wm)
        assert rc == TCR_ERR_UNSUPPORTED and not h.value, (name, t, rc, _err(emu.lib))
        assert f"{name}: max_batch {mb} x {t} {what} exceeds the grid's {GRID} CTAs" in _err(emu.lib), (name, t, _err(emu.lib))
        checked += 1
    assert checked >= (0 if (T, Fq) == (3, 9) else 1)


def _breakpoints():
    """Width multipliers where a channel count changes (k / x for x in 16, 24, 32, 48), and the midpoints between them, up to the
    first refused one."""
    b = sorted({k / x for x in (16, 24, 32, 48) for k in range(1, x * 129 // 48 + 2)})
    mids = [(u + v) / 2 for u, v in zip(b, b[1:])]
    return np.array(sorted(set(b) | set(mids)))


def test_sweep_of_the_accepted_space():
    """reach() over every width breakpoint and the midpoints between them, every F up to past the conv0 channel cap, and every T
    that puts each block's height at 1 to 8 (past 8 rows and 16 columns the plan before balancing is the same, and balancing only
    shrinks it): no plan passes 227 KB, so the two shared-memory refusals of res2d_define cannot be reached; the largest plans and
    the widest F are GEOMETRIES' rows; COT goes below 32."""
    wms = _breakpoints()
    Fs = np.arange(1, 1300)
    W, F = np.meshgrid(wms, Fs, indexing="ij")
    ok = channels(F, W)
    ok = np.logical_and.reduce([(c >= 1) & (c <= MAX_CHANNELS) for c in ok])
    assert not ok[:, -1].any()                                     # F = 1299 is past the cap at every width
    W, F = W[ok], F[ok]
    best, cots, conv0_max, configs = (0, None), set(), 0, 0
    for model, Ts, Fmin in (("ResNet2D8", range(1, 65), 1), ("ResNet2D8Pool", range(4, 260, 4), 4)):
        Fm, Wm = F[F >= Fmin], W[F >= Fmin]
        for T in Ts:
            _, ch, conv0, blocks = plan(model, T, Fm, Wm)
            conv0_max = max(conv0_max, int(conv0["smem"].max()))
            configs += Fm.size
            for i, b in enumerate(blocks):
                cots |= set(np.unique(b["COT"]).tolist())
                j = int(np.argmax(b["smem"]))
                if b["smem"][j] > best[0]:
                    best = (int(b["smem"][j]), (model, T, int(Fm[j]), float(Wm[j]), i, tuple(int(c[j]) for c in ch)))
    print(f"  {configs} configurations; largest block plan {best[0]} B, first at {best[1]} (model, T, F, wm, block, channels); "
          f"conv0 at most {conv0_max} B; COT {sorted(cots)}")
    assert best[0] == 204784 and best[1][0] == "ResNet2D8" and best[1][4] == 2 and best[1][5][1:] == (62, 83, 125), best
    assert best[0] <= SMEM_LIMIT and conv0_max <= SMEM_LIMIT and conv0_max == 4 * (10 * 1242 + 11 * 128)
    assert sorted(cots) == list(range(4, 52, 4))
    assert max(reach(m, T, f, wm)[b]["smem"] for m, T, f, wm, _, _ in GEOMETRIES for b in ("b0", "b1", "b2")) == best[0]
    assert int(F.max()) == 1240 and 1240 in {f for m, T, f, wm, _, _ in GEOMETRIES if m == "ResNet2D8Pool"}
    assert not plan("ResNet2D8", 8, np.array([1241]), np.array([0.09]))[0].any()


def _refused(lib, model, T, Fq, wm, needle):
    rc, h = create(lib, model, T, Fq, wm=wm)
    assert rc == TCR_ERR_UNSUPPORTED and not h.value and needle in _err(lib), (model, T, Fq, wm, _err(lib))


def _accepted(lib, model, T, Fq, wm, ch):
    rc, h = create(lib, model, T, Fq, wm=wm)
    assert rc == 0, (model, T, Fq, wm, _err(lib))
    try:
        conv = {n: s for n, s, _ in table(lib, h)[0] if n.endswith("/weights")}
        got = (conv[f"{model}/conv0/weights"][3],) + tuple(conv[f"{model}/block{i}/conv{i}_1/weights"][3] for i in range(3))
        assert got == ch == reach(model, T, Fq, wm)["ch"], (got, ch)
    finally:
        lib.tcr_dscnn_destroy(h)


def test_refusals_at_the_channel_bounds(emu):
    """Accepted at the last configuration of each bound and refused one step past it, naming the count: width 2.6874 / 2.6875
    (128 / 129 channels in block 2), 0.0625 / 0.0624 (1 / 0 in conv0), and conv0's 128 / 129 channels at the widest F of widths
    0.0625 (813), 1.0 (589) and 0.09 (1240, the widest F of all); the pool variant at 4 x 4 and not at 3 rows or columns."""
    lib = emu.lib
    for model in ("ResNet2D8", "ResNet2D8Pool"):
        _accepted(lib, model, 98, 40, 2.6874, (49, 64, 85, 128))
        _refused(lib, model, 98, 40, 2.6875, f"{model} at width_multiplier 2.6875 and width 40 needs 129 channels in a block; "
                                             "res2d_block takes 1 to 128")
        _accepted(lib, model, 98, 40, 0.0625, (6, 1, 2, 3))
        _refused(lib, model, 98, 40, 0.0624, "at width_multiplier 0.0624 and width 40 needs 0 channels in conv0")
        for wm, F, ch in ((0.0625, 813, (128, 1, 2, 3)), (1.0, 589, (128, 24, 32, 48)), (0.09, 1240, (128, 2, 2, 4))):
            _accepted(lib, model, 8, F, wm, ch)
            _refused(lib, model, 8, F + 1, wm, f"at width_multiplier {wm:g} and width {F + 1} needs 129 channels in conv0")
    _accepted(emu.lib, "ResNet2D8Pool", 4, 4, 0.0, tuple(R.channels(4)))
    for T, Fq in ((3, 4), (4, 3), (3, 40), (98, 3)):
        _refused(lib, "ResNet2D8Pool", T, Fq, 1.0, "ResNet2D8Pool needs height >= 4 and width >= 4")


@pytest.mark.parametrize("model,T,Fq,wm,claims,why", GEOMETRIES, ids=IDS)
def test_table_and_flops(emu, model, T, Fq, wm, claims, why):
    """tcr_dscnn_param_table and the FLOP count against res2d_oracle at each row, and reach()'s maps against the oracle's."""
    rc, h = create(emu.lib, model, T, Fq, wm=wm)
    assert rc == 0, _err(emu.lib)
    try:
        rows, nparams, flops = table(emu.lib, h)
        spec = R.build_spec(model, T, Fq, 12, wm)
        assert [(n, s) for n, s, _ in rows] == [(n, spec.var_shapes[n]) for n in spec.var_names]
        assert nparams == sum(int(np.prod(s)) for s in spec.var_shapes.values()) and flops == R.forward_flops(spec)
        got = reach(model, T, Fq, wm)
        assert [(got["conv0"]["hout"], got["conv0"]["wout"], got["ch"][0])] + [
            (got[f"b{i}"]["hout"], got[f"b{i}"]["wout"], got[f"b{i}"]["cout"]) for i in range(3)] == R.geometry(spec)
        assert all(got[f"b{i}"]["down"] == spec.blocks[i]["down"] for i in range(3))
    finally:
        emu.lib.tcr_dscnn_destroy(h)


def _wide(net):
    net.p = wide_range(net.spec, net.p)
    net.params = net.b.upload(R.flatten(net.spec, net.p))


@pytest.mark.parametrize("model,T,Fq,wm,claims,why", [g for g in GEOMETRIES if g[1:3] not in BIG],
                         ids=[i for g, i in zip(GEOMETRIES, IDS) if g[1:3] not in BIG])
def test_emulated_layers_and_logits(emu, model, T, Fq, wm, claims, why):
    """res2d_conv0, res2d_block and res2d_head layer by layer within 1e-5 with the NaN canary after the last utterance, and the
    logits within 1e-4: n = 2 (n = 1 past 4,000 input floats); at the WIDE rows once more with wide-range weights."""
    n = 1 if T * Fq > 4000 else 2
    net = Res2dNet(emu, model, T, Fq, n, seed=T + Fq, wm=wm)
    try:
        feat = features("randn", n, T, Fq, seed=T + Fq)
        for run in ("seeded", "wide-range") if (model, T, Fq, wm) in WIDE else ("seeded",):
            if run == "wide-range":
                _wide(net)
            errs, _ = check_net(net, feat)
            print(f"  {model} {T}x{Fq} w{wm:.6g} n={n} {run}: " + " ".join(f"{k} {e:.1e}" for k, e in errs.items()))
    finally:
        net.close()


def check_classes(b, model, T, Fq, classes, n):
    """n utterances at width 1.3 on a handle of `classes` classes: the logits and softmax against the oracle, the logits-only and
    probs-only calls equal to the call with both, and the evaluation counts of the logits against metrics_oracle's top-k counts."""
    net = Res2dNet(b, model, T, Fq, n, seed=classes, classes=classes, wm=1.3)
    try:
        assert reach(model, T, Fq, 1.3)["head_scalar"]
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
MODELS = pytest.mark.parametrize("model", ["ResNet2D8", "ResNet2D8Pool"])


@MODELS
@CLASS_COUNTS
def test_emulated_class_counts(emu, model, classes):
    """n = 5 on small maps (ResNet2D8 13 x 8, ResNet2D8Pool 16 x 16)."""
    check_classes(emu, model, *((13, 8) if model == "ResNet2D8" else (16, 16)), classes, 5)


# front-ends of the listener cases (tcr_config fields), keyed T x F: 128 log-mel bins, 41 and 42 of 64 MFCCs (odd and even history
# rows), and a clip of the smallest height each model takes (1 frame for ResNet2D8, 4 for ResNet2D8Pool's pool)
LISTENER_FRONTENDS = {
    "49x128-logmel": dict(feature_kind=L.TCR_FEATURE_LOG_MEL, num_mel_bins=128),
    "49x41": dict(num_mfccs=41, num_mel_bins=64),
    "49x42": dict(num_mfccs=42, num_mel_bins=64),
    "1x40": dict(clip_samples=640),
    "4x40": dict(clip_samples=1600),
}
LISTENER_CASES = [(m, c, wm) for m in ("ResNet2D8", "ResNet2D8Pool") for c in LISTENER_FRONTENDS for wm in (1.3, 2.6874)
                  if c not in ("1x40", "4x40") or (c == "4x40") == m.endswith("Pool")]
LISTENER_IDS = [f"{m}-{c}-w{wm:g}" for m, c, wm in LISTENER_CASES]


def _listen(b, model, case, wm, S, K_, pushes):
    """pushes fp32 and int16 chunks in turn, with a reset of every stream before the second to last push and of the last stream
    before the last one; hop = T - 1 (hop = K = 1 at T = 1)."""
    T = int(case.split("x")[0])
    resets = ((pushes - 2, -1), (pushes - 1, S - 1))
    run_listener(b, model, S=S, hop=max(1, T - 1), K_=1 if T == 1 else K_, pushes=pushes, reset_at=resets, pcm_every=2,
                 case=LISTENER_FRONTENDS[case], wm=wm)


@pytest.mark.parametrize("model,case,wm", LISTENER_CASES, ids=LISTENER_IDS)
def test_emulated_listener(emu, model, case, wm):
    """2 streams x 1 window (1 stream for ResNet2D8 on 49 frames: the emulator's slowest forwards), 3 pushes: each push equal bit for
    bit to the forward on the cut clips, and the carried history to the front-end's frames."""
    _listen(emu, model, case, wm, S=1 if model == "ResNet2D8" and case.startswith("49x") else 2, K_=1, pushes=3)


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
        kind = "logits" if k == "logits" else "res2d_conv0" if k == 1 else "res2d_block"
        kinds[kind] = max(kinds.get(kind, 0.0), e)
        if e >= WORST.get(kind, (0.0,))[0]:
            WORST[kind] = (e, f"{where} n={n}")
    print(f"  {where} n={n}: " + " ".join(f"{k} {e:.1e}" for k, e in sorted(kinds.items())))


@pytest.fixture(scope="module")
def worst_errors():
    yield WORST
    print("\n  worst error per kernel: " + "; ".join(f"{k} {e:.1e} ({w})" for k, (e, w) in sorted(WORST.items())))


@pytest.mark.gpu
@pytest.mark.parametrize("model,T,Fq,wm,claims,why", GEOMETRIES, ids=IDS)
def test_cuda_layers_logits_and_invariance(cuda, worst_errors, model, T, Fq, wm, claims, why):
    """Each layer within 1e-5 with the kernel it launches named, the logits within 1e-4, at n = 1, 3, 39 and 100 (n = 1 and 2 at
    998 x 128); then the logits of the largest batch are the same bits repeated, permuted, sliced and on a handle with another
    max_batch; at the WIDE rows the largest batch once more with wide-range weights."""
    ns = (1, 2) if (T, Fq) in BIG else (1, 3, 39, 100)
    where = f"{model} {T}x{Fq} w{wm:.6g}"
    net = Res2dNet(cuda, model, T, Fq, ns[-1] + 3, seed=1, wm=wm)
    other = Res2dNet(cuda, model, T, Fq, ns[-1], seed=1, wm=wm)
    try:
        for n in ns:
            _report(net, features("randn", n, T, Fq, seed=n), where)
        check_invariance(net, features("randn", ns[-1], T, Fq, seed=ns[-1]), other)
        if (model, T, Fq, wm) in WIDE:
            _wide(net)
            _report(net, features("randn", ns[-1], T, Fq, seed=1), where + " wide-range")
    finally:
        net.close()
        other.close()


@pytest.mark.gpu
@MODELS
@CLASS_COUNTS
def test_cuda_class_counts(cuda, model, classes):
    """n = 37 at 98 x 40."""
    check_classes(cuda, model, 98, 40, classes, 37)


@pytest.mark.gpu
@pytest.mark.parametrize("model,case,wm", LISTENER_CASES, ids=LISTENER_IDS)
def test_cuda_listener(cuda, model, case, wm):
    """13 streams x 3 windows at hop = T - 1 (7 streams x 1 window at T = 1), 5 pushes: each push equal bit for bit to the forward on
    the cut clips, and the push's first kernel is res2d_conv0:win."""
    _listen(cuda, model, case, wm, S=13 if case != "1x40" else 7, K_=3, pushes=5)


@pytest.mark.gpu
@MODELS
def test_cuda_tc_mode_leaves_res2d_kernels_unchanged(cuda, monkeypatch, model):
    """TCR_DSCNN_TC selects DS-CNN's kernels only: unset, 0 and 1 launch the same 2-D ablation kernels and give the same logits bit
    for bit, at width 1.3 (the scalar store tail and the head's scalar path)."""
    feat = features("mfcc", 39, 98, 40, seed=4)
    runs = []
    for mode in (None, "0", "1"):
        if mode is None:
            monkeypatch.delenv("TCR_DSCNN_TC", raising=False)
        else:
            monkeypatch.setenv("TCR_DSCNN_TC", mode)
        net = Res2dNet(cuda, model, 98, 40, 39, seed=3, wm=1.3)
        try:
            got = {}
            counts = launched(cuda.lib, lambda: got.setdefault("out", net.forward(feat)))
            runs.append((dict(counts), got["out"][0]))
        finally:
            net.close()
    assert runs[0][0] == {"res2d_conv0": 1, "res2d_block": 3, "res2d_head": 1}, runs[0][0]
    for names, logits in runs[1:]:
        assert names == runs[0][0] and np.array_equal(logits, runs[0][1])
    spec = R.build_spec(model, 98, 40, 12, 1.3)
    assert rel_err(runs[0][1], R.forward(spec, R.init_variables(spec, 3), feat.astype(np.float64))) <= 1e-4
