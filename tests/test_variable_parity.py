"""One training step held to the fp64 oracle variable by variable and layer by layer, across the weight-gradient launch's plan.

The flat checks of parity_cases.check_step bound max|x - ref| / max|ref| over whole buffers, and one variable sets that max:
conv0/weights sees the MFCC features (coefficient 0 is large), every other gradient is 1 to 5 orders of magnitude smaller, so a
wrong block-conv or BatchNorm gradient can pass them by percents.  Here every variable and every layer tensor is held to 1e-4 of
ITS OWN max, with the oracle taking the CUDA path's ReLU decisions (cuda_relu_masks):
  * gradient, momentum slot: max|x - ref| / max|ref| <= 1e-4 per variable;
  * update dp = p1 - p0 against the oracle's: |dp - dp_ref| <= 1e-4 max|dp_ref| + 1 fp32 ulp of the stored p1, elementwise (the
    flat parameter comparison is dominated by p0); the same rule for the moving statistics' update;
  * per conv: pre-BatchNorm output y, batch mean, rstd and biased variance, the masked gradient dz the weight-gradient launch reads
    (g:<conv> for conv0 / conv_a, g:block<i> for conv_b / the shortcut conv) and the BatchNorm-backward sums (sum dz, sum dz xhat).
A wrong dz points at backward-data, a right dz with a wrong weights gradient at the weight-gradient launch (dw_grouped).

dw_grouped runs a static plan (plan_bwd_weight, csrc/tcr_net_bwd.cu, built at tcr_create from max_batch, the SM count and the
knobs TCR_DW_UPC / TCR_DW_SLOTS) at the runtime n.  dw_plan restates it; each case asserts the plan features it was built to
exercise, and the plan is pinned against the handle through its debug timeline (TCR_DEBUG_TIMELINE=1: CTA vb of dw_grouped
records its table row and row chunk at timeline row 4096 + vb).
"""
import ctypes as C
import time

import numpy as np
import pytest

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L
from oracle import tcr_oracle as O
from parity_cases import cuda_relu_masks, perturbed_variables, reference_features
from tcr_harness import Engine, NumpyBackend, rel_err

TOL = 1e-4
DW_THREADS = 256                      # kDwThreads
SMEM_BUDGET_W = 64 * 1024             # kSmemBudgetW: staged utterances are cut down to this
SMEM_BUDGET = 110 * 1024              # kSmemBudget: row groups are cut down to this
TL_DW_ROW, TL_ROWS = 4096, 16 * 8192 // 8    # timeline: 8 int64 per CTA, dw_grouped's CTAs from row 4096


# ------------------------------------------------------------------------------------------------
# plan_bwd_weight, restated
# ------------------------------------------------------------------------------------------------
def bwd_weight_smem(cv, cot, RG, UB):
    pad_right = max((cv.t_out - 1) * cv.stride + cv.k - cv.pad_left - cv.t_in, 0)
    tp = cv.pad_left + cv.t_in + pad_right
    tiles = (UB * tp * cv.cin + UB * cv.t_out * cot + 4 * cv.cin + 2 * cv.cout + DW_THREADS) * 4
    scratch = (RG - 1) * (cv.cin // 2) * (cot // 4) * cv.k * 8 * 4
    return max(tiles, scratch)


def dw_plan(spec, sms, max_batch, slots=None, upc_cap=None, trained_convs=None):
    """Per layer of the grouped launch's table (conv0, then conv_a, shortcut, conv_b of each block, only the convs whose weights
    are trained): dict(cv, cot, ncot, RG, R, UB).  The chunking is planned over every conv, trained or not."""
    slots = 2 * sms if slots is None else slots
    upc_cap = 256 if upc_cap is None else upc_cap
    plan = {}
    for cv in spec.convs():
        cot = 4
        for c in range(4, cv.cout + 1, 4):
            if cv.cout % c == 0 and (cv.cin // 2) * (c // 4) <= DW_THREADS:
                cot = c
        tau = 0.9 + float(cv.t_out * cv.k * cv.cin * cot) / 70e3
        plan[cv.name] = dict(cv=cv, cot=cot, ncot=cv.cout // cot, tau=tau)

    def upc_at(d, p):
        return max(1, min(upc_cap, int(d / p["tau"])))

    def ctas_at(d):
        return sum(p["ncot"] * -(-max_batch // upc_at(d, p)) for p in plan.values())

    d = 1.0
    while ctas_at(d) > slots and d < 1e5:
        d *= 1.05
    for p in plan.values():
        cv = p["cv"]
        rg = max(1, min(4, DW_THREADS // ((cv.cin // 2) * (p["cot"] // 4))))
        p["R"] = max(1, -(-max_batch // upc_at(d, p)))
        ub = 8
        while ub > 1 and bwd_weight_smem(cv, p["cot"], rg, ub) > SMEM_BUDGET_W:
            ub -= 1
        while rg > 1 and bwd_weight_smem(cv, p["cot"], rg, ub) > SMEM_BUDGET:
            rg -= 1
        p["RG"], p["UB"] = rg, ub
    order = [spec.conv0.name]
    for b in spec.blocks:
        order += [b.conv_a.name] + ([b.down.name] if b.down is not None else []) + [b.conv_b.name]
    return [plan[c] for c in order if trained_convs is None or c in trained_convs]


def plan_features(table, n):
    """The plan features layer by layer at runtime batch n: {feature: [conv names]}."""
    feats = {}

    def add(f, name):
        feats.setdefault(f, []).append(name)

    for p in table:
        cv, upc = p["cv"], -(-n // p["R"])
        sizes = [max(0, min(n, (c + 1) * upc) - c * upc) for c in range(p["R"])]
        name = cv.name
        add(f"K{cv.k}", name)
        if cv.stride == 2:
            add("stride2", name)
        if p["R"] > 1:
            add("chunks", name)
            if any(0 < s < upc for s in sizes):
                add("partial_chunk", name)
        if 0 in sizes:
            add("empty_chunks", name)
        if any(s % p["UB"] for s in sizes if s):
            add("partial_stage", name)
        if cv.t_out % p["RG"]:
            add("t_out_rem", name)
        if p["ncot"] > 1:
            add("ncot", name)
    return feats


# ------------------------------------------------------------------------------------------------
# workspace access
# ------------------------------------------------------------------------------------------------
def fill(eng, name, byte):
    """memset a workspace tensor (0xFF: NaN as fp32, -1 as int64)."""
    p, numel = C.c_void_p(), C.c_int64()
    L.check(eng.lib, eng.lib.tcr_workspace_tensor(eng.h, name.encode(), C.byref(p), C.byref(numel)), name)
    if eng.b.name == "emu":
        C.memset(p.value, byte, numel.value * 4)
    else:
        rt = C.CDLL("libcudart.so.12")
        rt.cudaMemset.argtypes = [C.c_void_p, C.c_int, C.c_size_t]
        assert rt.cudaMemset(p.value, byte, numel.value * 4) == 0
        eng.b.sync()


def sm_count(backend):
    if backend.name == "emu":
        return 1                                          # the emulator's handle keeps h->sms = 1
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def pin_plan(eng, table):
    """dw_grouped CTA vb = cta_begin(l) + bx + ncot * by: the rows the launch wrote must be exactly the restated table's."""
    tl = eng.workspace("timeline").view(np.int64).reshape(-1, 8)
    want = np.array([(l, local // p["ncot"]) for l, p in enumerate(table) for local in range(p["ncot"] * p["R"])], np.int64)
    got = tl[TL_DW_ROW:TL_DW_ROW + len(want), 3:5]
    assert np.array_equal(got, want), "dw_grouped's (layer, row chunk) per CTA differs from the restated plan"
    if TL_DW_ROW + len(want) < TL_ROWS:
        assert tl[TL_DW_ROW + len(want), 3] == -1, "dw_grouped launched more CTAs than the restated plan"


# ------------------------------------------------------------------------------------------------
# the step
# ------------------------------------------------------------------------------------------------
def step_case(backend, monkeypatch, model="TCResNet8", wm=1.0, n=8, max_batch=None, keep=0.5, window=640, stride=320, clip=16000,
              upc=None, slots=None, trained_prefixes=None, expect=(), tag=""):
    t0 = time.time()
    max_batch = max_batch or n
    t = O.num_frames(clip, window, stride)
    spec = O.build_spec(model, wm, t)
    sc = spec.scope
    trained = None
    if trained_prefixes is not None:
        trained = [v for v in spec.var_names if any(v.startswith(f"{sc}/{p}/") for p in trained_prefixes)]
    trained_convs = None if trained is None else {cv.name for cv in spec.convs() if f"{sc}/{cv.name}/weights" in trained}
    bwd_convs = [cv for cv in spec.convs() if trained is None or any(v.startswith(f"{sc}/{cv.name}/") for v in trained)]

    table = dw_plan(spec, sm_count(backend), max_batch, slots, upc, trained_convs)
    feats = plan_features(table, n)
    missing = set(expect) - set(feats)
    assert not missing, (f"plan no longer exercises {sorted(missing)}", {k: v for k, v in feats.items()})
    assert sum(p["ncot"] * p["R"] for p in table) <= TL_ROWS - TL_DW_ROW

    monkeypatch.setenv("TCR_DEBUG_TIMELINE", "1")
    for knob, v in (("TCR_DW_UPC", upc), ("TCR_DW_SLOTS", slots)):
        if v is None:
            monkeypatch.delenv(knob, raising=False)
        else:
            monkeypatch.setenv(knob, str(v))
    eng = Engine(backend, model=int(model[len("TCResNet"):]), width_multiplier=wm, max_batch=max_batch, dropout_keep_prob=keep,
                 window_size_samples=window, window_stride_samples=stride, clip_samples=clip)
    try:
        assert eng.info.frames == t
        if trained is not None:
            flags = (C.c_int32 * len(spec.var_names))(*[int(v in trained) for v in spec.var_names])
            L.check(eng.lib, eng.lib.tcr_set_trainable(eng.h, flags, len(spec.var_names)), "tcr_set_trainable")
        params, moving = perturbed_variables(spec)
        rng = np.random.RandomState(7)
        slots0 = {k: 0.01 * rng.randn(*v.shape) for k, v in params.items()}
        wav, onehot = O.synthetic_batch(n, num_samples=clip, adversarial=True)
        feat = reference_features(wav, window, stride)
        mask = (rng.rand(n, spec.c_last) < keep).astype(np.float32) if keep < 1 else None
        lr, mom, wd = 0.1, 0.9, 1e-3
        pf, mf, sf = O.flatten_vars(spec, params), O.flatten_moving(spec, moving), O.flatten_vars(spec, slots0)

        # whatever is checked below must come from this step: NaN into the backward tensors, -1 into the timeline
        for cv in spec.convs():
            fill(eng, f"bsum:{cv.name}", 0xFF)
            if cv is spec.conv0 or any(cv is b.conv_a for b in spec.blocks):
                fill(eng, f"g:{cv.name}", 0xFF)
        for b in spec.blocks:
            fill(eng, f"g:block{b.index}", 0xFF)
        fill(eng, "timeline", 0xFF)

        ts = eng.train_step(wav, onehot, pf, sf, mf, lr, mom, wd, mask_np=mask)
        pin_plan(eng, table)
        forced = cuda_relu_masks(eng, spec, n)
        p0, mv0, s0 = O.unflatten_vars(spec, pf), O.unflatten_moving(spec, mf), O.unflatten_vars(spec, sf)
        p1_ref, mv1_ref, s1_ref, ref = O.train_step(spec, p0, mv0, s0, feat, onehot, lr, mom, wd, keep, mask, 0.0,
                                                    forced_masks=forced)
        var_err = check_variables(spec, ts, ref, p0, s0, p1_ref, s1_ref, mv0, mv1_ref, trained)
        layer_err = check_layers(eng, spec, ref["cache"], ref["grads"], n, bwd_convs)
        assert rel_err(ts["logits"], ref["logits"]) <= TOL
        assert abs(ts["losses"][0] - ref["total_loss"]) <= 1e-4 * abs(ref["total_loss"]) + 1e-6
        assert abs(ts["losses"][1] - ref["model_loss"]) <= 1e-4 * abs(ref["model_loss"]) + 1e-6
    finally:
        eng.close()
    worst = []
    for kind in ("grad", "update", "slot", "moving"):
        k = max((k for k in var_err if k[0] == kind), key=var_err.get)
        worst.append(f"{kind} {var_err[k]:.2e} ({k[1][len(sc) + 1:]})")
    wl = max(layer_err, key=layer_err.get)
    print(f"\n[{tag}] worst per variable: {'; '.join(worst)}; worst layer tensor {layer_err[wl]:.2e} ({wl}); "
          f"plan features {sorted(feats)}; {time.time() - t0:.1f} s")
    return var_err, layer_err, feats


def check_variables(spec, ts, ref, p0, s0, p1_ref, s1_ref, mv0, mv1_ref, trained):
    g = O.unflatten_vars(spec, ts["grads"])
    p1 = O.unflatten_vars(spec, ts["params"], np.float32)
    s1 = O.unflatten_vars(spec, ts["slots"])
    mv1 = O.unflatten_moving(spec, ts["moving"], np.float32)
    err, fails = {}, []

    def bound(kind, name, got, ref_v):
        err[kind, name] = e = rel_err(got, ref_v)
        if not e <= TOL:
            fails.append((e, kind, name))

    def update(kind, name, new32, old, new_ref):
        """new - old against new_ref - old, to 1e-4 of the oracle's largest step plus one ulp of the stored fp32 value."""
        d, d_ref = np.asarray(new32, np.float64) - old, new_ref - old
        lim = TOL * np.abs(d_ref).max() + np.spacing(np.abs(np.asarray(new32, np.float32))).astype(np.float64)
        err[kind, name] = np.abs(d - d_ref).max() / max(np.abs(d_ref).max(), 1e-30)
        if not np.all(np.abs(d - d_ref) <= lim):
            fails.append((float(np.max(np.abs(d - d_ref) / lim)) * TOL, kind, name))

    for name in spec.var_names:
        if trained is not None and name not in trained:      # frozen: zero gradient, parameter and slot untouched
            assert not g[name].any() and np.array_equal(p1[name], p0[name].astype(np.float32)), name
            assert np.array_equal(s1[name], s0[name]), name
            continue
        bound("grad", name, g[name], ref["grads"][name])
        bound("slot", name, s1[name], s1_ref[name])
        update("update", name, p1[name], p0[name], p1_ref[name])
    for name in O.moving_names(spec):
        update("moving", name, mv1[name], mv0[name], mv1_ref[name])
    fails.sort(reverse=True)
    assert not fails, f"worst: {fails[0][1]} of {fails[0][2]} at {fails[0][0]:.3e} of its own scale; all failing: {fails}"
    return err


def check_layers(eng, spec, cache, grads, n, bwd_convs):
    err, fails = {}, []

    def bound(key, got, ref_v):
        err[key] = e = rel_err(got, ref_v)
        if not e <= TOL:                                   # NaN (a tensor this step did not write) fails too
            fails.append((e, key))

    sc = spec.scope
    for cv in spec.convs():
        c = cache[cv.name]
        bound(f"y:{cv.name}", eng.workspace(f"y:{cv.name}").reshape(-1, cv.t_out, cv.cout)[:n], c["y"])
        bnf = eng.workspace(f"bnf:{cv.name}").reshape(4, cv.cout)
        _, rstd, mean, var, _ = c["bn"]
        bound(f"mean:{cv.name}", bnf[0], mean)
        bound(f"rstd:{cv.name}", bnf[1], rstd)
        bound(f"var:{cv.name}", eng.workspace(f"var:{cv.name}"), var)
    for cv in bwd_convs:
        if cv is spec.conv0 or any(cv is b.conv_a for b in spec.blocks):
            bound(f"g:{cv.name}", eng.workspace(f"g:{cv.name}").reshape(-1, cv.t_out, cv.cout)[:n], cache[cv.name]["dz"])
        bs = eng.workspace(f"bsum:{cv.name}").reshape(2, cv.cout)
        bound(f"sum_dz:{cv.name}", bs[0], grads[f"{sc}/{cv.name}/BatchNorm/beta"])
        bound(f"sum_dz_xhat:{cv.name}", bs[1], grads[f"{sc}/{cv.name}/BatchNorm/gamma"])
    names = {cv.name for cv in bwd_convs}
    for b in spec.blocks:
        if b.conv_b.name in names or (b.down is not None and b.down.name in names):
            key = f"g:block{b.index}"
            bound(key, eng.workspace(key).reshape(-1, b.conv_b.t_out, b.conv_b.cout)[:n], cache[f"block{b.index}"]["g"])
    fails.sort(reverse=True)
    assert not fails, f"worst layer tensor: {fails[0][1]} at {fails[0][0]:.3e} of its own scale; all failing: {fails}"
    return err


# ------------------------------------------------------------------------------------------------
# emulator cases (CPU)
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return NumpyBackend()


ALL_BODIES = ("K1", "K3", "K9", "stride2", "t_out_rem")
EMU_KNOBS = {
    # sms = 1 on the emulator: the default plan already fits one chunk per layer
    "default": (dict(n=8, max_batch=8), ()),
    # R = max_batch: one utterance per chunk, every staging batch partial
    "upc1": (dict(n=8, max_batch=8, upc=1), ("chunks", "partial_stage")),
    # upc 3 of 16: R = 6; n = 7 runs chunks of 2, 2, 2, 1, 0, 0
    "upc3-n7-of-16": (dict(n=7, max_batch=16, upc=3), ("chunks", "partial_chunk", "empty_chunks", "partial_stage")),
    # one chunk of all 5 utterances on a 16-utterance plan: 5 < UB staged
    "slots1-n5-of-16": (dict(n=5, max_batch=16, slots=1), ("partial_stage",)),
}


@pytest.mark.parametrize("knobs", list(EMU_KNOBS))
@pytest.mark.parametrize("model", ["TCResNet8", "TCResNet14"])
def test_emulated_step_per_variable(emu, monkeypatch, model, knobs):
    """TCResNet14 adds identity-shortcut blocks (1, 3, 5) to the downsampling ones."""
    kw, expect = EMU_KNOBS[knobs]
    step_case(emu, monkeypatch, model=model, expect=ALL_BODIES + expect, tag=f"{model}-{knobs}", **kw)


def test_emulated_three_output_channel_tiles(emu, monkeypatch):
    """TCResNet8-1.5: the 72 -> 72 conv2_1 runs three 24-channel tiles (bx = 0, 1, 2) of every row chunk."""
    _, _, feats = step_case(emu, monkeypatch, wm=1.5, n=6, max_batch=8, upc=2, expect=ALL_BODIES + ("ncot", "chunks"),
                            tag="TCResNet8x1.5-upc2")
    assert "block2/conv2_1" in feats["ncot"]


def test_emulated_trainable_subset(emu, monkeypatch):
    """Block 2 and fc trained: the grouped table holds conv2_0, down, conv2_1 only, from cta_begin 0; frozen variables keep a zero
    gradient and their values."""
    step_case(emu, monkeypatch, n=7, max_batch=16, upc=3, trained_prefixes=("block2", "fc"),
              expect=("K1", "K9", "stride2", "chunks", "partial_chunk", "empty_chunks"), tag="TCResNet8-block2+fc")


# ------------------------------------------------------------------------------------------------
# GPU cases
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


@pytest.mark.gpu
@pytest.mark.parametrize("resident", [None, "0", "1"], ids=["default", "resident0", "resident1"])
def test_step_per_variable_n512(cuda, monkeypatch, resident):
    """Backward-data differs between the kernel modes; the weight-gradient launch does not."""
    if resident is not None:
        monkeypatch.setenv("TCR_RESIDENT", resident)
    step_case(cuda, monkeypatch, n=512, expect=ALL_BODIES + ("chunks", "partial_chunk", "partial_stage", "ncot"),
              tag=f"TCResNet8-n512-{resident or 'default'}")


@pytest.mark.gpu
def test_step_per_variable_below_max_batch(cuda, monkeypatch):
    """n = 133 and 1 on a plan made for 512: the real plan's chunks are partly or entirely empty."""
    step_case(cuda, monkeypatch, n=133, max_batch=512, expect=ALL_BODIES + ("partial_chunk", "empty_chunks"), tag="TCResNet8-n133-of-512")
    step_case(cuda, monkeypatch, n=1, max_batch=512, expect=ALL_BODIES + ("empty_chunks", "partial_stage"),
              tag="TCResNet8-n1-of-512")


@pytest.mark.gpu
def test_step_per_variable_tcresnet14x15_n1024(cuda, monkeypatch):
    step_case(cuda, monkeypatch, model="TCResNet14", wm=1.5, n=1024, expect=ALL_BODIES + ("chunks", "partial_chunk", "ncot"),
              tag="TCResNet14x1.5-n1024")


@pytest.mark.gpu
def test_step_per_variable_width_2_5_t98(cuda, monkeypatch):
    step_case(cuda, monkeypatch, wm=2.5, n=256, window=480, stride=160, expect=ALL_BODIES + ("ncot", "chunks"),
              tag="TCResNet8x2.5-T98-n256")


@pytest.mark.gpu
def test_step_per_variable_t148(cuda, monkeypatch):
    """1.5 s clips at 30/10 ms windows: T = 148.  The longer staging tiles cut the staged utterances of the layers named below."""
    spec98, spec148 = O.build_spec("TCResNet8", 1.0, 98), O.build_spec("TCResNet8", 1.0, 148)
    sms = sm_count(cuda)
    shrunk = [a["cv"].name for a, b in zip(dw_plan(spec98, sms, 256), dw_plan(spec148, sms, 256)) if b["UB"] < a["UB"]]
    assert shrunk, "T = 148 no longer stages fewer utterances than T = 98 in any layer"
    print(f"\nT = 148 stages fewer utterances than T = 98 in {shrunk}")
    step_case(cuda, monkeypatch, n=256, window=480, stride=160, clip=24000, expect=ALL_BODIES + ("chunks",), tag="TCResNet8-T148-n256")


@pytest.mark.gpu
def test_step_per_variable_one_utterance_per_chunk(cuda, monkeypatch):
    step_case(cuda, monkeypatch, n=512, upc=1, expect=ALL_BODIES + ("chunks", "partial_stage"), tag="TCResNet8-n512-upc1")
