"""CPU oracle for the KWS baselines' forward pass (TEST INFRASTRUCTURE ONLY): cnn-trad-fpool3 and cnn-one-fstride4.

NumPy restatement in float64 of the two Sainath & Parada CNNs of audio_nets/kws.py in evaluation mode (the training dropouts are
the identity), as KWSModel --architecture trad_fpool3 / one_fstride4 builds them:
  trad_fpool3   20x8 conv 1 -> 64, ReLU, max-pool 1x3 / stride 1x3, 10x4 conv 64 -> 64, ReLU, flatten, three matmuls;
  one_fstride4  T x 8 conv 1 -> 186 with stride (1, 4), ReLU, flatten, four matmuls.
Every convolution and pool is VALID and every weight is bias-free; the input [N, T, F] is read as NHWC [N, T, F, 1].  The matmul
chain has no nonlinearity and is applied one matrix at a time.  Pinned by a torch.nn.functional cross-check in tests/test_kws.py.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List

import numpy as np

# size code of tcr_dscnn_config (include/tcr_b200.h) per --architecture
CODES = {"trad_fpool3": "P", "one_fstride4": "F"}


@dataclass
class KwsSpec:
    arch: str
    h: int
    w: int
    num_classes: int
    var_names: List[str]
    var_shapes: Dict[str, tuple]
    convs: List[tuple]           # (weight name, stride (time, freq), pool width) per conv layer
    mats: List[str]              # the matmul chain, in order


def conv_geometry(arch, h, w):
    """Output shapes (H, W, C) of the conv layers (after the pool for trad_fpool3's first)."""
    if arch == "trad_fpool3":
        h1, w1 = h - 19, (w - 7) // 3
        return [(h1, w1, 64), (h1 - 9, w1 - 3, 64)]
    return [(1, (w - 8) // 4 + 1, 186)]


def build_spec(arch="trad_fpool3", h=49, w=40, num_classes=12) -> KwsSpec:
    geo = conv_geometry(arch, h, w)
    k = int(np.prod(geo[-1]))
    if arch == "trad_fpool3":
        shapes = [("first_weights", (20, 8, 1, 64)), ("second_weights", (10, 4, 64, 64)), ("linear_weights", (k, 32)),
                  ("first_fc_weights", (32, 128)), ("final_fc_weights", (128, num_classes))]
        convs = [("first_weights", (1, 1), 3), ("second_weights", (1, 1), 1)]
    elif arch == "one_fstride4":
        shapes = [("first_weights", (h, 8, 1, 186)), ("first_linear_weights", (k, 32)), ("first_fc_weights", (32, 128)),
                  ("second_fc_weights", (128, 128)), ("final_fc_weights", (128, num_classes))]
        convs = [("first_weights", (1, 4), 1)]
    else:
        raise ValueError(arch)
    names = [n for n, _ in shapes]
    return KwsSpec(arch, h, w, num_classes, names, dict(shapes), convs, names[len(convs):])


def init_variables(spec: KwsSpec, seed=0, dtype=np.float64):
    """Seeded N(0, 2 / fan_in) weights, so that activations stay O(1) through the net (the reference's truncated normal with
    sigma = 0.01 would make every logit nearly zero)."""
    rng = np.random.RandomState(seed)
    out = {}
    for n in spec.var_names:
        s = spec.var_shapes[n]
        fan_in = int(np.prod(s[:-1]))
        out[n] = (rng.randn(*s) * np.sqrt(2.0 / fan_in)).astype(dtype)
    return out


def flatten(spec: KwsSpec, p, dtype=np.float32):
    return np.concatenate([np.asarray(p[n], dtype).ravel() for n in spec.var_names])


def _conv_valid(x, w, stride):
    """NHWC cross-correlation, VALID, HWIO weights.  A single input channel is one matmul of the im2col patches (a batch chunk at a
    time); more channels, one matmul per tap."""
    n, h, wd, cin = x.shape
    kh, kw, _, cout = w.shape
    oh, ow = (h - kh) // stride[0] + 1, (wd - kw) // stride[1] + 1
    out = np.zeros((n, oh, ow, cout), x.dtype)
    if cin == 1:
        win = np.lib.stride_tricks.sliding_window_view(x[..., 0], (kh, kw), axis=(1, 2))[:, ::stride[0], ::stride[1]]
        step = max(1, (1 << 22) // (oh * ow * kh * kw))
        for b in range(0, n, step):
            out[b:b + step] = win[b:b + step].reshape(-1, oh, ow, kh * kw) @ w.reshape(kh * kw, cout)
        return out
    for i in range(kh):
        for j in range(kw):
            out += x[:, i:i + stride[0] * (oh - 1) + 1:stride[0], j:j + stride[1] * (ow - 1) + 1:stride[1], :] @ w[i, j]
    return out


def layer(spec: KwsSpec, p, l, x):
    """Conv layer l (conv + ReLU, then trad_fpool3's 1x3 max-pool after its first): x [N, H, W, Cin] NHWC (layer 0 also takes the
    features [N, H, W]) -> [N, Hout, Wout, Cout]."""
    name, stride, pool = spec.convs[l]
    if x.ndim == 3:
        x = x[..., None]
    y = np.maximum(_conv_valid(x, p[name], stride), 0)
    if pool > 1:
        n, h, w, c = y.shape
        wp = w // pool
        y = y[:, :, :wp * pool, :].reshape(n, h, wp, pool, c).max(axis=3)
    return y


def forward_layers(spec: KwsSpec, p, feat):
    acts, x = [], feat
    for l in range(len(spec.convs)):
        x = layer(spec, p, l, x)
        acts.append(x)
    return acts


def head(spec: KwsSpec, p, x):
    """flatten (NHWC order) and the matmul chain: [N, H, W, C] -> logits [N, classes]."""
    y = x.reshape(x.shape[0], -1)
    for name in spec.mats:
        y = y @ p[name]
    return y


def forward(spec: KwsSpec, p, feat):
    """feat [N, T, F] -> logits [N, classes]."""
    return head(spec, p, forward_layers(spec, p, feat)[-1])


def forward_flops(spec: KwsSpec) -> int:
    """2 x multiply-adds of the convs (before the pool) and the matmuls; the pool is not counted."""
    f, h, w, cin = 0, spec.h, spec.w, 1
    for name, stride, pool in spec.convs:
        kh, kw, _, cout = spec.var_shapes[name]
        oh, ow = (h - kh) // stride[0] + 1, (w - kw) // stride[1] + 1
        f += 2 * oh * ow * kh * kw * cin * cout
        h, w, cin = oh, ow // pool, cout
    return f + sum(2 * int(np.prod(spec.var_shapes[m])) for m in spec.mats)


def l2_loss(p):
    """sum of tf.nn.l2_loss over every weight: sum(w ** 2) / 2."""
    return sum(0.5 * float(np.sum(np.asarray(v, np.float64) ** 2)) for v in p.values())
