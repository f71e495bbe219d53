"""CPU oracle for the DS-CNN forward pass (TEST INFRASTRUCTURE ONLY) — config 5 of BASELINE.json.

NumPy restatement of audio_nets/ds_cnn.py (Hello-Edge DS-CNN) in inference mode under DSCNN_arg_scope
(ds_cnn.py:104-118): slim.conv2d / slim.separable_convolution2d with zero-initialised BIASES and no activation,
each followed by slim.batch_norm(decay 0.96, scale=False -> no gamma, center=True, eps 0.001, ReLU), global
average pool, fully connected with bias (ds_cnn.py:46-101).  Input [N, H, W, 1] (H = frames, W = coefficients).
PARITY UNPINNED (no TF, no reference goldens): pinned by a torch.nn.functional cross-check in tests/test_dscnn.py.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List

import numpy as np

BN_EPS = 1e-3

# Block(type, depth, kernel, stride, scope): S/M/L_NET_DEF, ds_cnn.py:20-43
NET_DEFS = {
    "S": [("conv", 64, (10, 4), (2, 2), "conv_1")] + [("separable", 64, (3, 3), (1, 1), f"conv_ds_{i}") for i in range(1, 5)],
    "M": [("conv", 172, (10, 4), (2, 1), "conv_1"), ("separable", 172, (3, 3), (2, 2), "conv_ds_1")]
         + [("separable", 172, (3, 3), (1, 1), f"conv_ds_{i}") for i in range(2, 5)],
    "L": [("conv", 276, (10, 4), (2, 1), "conv_1"), ("separable", 276, (3, 3), (2, 2), "conv_ds_1")]
         + [("separable", 276, (3, 3), (1, 1), f"conv_ds_{i}") for i in range(2, 6)],
}


def same_pad(length, k, s):
    out = -(-length // s)
    total = max((out - 1) * s + k - length, 0)
    return out, total // 2, total - total // 2


@dataclass
class DsSpec:
    size: str
    h: int
    w: int
    num_classes: int
    var_names: List[str]
    var_shapes: Dict[str, tuple]


def build_spec(size="S", h=49, w=40, num_classes=12) -> DsSpec:
    names, shapes = [], {}

    def add(n, s):
        names.append(n)
        shapes[n] = tuple(s)

    cin = 1
    for typ, depth, k, _, scope in NET_DEFS[size]:
        if typ == "conv":
            add(f"DSCNN/{scope}/weights", (k[0], k[1], cin, depth))
            add(f"DSCNN/{scope}/biases", (depth,))
            for p in ("beta", "moving_mean", "moving_variance"):
                add(f"DSCNN/{scope}/batch_norm/{p}", (depth,))
        else:
            add(f"DSCNN/{scope}/depthwise_conv/depthwise_weights", (k[0], k[1], cin, 1))
            add(f"DSCNN/{scope}/depthwise_conv/biases", (cin,))
            for p in ("beta", "moving_mean", "moving_variance"):
                add(f"DSCNN/{scope}/dw_batch_norm/{p}", (cin,))
            add(f"DSCNN/{scope}/pointwise_conv/weights", (1, 1, cin, depth))
            add(f"DSCNN/{scope}/pointwise_conv/biases", (depth,))
            for p in ("beta", "moving_mean", "moving_variance"):
                add(f"DSCNN/{scope}/pw_batch_norm/{p}", (depth,))
        cin = depth
    add("DSCNN/fc1/weights", (cin, num_classes))
    add("DSCNN/fc1/biases", (num_classes,))
    return DsSpec(size, h, w, num_classes, names, shapes)


def init_variables(spec: DsSpec, seed=0, dtype=np.float64):
    """Random but non-trivial values for every variable (training is out of scope: weights are always injected)."""
    rng = np.random.RandomState(seed)
    out = {}
    for n in spec.var_names:
        s = spec.var_shapes[n]
        if n.endswith("weights"):
            fan_in = int(np.prod(s[:-1])) if len(s) == 4 else s[0]
            fan_out = s[-1] * (s[0] * s[1] if len(s) == 4 else 1)
            lim = np.sqrt(6.0 / (fan_in + fan_out))
            out[n] = rng.uniform(-lim, lim, size=s)
        elif n.endswith("moving_variance"):
            out[n] = rng.uniform(0.5, 1.5, size=s)
        else:
            out[n] = 0.1 * rng.randn(*s)
        out[n] = out[n].astype(dtype)
    return out


def _bn_relu(x, p, scope):
    y = (x - p[scope + "/moving_mean"]) / np.sqrt(p[scope + "/moving_variance"] + x.dtype.type(BN_EPS)) + p[scope + "/beta"]
    return np.maximum(y, 0)


def _conv2d(x, w, stride):
    """NHWC cross-correlation, SAME padding, HWIO weights."""
    n, h, wd, cin = x.shape
    kh, kw, _, cout = w.shape
    oh, pt, pb = same_pad(h, kh, stride[0])
    ow, pl, pr = same_pad(wd, kw, stride[1])
    xp = np.pad(x, [[0, 0], [pt, pb], [pl, pr], [0, 0]])
    out = np.zeros((n, oh, ow, cout), x.dtype)
    for i in range(kh):
        for j in range(kw):
            patch = xp[:, i:i + stride[0] * oh:stride[0], j:j + stride[1] * ow:stride[1], :]
            out += patch @ w[i, j]
    return out


def _depthwise(x, w, stride):
    n, h, wd, c = x.shape
    kh, kw = w.shape[:2]
    oh, pt, pb = same_pad(h, kh, stride[0])
    ow, pl, pr = same_pad(wd, kw, stride[1])
    xp = np.pad(x, [[0, 0], [pt, pb], [pl, pr], [0, 0]])
    out = np.zeros((n, oh, ow, c), x.dtype)
    for i in range(kh):
        for j in range(kw):
            out += xp[:, i:i + stride[0] * oh:stride[0], j:j + stride[1] * ow:stride[1], :] * w[i, j, :, 0]
    return out


def layer(spec: DsSpec, p, l, x):
    """Layer l of the net (conv + BN + ReLU, or depthwise + BN + ReLU + pointwise + BN + ReLU): x [N, H, W, Cin] NHWC
    (layer 0 also takes the features [N, H, W]) -> [N, Hout, Wout, Cout]."""
    typ, _, _, stride, scope = NET_DEFS[spec.size][l]
    s = f"DSCNN/{scope}"
    if x.ndim == 3:
        x = x[..., None]
    if typ == "conv":
        x = _conv2d(x, p[s + "/weights"], stride) + p[s + "/biases"]
        return _bn_relu(x, p, s + "/batch_norm")
    x = _depthwise(x, p[s + "/depthwise_conv/depthwise_weights"], stride) + p[s + "/depthwise_conv/biases"]
    x = _bn_relu(x, p, s + "/dw_batch_norm")
    x = _conv2d(x, p[s + "/pointwise_conv/weights"], (1, 1)) + p[s + "/pointwise_conv/biases"]
    return _bn_relu(x, p, s + "/pw_batch_norm")


def forward_layers(spec: DsSpec, p, feat):
    """feat [N, H, W] -> [output of layer 0, ..., output of the last layer], each NHWC."""
    acts, x = [], feat
    for l in range(len(NET_DEFS[spec.size])):
        x = layer(spec, p, l, x)
        acts.append(x)
    return acts


def head(spec: DsSpec, p, x):
    """Global average pool + fully connected: [N, H, W, C] -> logits [N, classes]."""
    return x.mean(axis=(1, 2)) @ p["DSCNN/fc1/weights"] + p["DSCNN/fc1/biases"]


def forward(spec: DsSpec, p, feat):
    """feat [N, H, W] -> logits [N, classes] (DSCNN(), ds_cnn.py:89-101, is_training=False)."""
    return head(spec, p, forward_layers(spec, p, feat)[-1])


def forward_flops(spec: DsSpec) -> int:
    h, w, cin, f = spec.h, spec.w, 1, 0
    for typ, depth, k, stride, _ in NET_DEFS[spec.size]:
        h, w = same_pad(h, k[0], stride[0])[0], same_pad(w, k[1], stride[1])[0]
        if typ == "conv":
            f += 2 * h * w * k[0] * k[1] * cin * depth
        else:
            f += 2 * h * w * k[0] * k[1] * cin + 2 * h * w * cin * depth
        cin = depth
    return f + 2 * cin * spec.num_classes


def flatten(spec, p, dtype=np.float32):
    return np.concatenate([np.asarray(p[n], dtype).ravel() for n in spec.var_names])
