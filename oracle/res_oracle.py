"""CPU oracle for Honk's ResNets as the reference builds them (TEST INFRASTRUCTURE ONLY): Res8, Res8Narrow, Res15, Res15Narrow.

NumPy restatement in float64 of audio_nets/res.py's resnet(...) under Res_arg_scope, in evaluation mode (BatchNorm uses the
moving statistics):
  f_conv 3x3 1 -> C + ReLU (no BatchNorm); Res8 / Res8Narrow then avg_pool 4x3 at stride 1, VALID;
  block i (num_layers // 2 of them) on input x: a = BN_{conv2i_bn}(ReLU(conv{2i}(x))); y = BN_{conv2i+1_bn}(ReLU(conv{2i+1}(a)) + x),
  no ReLU after the add; Res15 (13 layers) then conv12: BN_{conv12_bn}(ReLU(conv12(y)));
  global average pool; fc (1x1, no bias, no activation); softmax.
Every conv is 3x3, stride 1, TF SAME and bias-free; Res15 dilates conv{k} by rate 2 ** (k // 3), and SAME at stride 1 pads `rate`
zeros on every side (written out here).  BatchNorm has no beta and no gamma: (x - mean) / sqrt(var + 1e-3).  The input [N, T, F]
is read as NHWC [N, T, F, 1].  Pinned by torch.nn.functional.conv2d(..., dilation=d, padding=d) and avg_pool2d in tests/test_res.py.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Tuple

import numpy as np

# size code of tcr_dscnn_config (include/tcr_b200.h) per model
CODES = {"Res8": "E", "Res8Narrow": "N", "Res15": "D", "Res15Narrow": "T"}
MODELS = list(CODES)
EPS = 1e-3
SCOPE = "Res"


@dataclass
class ResSpec:
    model: str
    h: int
    w: int
    num_classes: int
    c: int            # channels
    layers: int       # convs after f_conv
    pool: bool        # Res8's 4x3 / stride-1 average pool after f_conv
    dilate: bool

    def rate(self, k: int) -> int:
        return 2 ** (k // 3) if self.dilate else 1

    @property
    def var_names(self) -> List[str]:
        s = SCOPE + "/"
        rows = [s + "f_conv/weights"] + [f"{s}conv{k}/Conv/weights" for k in range(self.layers)] + [s + "fc/weights"]
        for k in range(self.layers):
            rows += [f"{s}conv{k}_bn/moving_mean", f"{s}conv{k}_bn/moving_variance"]
        return rows

    @property
    def var_shapes(self) -> Dict[str, tuple]:
        s, c = SCOPE + "/", self.c
        out = {s + "f_conv/weights": (3, 3, 1, c), s + "fc/weights": (1, 1, c, self.num_classes)}
        for k in range(self.layers):
            out[f"{s}conv{k}/Conv/weights"] = (3, 3, c, c)
            out[f"{s}conv{k}_bn/moving_mean"] = (c,)
            out[f"{s}conv{k}_bn/moving_variance"] = (c,)
        return out


def build_spec(model="Res8", h=98, w=40, num_classes=12) -> ResSpec:
    r8 = model.startswith("Res8")
    return ResSpec(model, h, w, num_classes, 19 if model.endswith("Narrow") else 45, 6 if r8 else 13, r8, not r8)


def block_map(spec: ResSpec) -> Tuple[int, int]:
    """(H, W) the convs after f_conv run on."""
    return (spec.h - 3, spec.w - 2) if spec.pool else (spec.h, spec.w)


def geometry(spec: ResSpec) -> List[Tuple[int, int, int]]:
    """Output shapes (H, W, C) of forward_partial's layers: f_conv (+ pool), conv0 .. conv{L-1}."""
    h, w = block_map(spec)
    return [(h, w, spec.c)] * (spec.layers + 1)


def forward_flops(spec: ResSpec) -> int:
    """2 x multiply-adds of every conv (f_conv at its pre-pool size) and fc; pools are not counted."""
    h, w = block_map(spec)
    return 2 * spec.h * spec.w * 9 * spec.c + spec.layers * 2 * h * w * 9 * spec.c * spec.c + 2 * spec.c * spec.num_classes


def init_variables(spec: ResSpec, seed=0) -> Dict[str, np.ndarray]:
    """Seeded variables in float64: He-scaled weights and moving statistics away from the identity (mean and variance vary per
    channel), so that a missing or misplaced term shows."""
    rng = np.random.RandomState(seed)
    p = {}
    for name, shape in spec.var_shapes.items():
        if name.endswith("/weights"):
            p[name] = rng.randn(*shape) * np.sqrt(2.0 / np.prod(shape[:-1]))
        elif name.endswith("moving_mean"):
            p[name] = rng.uniform(-0.3, 0.3, shape)
        else:
            p[name] = rng.uniform(0.5, 2.0, shape)
    return p


def flatten(spec: ResSpec, p: Dict[str, np.ndarray]) -> np.ndarray:
    """The flat fp32 parameter buffer in tcr_dscnn_param_table's order."""
    return np.concatenate([np.asarray(p[n], np.float32).ravel() for n in spec.var_names])


def conv_same(x: np.ndarray, w: np.ndarray, rate: int = 1) -> np.ndarray:
    """3x3 TF SAME conv at stride 1 and dilation `rate`, NHWC x [N, H, W, C], HWIO w: `rate` zeros on every side."""
    n, h, wd, _ = x.shape
    xp = np.pad(x, ((0, 0), (rate, rate), (rate, rate), (0, 0)))
    out = np.zeros((n, h, wd, w.shape[3]))
    for i in range(3):
        for j in range(3):
            out += xp[:, i * rate:i * rate + h, j * rate:j * rate + wd, :] @ w[i, j]
    return out


def avg_pool_4x3(x: np.ndarray) -> np.ndarray:
    """avg_pool2d([4, 3], stride=1), VALID, NHWC."""
    n, h, w, c = x.shape
    out = np.zeros((n, h - 3, w - 2, c))
    for i in range(4):
        for j in range(3):
            out += x[:, i:i + h - 3, j:j + w - 2]
    return out / 12.0


def _bn(p, k, x):
    s = f"{SCOPE}/conv{k}_bn/"
    return (x - p[s + "moving_mean"]) / np.sqrt(p[s + "moving_variance"] + EPS)


def _conv(spec, p, k, x):
    return np.maximum(conv_same(x, np.asarray(p[f"{SCOPE}/conv{k}/Conv/weights"], np.float64), spec.rate(k)), 0)


def layer(spec: ResSpec, p, l: int, x: np.ndarray, block_in: np.ndarray = None) -> np.ndarray:
    """forward_partial's layer l on its input x: l = 0 is f_conv (+ pool) of [N, T, F] features; l = k + 1 is conv{k} of the previous
    layer's NHWC output, and for odd k (the second conv of a block) block_in is the block's input, layer l - 2's output."""
    if l == 0:
        y = np.maximum(conv_same(np.asarray(x, np.float64)[..., None], np.asarray(p[SCOPE + "/f_conv/weights"], np.float64)), 0)
        return avg_pool_4x3(y) if spec.pool else y
    k = l - 1
    y = _conv(spec, p, k, x)
    if k % 2:
        y = y + block_in
    return _bn(p, k, y)


def forward_layers(spec: ResSpec, p, feat: np.ndarray) -> List[np.ndarray]:
    out = []
    x = np.asarray(feat, np.float64)
    for l in range(spec.layers + 1):
        x = layer(spec, p, l, x, out[l - 2] if l >= 2 else None)
        out.append(x)
    return out


def head(spec: ResSpec, p, x: np.ndarray) -> np.ndarray:
    """Global average pool and fc (no bias): logits [N, classes]."""
    return x.mean(axis=(1, 2)) @ np.asarray(p[SCOPE + "/fc/weights"], np.float64)[0, 0]


def forward(spec: ResSpec, p, feat: np.ndarray) -> np.ndarray:
    return head(spec, p, forward_layers(spec, p, feat)[-1])


def l2_loss(spec: ResSpec, p, weight_decay: float) -> float:
    """build_loss's regularisation: weight_decay * sum(tf.nn.l2_loss(v)) over the trainable variables, here every weight."""
    return weight_decay * sum(0.5 * float(np.sum(np.asarray(p[n], np.float64) ** 2)) for n in spec.var_names
                              if n.endswith("/weights"))
