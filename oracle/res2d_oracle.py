"""CPU oracle for the 2-D ablations of TC-ResNet8 (TEST INFRASTRUCTURE ONLY): ResNet2D8 and ResNet2D8Pool.

NumPy restatement in float64 of audio_nets/tc_resnet.py's tc_resnet(..., debug_2d=True) as ResNet2D8 / ResNet2D8Pool build it, in
evaluation mode (dropout is the identity, BatchNorm uses the moving statistics):
  conv0 3x3 / stride 1 + BN + ReLU, for ResNet2D8Pool then avg_pool 4x4 / stride 4 VALID;
  block i (three): where the channel count changes, stride 2 and the shortcut down = 1x1 / stride 2 conv + BN + ReLU, else stride
  1 and the block's input; conv{i}_0 3x3 at that stride + BN + ReLU; conv{i}_1 3x3 + BN; add the shortcut; ReLU;
  global average pool; fc (1x1, no bias, no BN); softmax.  fc2 is a dead head and is not computed.
The input [N, T, F] is read as NHWC [N, T, F, 1].  Every conv is bias-free and TF SAME, written out here: per axis
out = ceil(in / s), pad = max((out - 1) * s + k - in, 0), pad_before = pad // 2.  BatchNorm: center and scale, eps 1e-3.
Pinned by a torch.nn.functional.conv2d cross-check with explicit asymmetric pads in tests/test_res2d.py.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Tuple

import numpy as np

# size code of tcr_dscnn_config (include/tcr_b200.h) per model scope
CODES = {"ResNet2D8": "R", "ResNet2D8Pool": "A"}
EPS = 1e-3


def channels(width: int, width_multiplier: float = 1.0) -> List[int]:
    """tc_resnet.py:74-81: int(x * wm) of [16, 24, 32, 48], then first_c replaces the first entry."""
    n = [int(x * width_multiplier) for x in [16, 24, 32, 48]]
    c1, c2 = n[0:2]
    n[0] = int((3 * width * c1 + 10 * c1 * c2) / (9 + 10 * c2))
    return n


def same(n: int, k: int, s: int) -> Tuple[int, int]:
    """TF SAME along one axis: (output length, leading pad)."""
    out = -(-n // s)
    return out, max((out - 1) * s + k - n, 0) // 2


@dataclass
class Res2dSpec:
    model: str
    h: int
    w: int
    num_classes: int
    ch: List[int]
    convs: List[Tuple[str, int, int, int]]     # (name under the scope, k, cin, cout) in creation order
    blocks: List[dict]                          # per block: stride, down (bool), conv names

    @property
    def var_names(self) -> List[str]:
        s = self.model + "/"
        rows = []
        for name, _, _, _ in self.convs:
            rows += [s + name + "/weights", s + name + "/BatchNorm/beta", s + name + "/BatchNorm/gamma"]
        rows += [s + "fc/weights", s + "fc2/weights"]
        for name, _, _, _ in self.convs:
            rows += [s + name + "/BatchNorm/moving_mean", s + name + "/BatchNorm/moving_variance"]
        return rows

    @property
    def var_shapes(self) -> Dict[str, tuple]:
        s, out = self.model + "/", {}
        for name, k, cin, cout in self.convs:
            out[s + name + "/weights"] = (k, k, cin, cout)
            for v in ("beta", "gamma", "moving_mean", "moving_variance"):
                out[s + name + "/BatchNorm/" + v] = (cout,)
        out[s + "fc/weights"] = (1, 1, self.ch[3], self.num_classes)
        out[s + "fc2/weights"] = (1, 1, self.ch[3], 2)
        return out


def build_spec(model="ResNet2D8", h=98, w=40, num_classes=12, width_multiplier=1.0) -> Res2dSpec:
    ch = channels(w, width_multiplier)
    convs, blocks, cin = [("conv0", 3, 1, ch[0])], [], ch[0]
    for i, n in enumerate(ch[1:]):
        b = {"down": n != cin, "stride": 2 if n != cin else 1, "conv0": f"block{i}/conv{i}_0", "conv1": f"block{i}/conv{i}_1"}
        if b["down"]:
            convs.append((f"block{i}/down", 1, cin, n))
        convs += [(b["conv0"], 3, cin, n), (b["conv1"], 3, n, n)]
        blocks.append(b)
        cin = n
    return Res2dSpec(model, h, w, num_classes, ch, convs, blocks)


def geometry(spec: Res2dSpec) -> List[Tuple[int, int, int]]:
    """Output shapes (H, W, C) of forward_partial's layers: conv0 (+ pool), block0, block1, block2."""
    h, w = spec.h, spec.w
    if spec.model == "ResNet2D8Pool":
        h, w = h // 4, w // 4
    out = [(h, w, spec.ch[0])]
    for i, b in enumerate(spec.blocks):
        h, w = same(h, 3, b["stride"])[0], same(w, 3, b["stride"])[0]
        out.append((h, w, spec.ch[i + 1]))
    return out


def forward_flops(spec: Res2dSpec) -> int:
    """2 x multiply-adds of every conv (conv0 at its pre-pool size) and fc; pools are not counted."""
    geo = geometry(spec)
    total = 2 * spec.h * spec.w * 9 * spec.ch[0]
    for i, b in enumerate(spec.blocks):
        ho, wo, n = geo[i + 1]
        cin = geo[i][2]
        total += 2 * ho * wo * (9 * cin * n + 9 * n * n + (cin * n if b["down"] else 0))
    return total + 2 * spec.ch[3] * spec.num_classes


def init_variables(spec: Res2dSpec, seed=0) -> Dict[str, np.ndarray]:
    """Seeded variables in float64: He-scaled weights, and BatchNorm statistics away from the identity (gamma, beta, mean and
    variance all vary per channel) so that a missing or misplaced term shows."""
    rng = np.random.RandomState(seed)
    p = {}
    for name, shape in spec.var_shapes.items():
        if name.endswith("/weights"):
            p[name] = rng.randn(*shape) * np.sqrt(2.0 / np.prod(shape[:-1]))
        elif name.endswith("gamma"):
            p[name] = rng.uniform(0.5, 1.5, shape)
        elif name.endswith("beta") or name.endswith("moving_mean"):
            p[name] = rng.uniform(-0.3, 0.3, shape)
        else:
            p[name] = rng.uniform(0.5, 2.0, shape)
    return p


def flatten(spec: Res2dSpec, p: Dict[str, np.ndarray]) -> np.ndarray:
    """The flat fp32 parameter buffer in tcr_dscnn_param_table's order."""
    return np.concatenate([np.asarray(p[n], np.float32).ravel() for n in spec.var_names])


def conv_same(x: np.ndarray, w: np.ndarray, s: int) -> np.ndarray:
    """TF SAME conv, NHWC x [N, H, W, C], HWIO w, stride s on both axes, with the asymmetric pads written out."""
    k = w.shape[0]
    (ho, pt), (wo, pl) = same(x.shape[1], k, s), same(x.shape[2], k, s)
    hp = max((ho - 1) * s + k - x.shape[1], 0)
    wp = max((wo - 1) * s + k - x.shape[2], 0)
    xp = np.pad(x, ((0, 0), (pt, hp - pt), (pl, wp - pl), (0, 0)))
    out = np.zeros((x.shape[0], ho, wo, w.shape[3]))
    for i in range(k):
        for j in range(k):
            out += xp[:, i:i + (ho - 1) * s + 1:s, j:j + (wo - 1) * s + 1:s, :] @ w[i, j]
    return out


def _bn(spec, p, name, x):
    s = spec.model + "/" + name + "/BatchNorm/"
    return (x - p[s + "moving_mean"]) / np.sqrt(p[s + "moving_variance"] + EPS) * p[s + "gamma"] + p[s + "beta"]


def _conv_bn(spec, p, name, x, s):
    return _bn(spec, p, name, conv_same(x, np.asarray(p[spec.model + "/" + name + "/weights"], np.float64), s))


def layer(spec: Res2dSpec, p, k: int, x: np.ndarray) -> np.ndarray:
    """forward_partial's layer k on its input x: k = 0 takes [N, T, F] features, k = 1..3 the previous layer's NHWC output."""
    if k == 0:
        y = np.maximum(_conv_bn(spec, p, "conv0", np.asarray(x, np.float64)[..., None], 1), 0)
        if spec.model == "ResNet2D8Pool":
            n, h, w, c = y.shape
            y = y[:, :h // 4 * 4, :w // 4 * 4].reshape(n, h // 4, 4, w // 4, 4, c).mean(axis=(2, 4))
        return y
    b = spec.blocks[k - 1]
    sc = np.maximum(_conv_bn(spec, p, f"block{k - 1}/down", x, 2), 0) if b["down"] else x
    y = np.maximum(_conv_bn(spec, p, b["conv0"], x, b["stride"]), 0)
    return np.maximum(_conv_bn(spec, p, b["conv1"], y, 1) + sc, 0)


def forward_layers(spec: Res2dSpec, p, feat: np.ndarray) -> List[np.ndarray]:
    x, out = np.asarray(feat, np.float64), []
    for k in range(4):
        x = layer(spec, p, k, x)
        out.append(x)
    return out


def head(spec: Res2dSpec, p, x: np.ndarray) -> np.ndarray:
    """Global average pool and fc (no bias): logits [N, classes]."""
    return x.mean(axis=(1, 2)) @ np.asarray(p[spec.model + "/fc/weights"], np.float64)[0, 0]


def forward(spec: Res2dSpec, p, feat: np.ndarray) -> np.ndarray:
    return head(spec, p, forward_layers(spec, p, feat)[-1])


def l2_loss(spec: Res2dSpec, p, weight_decay: float) -> float:
    """build_loss's regularisation: weight_decay * sum(tf.nn.l2_loss(v)) over every variable outside BatchNorm, fc2 included."""
    return weight_decay * sum(0.5 * float(np.sum(np.asarray(p[n], np.float64) ** 2)) for n in spec.var_names
                              if n.endswith("/weights"))
