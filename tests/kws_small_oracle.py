"""CPU oracle for KWSModel's speech_commands nets (TEST INFRASTRUCTURE ONLY): low_latency_conv and tiny_conv.

NumPy restatement in float64 of audio_nets/kws.py create_low_latency_conv_model and create_tiny_conv_model in evaluation mode
(the training dropouts are the identity), with the interface of oracle/kws_oracle.py (build_spec, layer, head, forward,
forward_flops, CODES):
  low_latency_conv  T x 8 conv 1 -> 186, VALID, stride 1, + bias, ReLU, flatten, fc 128 + bias, fc 128 + bias, fc classes + bias;
  tiny_conv         10 x 8 conv 1 -> 8, TF SAME at stride 2 x 2, + bias, ReLU, flatten, fc classes + bias.
TF SAME pads pad_total = max((out - 1) * stride + k - in, 0) zeros, the smaller half before.  The input [N, T, F] is read as NHWC
[N, T, F, 1] and flattened in NHWC order.  Pinned by a torch.nn.functional cross-check (explicit F.pad) in tests/test_kws_small.py.
"""
from __future__ import annotations

import numpy as np

from oracle.kws_oracle import KwsSpec, _conv_valid, flatten, l2_loss  # noqa: F401  (flatten, l2_loss: the same for these nets)

# size code of tcr_dscnn_config (include/tcr_b200.h) per --architecture
CODES = {"low_latency_conv": "C", "tiny_conv": "Y"}


def same_pad(n, k, s):
    """TF SAME along one axis: (output length, zeros before, zeros after)."""
    out = -(-n // s)
    total = max((out - 1) * s + k - n, 0)
    return out, total // 2, total - total // 2


def conv_geometry(arch, h, w):
    """Output shape (H, W, C) of the conv layer, as a one-element list."""
    if arch == "low_latency_conv":
        return [(1, w - 7, 186)]
    return [(same_pad(h, 10, 2)[0], same_pad(w, 8, 2)[0], 8)]


def build_spec(arch="low_latency_conv", h=49, w=40, num_classes=12) -> KwsSpec:
    """convs: (weight, bias, stride) of the conv; mats: (weight, bias) of each dense layer, in order."""
    k = int(np.prod(conv_geometry(arch, h, w)[0]))
    if arch == "low_latency_conv":
        shapes = [("first_weights", (h, 8, 1, 186)), ("first_bias", (186,)), ("first_fc_weights", (k, 128)), ("first_fc_bias", (128,)),
                  ("second_fc_weights", (128, 128)), ("second_fc_bias", (128,)), ("final_fc_weights", (128, num_classes)),
                  ("final_fc_bias", (num_classes,))]
        convs = [("first_weights", "first_bias", (1, 1))]
        mats = [("first_fc_weights", "first_fc_bias"), ("second_fc_weights", "second_fc_bias"), ("final_fc_weights", "final_fc_bias")]
    elif arch == "tiny_conv":
        shapes = [("first_weights", (10, 8, 1, 8)), ("first_bias", (8,)), ("final_fc_weights", (k, num_classes)),
                  ("final_fc_bias", (num_classes,))]
        convs = [("first_weights", "first_bias", (2, 2))]
        mats = [("final_fc_weights", "final_fc_bias")]
    else:
        raise ValueError(arch)
    return KwsSpec(arch, h, w, num_classes, [n for n, _ in shapes], dict(shapes), convs, mats)


def init_variables(spec: KwsSpec, seed=0, dtype=np.float64):
    """Seeded N(0, 2 / fan_in) weights, so that activations stay O(1) through the net, and N(0, 0.1^2) biases, so that every bias
    add is visible (the reference initialises them to zero)."""
    rng = np.random.RandomState(seed)
    out = {}
    for n in spec.var_names:
        s = spec.var_shapes[n]
        scale = 0.1 if len(s) == 1 else np.sqrt(2.0 / int(np.prod(s[:-1])))
        out[n] = (rng.randn(*s) * scale).astype(dtype)
    return out


def layer(spec: KwsSpec, p, l, x):
    """The conv layer (l = 0): x [N, T, F] or [N, T, F, 1] -> [N, Hout, Wout, Cout] after the bias and ReLU."""
    assert l == 0
    wname, bname, stride = spec.convs[0]
    if x.ndim == 3:
        x = x[..., None]
    if spec.arch == "tiny_conv":
        _, pt, pb = same_pad(x.shape[1], 10, 2)
        _, pl, pr = same_pad(x.shape[2], 8, 2)
        x = np.pad(x, ((0, 0), (pt, pb), (pl, pr), (0, 0)))
    return np.maximum(_conv_valid(x, p[wname], stride) + p[bname], 0)


def forward_layers(spec: KwsSpec, p, feat):
    return [layer(spec, p, 0, feat)]


def head(spec: KwsSpec, p, x):
    """flatten (NHWC order) and the dense layers, each + bias: [N, H, W, C] -> logits [N, classes]."""
    y = x.reshape(x.shape[0], -1)
    for w, b in spec.mats:
        y = y @ p[w] + p[b]
    return y


def forward(spec: KwsSpec, p, feat):
    """feat [N, T, F] -> logits [N, classes]."""
    return head(spec, p, forward_layers(spec, p, feat)[-1])


def forward_flops(spec: KwsSpec) -> int:
    """2 x multiply-adds of the conv (tiny_conv: the full 80-tap kernel at every output, padding included) and the matmuls; the
    bias adds are not counted."""
    oh, ow, cout = conv_geometry(spec.arch, spec.h, spec.w)[0]
    kh, kw = spec.var_shapes[spec.convs[0][0]][:2]
    return 2 * oh * ow * kh * kw * cout + sum(2 * int(np.prod(spec.var_shapes[w])) for w, _ in spec.mats)
