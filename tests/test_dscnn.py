"""DS-CNN forward (BASELINE.json config 5): oracle self-check against torch, emulated kernels on CPU, CUDA path on GPU."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dscnn_oracle as D
from tcr_harness import rel_err
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

    t, cin = torch.tensor(x)[:, None], 1
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
    ref = t.mean(dim=(2, 3)) @ torch.tensor(p["DSCNN/fc1/weights"]) + torch.tensor(p["DSCNN/fc1/biases"])
    np.testing.assert_allclose(D.forward(spec, p, x), ref.numpy(), rtol=1e-10, atol=1e-12)


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
    """TCR_DSCNN_TC picks the kernels when the net is created: 0 = register-tiled fp32 FMA, 1 = the lock-step wgmma kernels,
    default = the warp-specialised wgmma kernels (TMA input tiles).  Every path meets the same bound."""
    from tcr_harness import TorchBackend
    monkeypatch.setenv("TCR_DSCNN_TC", mode)
    assert _run(TorchBackend(), "S", 49, 40, 150) < 1e-5
    assert _run(TorchBackend(), "S", 49, 10, 39) < 1e-5
