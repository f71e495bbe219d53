"""bench.py's reference arm runs on a CPU box: exactly ONE JSON line on stdout with the keys the driver parses."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_json_line_with_the_contract_keys():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "2", "--warmup", "1", "--batch", "64"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, r.stdout[-1000:]
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["steps"] == 2 and d["warmup"] == 1 and d["higher_is_better"] is True
    assert d["unit"] == "utterances/sec" and d["value"] > 0 and d["vs_baseline"] is None
    assert "workload" in d["config"] and "model" not in d["config"]
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and "sample" in cb
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


def test_our_arm_fails_loudly_without_a_gpu():
    """No CPU fallback: on a box without CUDA the product arm must raise, not print a number."""
    import torch
    if torch.cuda.is_available():
        return
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "1"], capture_output=True, text=True,
                       timeout=600, cwd=ROOT)
    assert r.returncode != 0 and not [l for l in r.stdout.splitlines() if l.startswith("{")]


def test_every_kernel_the_step_can_launch_has_a_work_model():
    """bench.py:kernel_work feeds `kernels[*].GBps / TFLOPs` and the roofline block: every name a training step can launch
    (TCR_LAUNCH / res_launch names in csrc) must have its own bytes / flops, not fall through to the parameter-sized default
    (that is what `resident_bwd_data` did for a while: 53 GB/s reported for a 199 GB/s kernel)."""
    import importlib.util
    import re
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    sys.path.insert(0, ROOT)
    import tcresnet_b200  # noqa: F401
    from tcresnet_b200.plan import build_plan
    plan = build_plan("TCResNet8", 1.0, window_size_ms=40, window_stride_ms=20)
    src = ""
    for f in ("tcr_api.cu", "tcr_net_fwd.cu", "tcr_net_bwd.cu", "tcr_optim.cu", "tcr_resident.cu", "tcr_mfcc.cu"):
        src += open(os.path.join(ROOT, "tc-resnet_b200", "csrc", f)).read()
    names = set(re.findall(r'TCR_LAUNCH(?:_CLUSTER|_COOP)?\("([a-z_0-9]+)"', src)) | set(re.findall(r'res_launch\(h, "([a-z_0-9]+)"', src))
    small = {"grad_finalize", "update", "records_sum", "loss_only", "bn_table_eval"}          # parameter- or record-sized by nature
    default = bench.kernel_work(plan, "update", 512)
    heavy = sorted(n for n in names if n not in small)
    assert {"mfcc", "resident_fwd", "resident_bwd_data", "dw_grouped"} <= set(heavy), heavy
    for n in heavy:
        b, f = bench.kernel_work(plan, n, 512)
        assert (b, f) != default and b > 0, n
    c = plan.convs()[3]
    for kind in ("fwd", "dx"):
        b, f = bench.kernel_work(plan, f"{kind}:{c.name}", 512)
        assert b > 0 and f > 0
