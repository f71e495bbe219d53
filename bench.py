#!/usr/bin/env python
"""bench.py — utterances/sec of the TC-ResNet training step (MFCC front-end + fwd + bwd + SGD-momentum).

  python bench.py --gpus N --steps K --warmup W                 # our sm_90a CUDA path (one rank per GPU under torchrun)
  python bench.py --impl reference --gpus N --steps K --warmup W   # the reference's CPU path restated (oracle port)

Prints ONE JSON line (rank 0).  A "step" = one pass of the hot path over one batch of synthetic 16 kHz 1 s
clips U(-1,1) (BASELINE.json configs[1]: TCResNet8-1.0, batch 512 per GPU, MFCC 49x40, 12 classes).
`value` is device-timed with the batches already resident in HBM; `e2e` goes through the public Engine API
from pinned HOST buffers with the H2D copy and the D2H loss read inside the timed region.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = "utterances/sec (fwd+bwd+update) TCResNet8-1.0"     # BASELINE.json's metric; other models are named in config.workload
SMI_QUERY = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
             "clocks_event_reasons.sw_power_cap")


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--model", default="TCResNet8", choices=["TCResNet8", "TCResNet14"])
    ap.add_argument("--width", type=float, default=1.0)
    ap.add_argument("--batch", type=int, default=512, help="utterances per GPU per step")
    ap.add_argument("--window-ms", type=float, default=40.0)
    ap.add_argument("--stride-ms", type=float, default=20.0)
    ap.add_argument("--rotate", type=int, default=8, help="distinct resident input batches (footprint > L2)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-extra", action="store_true", help="skip the short runs of BASELINE.json configs 3 and 5 carried in `extra`")
    ap.add_argument("--cpu-seconds", type=float, default=12.0, help="budget of the bounded CPU-baseline sample")
    ap.add_argument("--frontend", default="auto", choices=["auto", "ordered", "ahead"],
                    help="ordered: the front-end is ordered on the step's stream; ahead (= auto): the timed inputs are resident and final, so "
                         "the call sets tcr_step_args::input_resident and the next step's front-end runs on the library's own stream behind "
                         "the previous step's weight-gradient launch, i.e. next to grad_finalize / update and the cross-GPU arrival wait "
                         "(measured: 0.348 -> 0.339 ms/step on 1 GPU, 0.359 -> 0.344 on 2)")
    ap.add_argument("--workload", default="train", choices=["train", "dscnn", "infer", "augment"],
                    help="train: the headline training step; dscnn: DS-CNN-S forward (BASELINE.json config 5, comparison point); "
                         "infer: evaluation-mode forward from wav (config 1 with --batch 1: latency); "
                         "augment: the device input stage (SURVEY.md 8f row 1), an HBM-bound elementwise pass")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the timed path computed in its last step (the arrays its caller receives) "
                         "as DIR/<name>.npy in float32; the inputs are seeded, so two builds can be compared output for output")
    return ap.parse_args()


DUMP_MAX_ELEMS = 4 << 20        # per array: at most 16 MB of float32 (a fixed, seeded sample of a larger output)


def dump_outputs(a, arrays):
    """--dump-outputs DIR: DIR/<name>.npy (float32) for every array; an array of more than DUMP_MAX_ELEMS elements is replaced by
    the elements at a fixed, seeded set of flat indices (the same on every run), so the files stay under 64 MB in all."""
    if not a.dump_outputs:
        return
    import numpy as np
    os.makedirs(a.dump_outputs, exist_ok=True)
    for name, t in arrays.items():
        x = t.detach().float().cpu().numpy().ravel() if hasattr(t, "detach") else np.asarray(t, np.float32).ravel()
        if x.size > DUMP_MAX_ELEMS:
            x = x[np.sort(np.random.default_rng(0).choice(x.size, DUMP_MAX_ELEMS, replace=False))]
        np.save(os.path.join(a.dump_outputs, name + ".npy"), x.astype(np.float32))


def l2_policy(a, clip=16000):
    rot = max(1, a.rotate)
    return f"inputs rotate over {rot} distinct batches ({rot * a.batch * clip * 4 / 1e6:.0f} MB; the H100's L2 is 50 MB)"


def make_config(a, world, exchange):
    """The SAME keys in both arms (the driver compares them)."""
    return {"workload": workload_name(a), "global_batch": a.batch * world, "l2": l2_policy(a), "exchange": exchange}


def pin_to_gpu_numa_node(dev_index):
    """Run this process on the CPU cores of the GPU's NUMA node (pinned-buffer copies and launches then stay local)."""
    try:
        import torch
        p = torch.cuda.get_device_properties(dev_index)
        bdf = f"{p.pci_domain_id:04x}:{p.pci_bus_id:02x}:{p.pci_device_id:02x}.0"
        node = int(open(f"/sys/bus/pci/devices/{bdf}/numa_node").read())
        if node < 0:
            return None
        cpus = set()
        for part in open(f"/sys/devices/system/node/node{node}/cpulist").read().strip().split(","):
            lo, _, hi = part.partition("-")
            cpus.update(range(int(lo), int(hi or lo) + 1))
        cpus &= os.sched_getaffinity(0)
        if cpus:
            os.sched_setaffinity(0, cpus)
            return {"node": node, "cpus": len(cpus)}
    except Exception:
        return None
    return None


def workload_name(a):
    t = 1 + (16000 - int(16 * a.window_ms)) // int(16 * a.stride_ms)
    return (f"{a.model}-{a.width:g} train step (MFCC {t}x40 front-end + fwd + bwd + SGD-momentum), synthetic 16 kHz 1 s clips, "
            f"batch {a.batch}/GPU, 12 classes")


# ------------------------------------------------------------------------------------------------
# clocks: nvidia-smi queried every 100 ms during the timed steps
# ------------------------------------------------------------------------------------------------
class ClockSampler:
    def __init__(self, index: int):
        self.proc, self.path = None, f"/tmp/tcr_clocks_{os.getpid()}.csv"
        try:
            self.f = open(self.path, "w")
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={SMI_QUERY}", "--format=csv,noheader,nounits",
                                          "-lms", "100", "-i", str(index)], stdout=self.f, stderr=subprocess.DEVNULL)
        except Exception:
            self.proc = None

    def stop(self):
        if self.proc is None:
            return None
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        self.f.close()
        sm, smax, power, reasons = [], [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for line in open(self.path):
            parts = [p.strip() for p in line.split(",")]
            if len(parts) < 9:
                continue
            try:
                sm.append(float(parts[1])); smax.append(float(parts[2])); power.append(float(parts[3]))
            except ValueError:
                continue
            for name, val in zip(names, parts[5:9]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        if not sm:
            return None
        return {"sm_mhz": statistics.median(sm), "sm_max_mhz": max(smax), "power_w_max": max(power),
                "samples": len(sm), "reasons": sorted(reasons)}


# ------------------------------------------------------------------------------------------------
# CPU arm: the reference's CPU path restated (oracle port, PyTorch-CPU fp32, all host threads)
# ------------------------------------------------------------------------------------------------
_CPU_THREADS = None


def cpu_port_step_fn(a, batch, threads=None):
    import numpy as np
    import torch
    from oracle import tcr_oracle as O
    from oracle.torch_port import TorchPort
    torch.set_num_threads(threads or _CPU_THREADS or os.cpu_count() or 1)
    window, stride = int(16 * a.window_ms), int(16 * a.stride_ms)
    spec = O.build_spec(a.model, a.width, O.num_frames(16000, window, stride))
    params, moving = O.init_variables(spec, 0, np.float32)
    port = TorchPort(spec, params, moving, window, stride, keep_prob=0.5)
    wav_np, onehot_np = O.synthetic_batch(batch, seed_wav=1234)
    wav, onehot = torch.from_numpy(wav_np), torch.from_numpy(onehot_np)

    def step():
        port.train_step(wav, onehot, 0.1, 0.9, 1e-3)
    return step, torch.get_num_threads()


def calibrate_cpu_threads(a):
    """The tensors of this path are tiny: on a many-core host, intra-op parallelism over all cores can be SLOWER than over 16.
    Give the CPU arm its best thread count: time one step of 128 utterances at each candidate and keep the fastest."""
    global _CPU_THREADS
    if _CPU_THREADS is not None:
        return _CPU_THREADS
    cores = os.cpu_count() or 1
    best = (float("inf"), cores)
    for t in sorted({c for c in (4, 8, 16, 32, 64, cores) if c <= cores}):
        step, _ = cpu_port_step_fn(a, 128, threads=t)
        step()
        t0 = time.perf_counter(); step(); dt = time.perf_counter() - t0
        best = min(best, (dt, t))
        if dt > 1.3 * best[0]:                # past the optimum: more threads only get slower (and the probes much longer)
            break
    _CPU_THREADS = best[1]
    return _CPU_THREADS


def run_cpu_sample(a, seconds):
    """Bounded sample of the same workload on the host cores: returns the cpu_baseline object."""
    batch = a.batch
    calibrate_cpu_threads(a)
    step, cores = cpu_port_step_fn(a, batch)
    step()
    t0 = time.perf_counter(); step(); dt = time.perf_counter() - t0
    while dt > seconds / 3 and batch > 32:          # keep >= 3 timed steps inside the budget
        batch //= 2
        step, cores = cpu_port_step_fn(a, batch)
        step()
        t0 = time.perf_counter(); step(); dt = time.perf_counter() - t0
    nsteps = max(3, min(50, int(seconds / max(dt, 1e-6))))
    t0 = time.perf_counter()
    for _ in range(nsteps):
        step()
    dt = (time.perf_counter() - t0) / nsteps
    return {"value": batch / dt, "unit": "utterances/sec", "cores": cores, "kind": "port",
            "sample": f"{nsteps} training steps of batch {batch} (same model/shape), PyTorch-CPU fp32 restatement of the "
                      f"reference's TF-1.13 graph (TF 1.13.1 not installable here), {dt * 1e3:.1f} ms/step, {cores} threads (the fastest of "
                      f"4..{os.cpu_count()} on this host)"}


def run_reference(a):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    batch = a.batch
    calibrate_cpu_threads(a)
    step, cores = cpu_port_step_fn(a, batch)
    step()
    t0 = time.perf_counter(); step(); dt = time.perf_counter() - t0
    budget = 150.0
    while dt * (a.steps + a.warmup) > budget and batch > 16:
        batch //= 2
        step, cores = cpu_port_step_fn(a, batch)
        step()
        t0 = time.perf_counter(); step(); dt = time.perf_counter() - t0
    for _ in range(a.warmup):
        step()
    t0 = time.perf_counter()
    for _ in range(a.steps):
        step()
    el = time.perf_counter() - t0
    value = batch * a.steps / el
    sample = (f"each step = one training step on a bounded sample of {batch} of the {a.batch} utterances, PyTorch-CPU fp32 "
              f"restatement of the reference graph (TF 1.13.1 not installable), {cores} threads (the fastest of 4..{os.cpu_count()} on this host)")
    out = {"impl": "reference", "metric": METRIC, "value": value, "unit": "utterances/sec", "n_gpus": a.gpus, "steps": a.steps,
           "warmup": a.warmup, "ms_per_step": el / a.steps * 1e3, "higher_is_better": True, "scaling": "weak",
           "vs_baseline": None, "dtype": "f32", "data": "synthetic",
           "config": make_config(a, a.gpus, "none (1 GPU)" if a.gpus == 1 else "peer-memory | nccl (GPU arm)"),
           "sample_batch": batch,
           "cpu_baseline": {"value": value, "unit": "utterances/sec", "cores": cores, "kind": "port", "sample": sample},
           "e2e": {"value": value, "unit": "utterances/sec", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    emit(out)


# ------------------------------------------------------------------------------------------------
# our arm
# ------------------------------------------------------------------------------------------------
def kernel_work(plan, name, n):
    """(algorithmic bytes, flops) of ONE launch of kernel `name` over n utterances (DESIGN.md section 5)."""
    convs = {c.name: c for c in plan.convs()}
    if name == "mfcc":
        return n * (4 * plan.clip + 4 * plan.frames * plan.features), n * plan.frontend_flops()
    kind, _, layer = name.partition(":")
    if layer in convs:
        c = convs[layer]
        down = next((b.down for b in plan.blocks if b.conv_a.name == layer and b.down is not None), None)
        macs = c.macs + (down.macs if (down and kind in ("fwd", "dx")) else 0)
        act_in, act_out = 4 * c.t_in * c.cin, 4 * c.t_out * c.cout
        if kind == "fwd":
            bytes_ = n * (act_in + act_out + (4 * down.t_out * down.cout if down else 0)) + 4 * c.weights
        elif kind == "dx":    # reads dz + y of this layer (+ down), y/out of the layer below, writes dz below
            bytes_ = n * (2 * act_out + (8 * down.t_out * down.cout if down else 0) + 3 * act_in) + 4 * c.weights
        else:                 # dw: reads x, dz, y; writes partials (counted once)
            bytes_ = n * (act_in + 2 * act_out) + 4 * c.weights
        return bytes_, 2.0 * n * macs
    if name == "head":
        return n * (3 * 4 * plan.t_last * plan.c_last), 2.0 * n * plan.c_last * plan.num_classes * 2
    if name == "dw_grouped":          # every layer's weight gradient in one launch: reads x, dz, y of each layer once
        b = sum(n * (4 * c.t_in * c.cin + 8 * c.t_out * c.cout) + 4 * c.weights for c in plan.convs())
        return b, 2.0 * n * sum(c.macs for c in plan.convs())
    if name == "weight_transpose":
        w = sum(c.weights for c in plan.convs())
        return 8.0 * w, 0.0
    fwd_flops = 2.0 * n * sum(c.macs for c in plan.convs())
    if name == "resident_fwd":        # all forward convs + head in one cooperative launch: reads the features, writes every pre-BN output
        b = n * (4 * plan.frames * plan.features + sum(4 * c.t_out * c.cout for c in plan.convs())) + 4 * sum(c.weights for c in plan.convs())
        return b, fwd_flops
    if name == "resident_bwd_data":   # the backward-data chain alone: reads every layer's pre-BN output, writes every layer's gradient
        b = n * sum(8 * c.t_out * c.cout for c in plan.convs()) + 4 * sum(c.weights for c in plan.convs()[1:])
        return b, fwd_flops - 2.0 * n * plan.convs()[0].macs
    if name == "resident_bwd":        # backward-data chain + all weight gradients + gradient reduction
        b = n * (4 * plan.frames * plan.features + sum(4 * c.t_out * c.cout for c in plan.convs())) + 12 * sum(c.weights for c in plan.convs())
        return b, 2 * fwd_flops - 2.0 * n * plan.convs()[0].macs
    return 12.0 * plan.num_trainable, 4.0 * plan.num_trainable      # grad_finalize / update: params, slots, grads


def run_ours(a):
    import numpy as np
    import torch
    import tcresnet_b200  # noqa: F401
    from tcresnet_b200.engine import Engine
    from tcresnet_b200.plan import build_plan

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    local_dev = local
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    numa = pin_to_gpu_numa_node(local)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
    n = a.batch
    eng = Engine(model=a.model, width_multiplier=a.width, window_size_ms=a.window_ms, window_stride_ms=a.stride_ms,
                 max_batch=n, dropout_keep_prob=0.5, device=local)
    if world > 1:
        eng.attach_process_group()
    plan = build_plan(a.model, a.width, window_size_ms=a.window_ms, window_stride_ms=a.stride_ms)
    params, slots, moving = eng.new_variables(seed=0)
    gen = torch.Generator(device=dev).manual_seed(1234 + rank)
    rot = max(1, a.rotate)
    wavs = [torch.rand(n, plan.clip, device=dev, generator=gen) * 2 - 1 for _ in range(rot)]
    labels = torch.randint(0, 12, (rot, n), device=dev, generator=torch.Generator(device=dev).manual_seed(4321))
    onehots = [torch.nn.functional.one_hot(labels[i], 12).float().contiguous() for i in range(rot)]
    losses = torch.zeros(2, device=dev)
    lr, mom, wd = 0.1, 0.9, 1e-3

    frontend_ahead = a.frontend != "ordered"

    def step(i):
        eng.train_step(wavs[i % rot], onehots[i % rot], params, slots, moving, lr, mom, wd, dropout_seed=i * world + rank, losses=losses,
                       input_resident=frontend_ahead)

    def barrier():
        if world > 1:
            torch.distributed.barrier()
        torch.cuda.synchronize()

    for i in range(max(a.warmup, 3)):
        step(i)
    barrier()
    sampler = ClockSampler(local) if rank == 0 else None
    launches0 = eng.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    e0.record()
    for i in range(a.steps):
        step(i)
    e1.record()
    barrier()
    ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
    if world > 1:
        torch.distributed.all_reduce(ms, op=torch.distributed.ReduceOp.MAX)
    ms = float(ms.item())
    launches = eng.launch_count() - launches0
    clocks = sampler.stop() if sampler else None
    if rank == 0:
        dump_outputs(a, {"losses": losses, "params": params, "slots": slots, "moving": moving})
    final_loss = float(losses[0].item())
    value = n * world * a.steps / (ms * 1e-3)

    metric = METRIC if (a.model == "TCResNet8" and a.width == 1.0) else f"utterances/sec (fwd+bwd+update) {a.model}-{a.width}"
    out = {"metric": metric, "value": value, "unit": "utterances/sec", "n_gpus": world, "steps": a.steps, "warmup": max(a.warmup, 3),
           "ms_per_step": ms / a.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
           "data": "synthetic", "impl": "ours",
           "config": make_config(a, world, "none (1 GPU)" if world == 1 else getattr(eng, "exchange", "nccl")),
           "parallelism": f"dp{world}", "final_total_loss": final_loss, "numa": numa,
           "frontend": ("ordered on the step's stream" if not frontend_ahead else
                        "runs ahead on the library's stream (tcr_step_args::input_resident: the timed inputs are resident and final)"),
           "gpu_launches": int(launches), "clocks": clocks}

    # ---- data-parallel self-check, outside the timed region (the driver's GPU-test box has one GPU and skips tests/test_dist.py):
    # (1) replicas are still bit-identical after the timed steps; (2) on a 16-utterance shard per rank, the gradient the exchange
    # hands to the update (averaged over ranks, fused into the update kernel over peer memory or all-reduced by NCCL) equals the mean
    # of the ranks' LOCAL gradients, each computed by an unattached handle of the same library and gathered through torch.distributed.
    if world > 1:
        import torch.distributed as dist
        digest = torch.stack([params.double().sum(), params.double().abs().sum(), slots.double().sum(), slots.double().abs().sum()])
        gathered = [torch.zeros_like(digest) for _ in range(world)]
        dist.all_gather(gathered, digest)
        identical = all(bool(torch.equal(g, gathered[0])) for g in gathered)     # trainables + momentum slots (BN moving statistics
        m = 16                                                                    # are per-replica batch statistics: no SyncBN)
        p_chk = params.clone()
        # the unattached handle has the attached one's geometry (same max_batch -> same tilings and summation orders), so its local
        # gradient is bit-for-bit what the attached handle computes before the exchange
        local = Engine(model=a.model, width_multiplier=a.width, window_size_ms=a.window_ms, window_stride_ms=a.stride_ms, max_batch=n,
                       dropout_keep_prob=0.5, device=local_dev)
        sl, mv = torch.zeros_like(params), moving.clone()
        seed = 12345 * world + rank                                  # the same dropout draws in both handles
        g_local = local.train_step(wavs[0][:m], onehots[0][:m], p_chk, sl, mv, lr, mom, wd, dropout_seed=seed, want_grads=True, apply_update=False)["grads"]
        g_avg = eng.train_step(wavs[0][:m], onehots[0][:m], p_chk, sl, mv, lr, mom, wd, dropout_seed=seed, want_grads=True, apply_update=False)["grads"]
        parts = [torch.zeros_like(g_local) for _ in range(world)]
        dist.all_gather(parts, g_local)
        mean = torch.stack([q.double() for q in parts]).mean(0)
        err = float((g_avg.double() - mean).abs().max() / mean.abs().max().clamp_min(1e-30))
        out["dp_check"] = {"replicas_bit_identical": identical, "averaged_gradient_rel_err_vs_mean_of_local": err,
                           "shard": f"{m} utterances per rank", "exchange": getattr(eng, "exchange", "nccl"), "ok": bool(identical and err < 1e-5),
                           "note": "digest over trainables and momentum slots; BN moving statistics stay per-replica (no SyncBN, as in the "
                                   "single-GPU reference)"}
        local.close()
        barrier()

    # ---- end to end through the public API: pinned host -> H2D -> step -> D2H loss, every step ----
    if not a.no_e2e:
        from tcresnet_b200.engine import HostFeed
        h_wavs = [w.cpu().pin_memory() for w in wavs[:min(rot, 4)]]
        h_hots = [o.cpu().pin_memory() for o in onehots[:min(rot, 4)]]
        esteps = a.steps

        def e2e_run(host_wavs, host_clips=None, background=None):
            feed = HostFeed(eng, lag=2)
            seen = []

            def e2e_step(i):                              # returns (step, total, model) of the step submitted 2 calls earlier
                r = feed.submit(host_wavs[i % len(host_wavs)], h_hots[i % len(h_hots)], params, slots, moving, lr, mom, wd,
                                dropout_seed=i * world + rank, h_clips=host_clips[i % len(host_clips)] if host_clips else None,
                                background=background)
                if r is not None:
                    seen.append(r)

            # warm-up: >= 12 steps, then blocks of 40 until two consecutive blocks agree within 5 % (at most 8 blocks).  On a box whose
            # previous process has just exited, the first second of host-buffer steps can run at half rate (the copy engines are still
            # busy with the driver's housekeeping); a fixed 12-step warm-up then lands inside that phase on some runs and not on others.
            for i in range(12):
                e2e_step(i)
            feed.flush()
            prev_rate = None
            for blk in range(8):
                tb = time.perf_counter()
                for i in range(40):
                    e2e_step(i)
                feed.flush()
                rate = 40 / (time.perf_counter() - tb)
                if prev_rate is not None and abs(rate - prev_rate) <= 0.05 * prev_rate:
                    break
                prev_rate = rate
            barrier()
            del seen[:]
            t0 = time.perf_counter()
            for i in range(esteps):
                e2e_step(i)
            seen.extend(feed.flush())                     # every step's loss is on the host before the clock stops
            barrier()
            el = torch.tensor([time.perf_counter() - t0], device=dev)
            if world > 1:
                torch.distributed.all_reduce(el, op=torch.distributed.ReduceOp.MAX)
            assert len(seen) == esteps, (len(seen), esteps)
            return n * world * esteps / float(el.item()), seen[-1]

        all_runs = {}

        def median3(host_bufs, host_clips=None, background=None, tag="fp32"):   # PCIe / host interference on a shared box: median of 3
            runs = sorted((e2e_run(host_bufs, host_clips, background) for _ in range(3)), key=lambda r: r[0])
            all_runs[tag] = [r[0] for r in runs]
            return runs[1]

        e2e_value, last = median3(h_wavs)
        # the same clips as the wav files store them (int16 PCM); decode_wav's 1/32768 scaling runs on the device
        h_pcm = [(w.clamp(-1, 1) * 32767.0).round().to(torch.int16).cpu().pin_memory() for w in wavs[:min(rot, 4)]]
        pcm_value, _ = median3(h_pcm, tag="pcm16")
        # the same int16 clips with the per-clip input stage (shift, background mix, clip) on the device: the host ships the
        # samples and 24 bytes of random draws per clip, i.e. the reference's augmented TRAINING input at half the fp32 bytes
        from tcresnet_b200.datasets import device_input_stage as D
        rs = np.random.RandomState(99)
        stage = D.DeviceInputStage(eng, [rs.uniform(-0.5, 0.5, 960000).astype(np.float32) for _ in range(6)])
        h_clips = [torch.from_numpy(np.frombuffer(D.draw_clips(rs, [plan.clip] * n, rs.uniform(size=n) < 0.1, plan.clip,
                                                                stage.bg_lengths).tobytes(), np.uint8).copy()).pin_memory()
                   for _ in h_pcm]
        aug_value, _ = median3(h_pcm, h_clips, stage.background, tag="pcm16_device_input_stage")
        h2d = int(h_wavs[0].numel() * 4 + h_hots[0].numel() * 4)
        # serial H2D bandwidth of the same buffers, for context
        c0, c1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        c0.record()
        for i in range(10):
            wavs[0].copy_(h_wavs[i % len(h_wavs)], non_blocking=True)
        c1.record()
        torch.cuda.synchronize()
        out["e2e"] = {"value": e2e_value, "unit": "utterances/sec",
                      "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 8, "steps": esteps, "runs": "median of 3 runs of `steps` steps",
                      "all_runs": all_runs,
                      "bound": f"fp32 samples: {h2d / 1e6:.1f} MB per step over PCIe; at the serial rate measured below the copy alone allows "
                               f"{n * world / (h2d / (54.8e9)):.0f} utt/s per 54.8 GB/s link (the step itself: `value`)",
                      "h2d_GBps_measured": 10 * h_wavs[0].numel() * 4 / (c0.elapsed_time(c1) * 1e-3) / 1e9,
                      "last_total_loss": last[1] if last else None,
                      "pcm16": {"value": pcm_value, "unit": "utterances/sec", "h2d_bytes_per_step": int(h_pcm[0].numel() * 2 + h_hots[0].numel() * 4),
                                "note": "same pipeline fed int16 PCM (TCR_INPUT_WAV_PCM16): for un-augmented evaluation/inference batches"},
                      "pcm16_device_input_stage": {"value": aug_value, "unit": "utterances/sec",
                                                   "h2d_bytes_per_step": int(h_pcm[0].numel() * 2 + h_hots[0].numel() * 4 + 24 * n),
                                                   "note": "int16 clips + 24-byte draws per clip; decode, shift, background mix and clip run "
                                                           "on the device inside the step (tcr_augment.cu): the augmented training input"},
                      "api": "C ABI tcr_train_step_host (tcresnet_b200.engine.HostFeed.submit, lag 2): pinned host fp32 wav + one-hot -> H2D on "
                             "the library's copy stream every step, the step, both losses of every step read back to the host"}

    # ---- BASELINE.json configs 3 and 5, short device-timed runs carried inside the N = 1 line (so a driver-run record exists) ----
    if rank == 0 and world == 1 and not a.no_extra and a.model == "TCResNet8" and a.width == 1.0:
        out["extra"] = {}
        try:
            out["extra"]["TCResNet14-1.5_b1024_train"] = quick_train(torch, dev, "TCResNet14", 1.5, 1024, a.window_ms, a.stride_ms, 0.0)
        except Exception as e:
            out["extra"]["TCResNet14-1.5_b1024_train"] = {"error": str(e)[:200]}
        try:
            out["extra"]["DSCNN-S_b512_forward"] = quick_dscnn(torch, dev, 512)
        except Exception as e:
            out["extra"]["DSCNN-S_b512_forward"] = {"error": str(e)[:200]}
    # (The end-to-end section runs BEFORE the FMA-peak measurement and the per-kernel pass: the 18 ms all-SM FMA burn of
    # tcr_measure_fp32_peak is followed by about a second of reduced clocks on a warm GPU, which used to land on the first
    # end-to-end variants and made them bimodal: 0.50-0.85 M utt/s for the same code on the same box.)
    # ---- per-kernel durations (separate pass: event brackets add overhead, so not the timed region).  Every rank runs
    # the steps (they contain the gradient all-reduce); rank 0 reports.
    psteps = min(a.steps, 30)
    fp32_peak = eng.fp32_peak_tflops() if rank == 0 else 0.0
    barrier()
    eng.profile(True)
    for i in range(psteps):
        step(i)
    torch.cuda.synchronize()
    stats = eng.profile_read()
    eng.profile(False)
    barrier()
    if rank == 0:
        peaks = {}
        try:
            peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        except Exception:
            pass
        hbm_peak = float(peaks.get("hbm_gbs", 3350.0))
        peak_src = "measured (MEASURED_PEAKS.json)" if "hbm_gbs" in peaks else "fallback 3350 GB/s (H100 SXM data sheet)"
        total_ms = sum(v[0] for v in stats.values())
        top = sorted(stats.items(), key=lambda kv: -kv[1][0])
        kernels = []
        for name, (tms, cnt) in top:
            b, f = kernel_work(plan, name, n)
            dur = tms / cnt * 1e-3
            kernels.append({"name": name, "us": dur * 1e6, "share": tms / total_ms, "GBps": b / dur / 1e9, "TFLOPs": f / dur / 1e12})
        dom = kernels[0]
        alg_bytes, alg_flops = kernel_work(plan, dom["name"], n)
        # which pipe binds this kernel: the larger of its two floors (bytes / HBM peak, flops / fp32-FMA peak)
        t_hbm, t_fma = alg_bytes / (hbm_peak * 1e9), alg_flops / max(fp32_peak * 1e12, 1.0)
        hbm_form = {"achieved": dom["GBps"], "peak": hbm_peak, "unit": "GB/s", "frac": dom["GBps"] / hbm_peak, "peak_source": peak_src}
        fma_form = {"achieved": dom["TFLOPs"], "peak": fp32_peak, "unit": "TFLOP/s", "frac": dom["TFLOPs"] / max(fp32_peak, 1e-9),
                    "peak_source": "fp32 FMA pipe, measured in this run (tcr_measure_fp32_peak: FMA loop on all SMs); the convolutions run on "
                                   "the FMA pipe because single TF32 / BF16 products miss the 1e-4 logit bound (DESIGN.md)"}
        binding = fma_form if t_fma > t_hbm else hbm_form
        out["roofline"] = {"bound": "fp32-fma" if t_fma > t_hbm else "hbm", "kernel": dom["name"], "achieved": binding["achieved"],
                           "peak": binding["peak"], "unit": binding["unit"], "frac": binding["frac"], "traffic": None,
                           "algorithmic_bytes_per_launch": alg_bytes,
                           "algorithmic_flops_per_launch": alg_flops, "floors_us": {"hbm": t_hbm * 1e6, "fp32_fma": t_fma * 1e6},
                           "kernel_us": dom["us"], "kernel_share_of_step": dom["share"], "hbm": hbm_form, "fp32": fma_form,
                           "step": {"train_flops_per_utt": plan.train_flops(), "min_bytes_per_utt": plan.min_bytes(n),
                                    "fp32_frac": plan.train_flops() * (value / world) / 1e12 / max(fp32_peak, 1e-9),
                                    "hbm_frac": plan.min_bytes(n) * (value / world) / 1e9 / hbm_peak}}
        out["kernels"] = kernels[:12]

    if rank == 0 and "extra" in out and isinstance(out["extra"].get("TCResNet14-1.5_b1024_train"), dict) \
            and "train_flops_per_utt" in out["extra"]["TCResNet14-1.5_b1024_train"]:
        x = out["extra"]["TCResNet14-1.5_b1024_train"]
        x["fp32_frac"] = x["train_flops_per_utt"] * x["value"] / 1e12 / max(fp32_peak, 1e-9)
    if rank == 0:
        if world == 1 and not a.no_cpu_baseline:
            try:
                out["cpu_baseline"] = run_cpu_sample(a, a.cpu_seconds)
            except Exception as e:  # the oracle port must never take the bench line down
                out["cpu_baseline"] = {"value": None, "unit": "utterances/sec", "cores": os.cpu_count(), "kind": "port",
                                       "sample": f"failed: {e}"}
        emit(out)
    if world > 1:
        torch.distributed.destroy_process_group()


def quick_train(torch, dev, model, width, batch, window_ms, stride_ms, fp32_peak, steps=40, warmup=6, rot=4):
    """Short device-timed training-step run of another configuration (inputs rotate over `rot` resident batches)."""
    from tcresnet_b200.engine import Engine
    from tcresnet_b200.plan import build_plan
    eng = Engine(model=model, width_multiplier=width, window_size_ms=window_ms, window_stride_ms=stride_ms, max_batch=batch, dropout_keep_prob=0.5)
    plan = build_plan(model, width, window_size_ms=window_ms, window_stride_ms=stride_ms)
    params, slots, moving = eng.new_variables(seed=0)
    gen = torch.Generator(device=dev).manual_seed(99)
    wavs = [torch.rand(batch, plan.clip, device=dev, generator=gen) * 2 - 1 for _ in range(rot)]
    hots = [torch.nn.functional.one_hot(torch.randint(0, 12, (batch,), device=dev, generator=gen), 12).float().contiguous() for _ in range(rot)]
    losses = torch.zeros(2, device=dev)
    for i in range(warmup):
        eng.train_step(wavs[i % rot], hots[i % rot], params, slots, moving, 0.1, 0.9, 1e-3, dropout_seed=i, losses=losses)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        eng.train_step(wavs[i % rot], hots[i % rot], params, slots, moving, 0.1, 0.9, 1e-3, dropout_seed=i, losses=losses)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    value = batch / (ms * 1e-3)
    eng.close()
    return {"metric": f"utterances/sec (fwd+bwd+update) {model}-{width:g}", "value": value, "ms_per_step": ms, "batch": batch, "steps": steps,
            "warmup": warmup, "l2": f"inputs rotate over {rot} resident batches ({rot * batch * plan.clip * 4 / 1e6:.0f} MB; the H100's L2 is 50 MB)",
            "final_total_loss": float(losses[0].item()), "train_flops_per_utt": plan.train_flops(),
            "fp32_frac": plan.train_flops() * value / 1e12 / max(fp32_peak, 1e-9)}


def quick_dscnn(torch, dev, n, steps=40, warmup=6, rot=8):
    from tcresnet_b200.dscnn import DsCnn
    net = DsCnn("S", 49, 40, 12, max_batch=n)
    gen = torch.Generator(device=dev).manual_seed(7)
    params = torch.randn(net.num_params, device=dev, generator=gen) * 0.1
    for d in net.table:
        if d["name"].endswith("moving_variance"):
            params[d["offset"]:d["offset"] + d["numel"]] = 1.0
    feats = [torch.randn(n, 49, 40, device=dev, generator=gen) for _ in range(rot)]
    for i in range(warmup):
        net.forward(feats[i % rot], params)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        net.forward(feats[i % rot], params)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    return {"metric": "utterances/sec (forward) DS-CNN-S", "value": n / (ms * 1e-3), "ms_per_step": ms, "batch": n, "steps": steps,
            "forward_flops_per_utt": net.forward_flops, "tflops": n / (ms * 1e-3) * net.forward_flops / 1e12,
            "pointwise": "wgmma 3xTF32 (csrc/tcr_dscnn.cu)" if os.environ.get("TCR_DSCNN_TC", "1") != "0" else "fp32 FMA"}


def run_infer(a):
    """Config 1: evaluation-mode forward (moving-statistics BN, no dropout) from wav; with --batch 1 this is the latency case.
    Device-timed per call (CUDA events), and synchronously from the host (call -> logits on the host)."""
    import torch
    import tcresnet_b200  # noqa: F401
    from tcresnet_b200.engine import Engine
    dev = torch.device("cuda", 0)
    n = a.batch
    eng = Engine(model=a.model, width_multiplier=a.width, window_size_ms=a.window_ms, window_stride_ms=a.stride_ms, max_batch=n)
    params, _, moving = eng.new_variables(seed=0)
    gen = torch.Generator(device=dev).manual_seed(1234)
    wavs = [torch.rand(n, 16000, device=dev, generator=gen) * 2 - 1 for _ in range(a.rotate)]
    for i in range(max(a.warmup, 3)):
        eng.forward(wavs[i % a.rotate], params, moving)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(a.steps):
        res = eng.forward(wavs[i % a.rotate], params, moving)
    e1.record()
    torch.cuda.synchronize()
    dump_outputs(a, {"logits": res["logits"], "probs": res["probs"]})
    ms = e0.elapsed_time(e1) / a.steps
    h_wav = wavs[0].cpu().pin_memory()
    d_wav = torch.empty_like(wavs[0])
    t0 = time.perf_counter()
    for i in range(a.steps):
        d_wav.copy_(h_wav, non_blocking=True)
        logits = eng.forward(d_wav, params, moving)["logits"].cpu()          # synchronises: the caller holds the prediction
    host_ms = (time.perf_counter() - t0) / a.steps * 1e3
    emit({"metric": f"utterances/sec (evaluation forward from wav) {a.model}-{a.width:g}", "value": n / (ms * 1e-3), "unit": "utterances/sec",
          "n_gpus": 1, "steps": a.steps, "warmup": max(a.warmup, 3), "ms_per_step": ms, "higher_is_better": True, "scaling": "weak",
          "vs_baseline": None, "dtype": "f32", "data": "synthetic", "impl": "ours",
          "config": {"workload": f"{a.model}-{a.width:g} evaluation forward (MFCC + network, moving-statistics BN), batch {n}"},
          "latency_ms_device": ms, "latency_ms_host_roundtrip": host_ms, "gpu_launches": eng.launch_count(),
          "argmax_first": int(logits[0].argmax())})


def run_augment(a):
    """Device input stage (tcr_augment_pcm16): int16 clips -> decoded, shifted, background-mixed, clipped fp32 wav."""
    import numpy as np
    import torch
    import tcresnet_b200  # noqa: F401
    from tcresnet_b200.engine import Engine
    from tcresnet_b200.datasets import device_input_stage as D
    dev = torch.device("cuda", 0)
    n, clip = a.batch, 16000
    eng = Engine(max_batch=n)
    rng = np.random.RandomState(0)
    bg_lengths = [960000] * 6                          # six one-minute background recordings, as in the dataset
    background = (torch.rand(sum(bg_lengths), device=dev) * 2 - 1) * 0.5
    rot = max(a.rotate, 4)
    pcm = [torch.randint(-32768, 32768, (n, clip), dtype=torch.int16, device=dev) for _ in range(rot)]
    clips = [D.pack(D.draw_clips(rng, [clip] * n, rng.uniform(size=n) < 0.1, clip, bg_lengths), dev) for _ in range(rot)]
    outs = [torch.empty(n, clip, device=dev) for _ in range(rot)]
    for i in range(max(a.warmup, 3)):
        eng.augment(pcm[i % rot], clips[i % rot], background, out=outs[i % rot])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(a.steps):
        eng.augment(pcm[i % rot], clips[i % rot], background, out=outs[i % rot])
    e1.record()
    torch.cuda.synchronize()
    dump_outputs(a, {"wav": outs[(a.steps - 1) % rot]})
    ms = e0.elapsed_time(e1) / a.steps
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm_peak = float(peaks.get("hbm_gbs", 3350.0))
    alg = n * clip * (2 + 4 + 4)                       # int16 read + background read + fp32 write per sample
    gbs = alg / (ms * 1e-3) / 1e9
    emit({"metric": "utterances/sec (device input stage: decode + shift + background mix + clip)", "value": n / (ms * 1e-3),
          "unit": "utterances/sec", "n_gpus": 1, "steps": a.steps, "warmup": max(a.warmup, 3), "ms_per_step": ms,
          "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic", "impl": "ours",
          "config": {"workload": f"tcr_augment_pcm16, batch {n} clips of 16000 samples, 6 background recordings of 60 s",
                     "l2": f"inputs/outputs rotate over {rot} buffers ({rot * alg / 1e6:.0f} MB; the H100's L2 is 50 MB)"},
          "roofline": {"bound": "hbm", "kernel": "augment", "achieved": gbs, "peak": hbm_peak, "unit": "GB/s", "frac": gbs / hbm_peak,
                       "traffic": None, "algorithmic_bytes_per_launch": alg},
          "gpu_launches": eng.launch_count()})


def run_dscnn(a):
    """Config 5: DS-CNN-S forward, MFCC 49x40 features resident in HBM, batch 512, one GPU (2-D-conv comparison point)."""
    import torch
    import tcresnet_b200  # noqa: F401
    from tcresnet_b200.dscnn import DsCnn
    dev = torch.device("cuda", 0)
    n = a.batch
    net = DsCnn("S", 49, 40, 12, max_batch=n)
    gen = torch.Generator(device=dev).manual_seed(7)
    params = torch.randn(net.num_params, device=dev, generator=gen) * 0.1
    for d in net.table:                                           # moving variances must be positive
        if d["name"].endswith("moving_variance"):
            params[d["offset"]:d["offset"] + d["numel"]] = 1.0
    feats = [torch.randn(n, 49, 40, device=dev, generator=gen) for _ in range(a.rotate)]
    for i in range(max(a.warmup, 3)):
        net.forward(feats[i % a.rotate], params)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(a.steps):
        res = net.forward(feats[i % a.rotate], params)
    e1.record()
    torch.cuda.synchronize()
    dump_outputs(a, {"logits": res[0], "probs": res[1]})
    ms = e0.elapsed_time(e1)
    value = n * a.steps / (ms * 1e-3)
    # per-kernel durations (separate pass: the event brackets add overhead) and the roofline of the dominant kernel
    lib = net.lib
    lib.tcr_profile_enable(1)
    for i in range(min(a.steps, 30)):
        net.forward(feats[i % a.rotate], params)
    torch.cuda.synchronize()
    import ctypes as C
    from tcresnet_b200 import _lib as L
    stats_p, cnt = C.POINTER(L.TcrKernelStat)(), C.c_int32()
    L.check(lib, lib.tcr_profile_read(C.byref(stats_p), C.byref(cnt)), "tcr_profile_read")
    stats = {stats_p[i].name.decode(): (float(stats_p[i].total_ms), int(stats_p[i].launches)) for i in range(cnt.value)}
    lib.tcr_profile_enable(0)
    total_ms = sum(v[0] for v in stats.values())
    # DS-CNN-S on 49x40 features: conv_1 (10x4, stride 2x2) -> 25x20x64, then four 3x3 separable blocks at 25x20x64
    hout, wout, ch = (49 + 1) // 2, (40 + 1) // 2, 64
    act = n * hout * wout * ch * 4
    work = {"dscnn_dsblock_ws": (2 * act, n * hout * wout * (2 * 9 * ch + 2 * ch * ch)),
            "dscnn_dsblock_tc": (2 * act, n * hout * wout * (2 * 9 * ch + 2 * ch * ch)),
            "dscnn_dsblock": (2 * act, n * hout * wout * (2 * 9 * ch + 2 * ch * ch)),
            "dscnn_conv_ws": (n * 49 * 40 * 4 + act, n * hout * wout * 2 * 40 * ch),
            "dscnn_conv_tc": (n * 49 * 40 * 4 + act, n * hout * wout * 2 * 40 * ch),
            "dscnn_conv": (n * 49 * 40 * 4 + act, n * hout * wout * 2 * 40 * ch),
            "dscnn_head": (act, n * (hout * wout * ch + 2 * ch * 12))}
    kernels = []
    for name, (tms, c) in sorted(stats.items(), key=lambda kv: -kv[1][0]):
        b, f = work.get(name, (0, 0))
        dur = tms / c * 1e-3
        kernels.append({"name": name, "us": dur * 1e6, "launches_per_step": c / min(a.steps, 30), "share": tms / total_ms,
                        "GBps": b / dur / 1e9, "TFLOPs": f / dur / 1e12})
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm_peak = float(peaks.get("hbm_gbs", 3350.0))
    dom = kernels[0]
    alg_b, alg_f = work.get(dom["name"], (0, 0))
    roofline = {"bound": "hbm", "kernel": dom["name"], "achieved": dom["GBps"], "peak": hbm_peak, "unit": "GB/s",
                "frac": dom["GBps"] / hbm_peak,
                "peak_source": "measured (MEASURED_PEAKS.json)" if "hbm_gbs" in peaks else "fallback 3350 GB/s (H100 SXM data sheet)",
                "traffic": None, "algorithmic_bytes_per_launch": alg_b, "algorithmic_flops_per_launch": alg_f,
                "kernel_us": dom["us"], "kernel_share_of_step": dom["share"],
                "note": "activations in + out once per block (fp32 NHWC); the 1x1 conv runs on wgmma as three TF32 passes "
                        "(6.3 GFLOP/launch incl. the split, a ~13 us floor at the H100's dense TF32 data-sheet rate), so HBM is the roofline"}
    # end to end through the public call with HOST features: pinned host -> H2D -> forward -> D2H probabilities, every step
    h_feats = [f.cpu().pin_memory() for f in feats[:4]]
    d_in = torch.empty(n, 49, 40, device=dev)
    h_out = torch.empty(n, 12).pin_memory()
    esteps = a.steps
    for i in range(12):
        d_in.copy_(h_feats[i % 4], non_blocking=True)
        h_out.copy_(net.forward(d_in, params)[1], non_blocking=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(esteps):
        d_in.copy_(h_feats[i % 4], non_blocking=True)
        h_out.copy_(net.forward(d_in, params)[1], non_blocking=True)
    torch.cuda.synchronize()
    e2e_v = n * esteps / (time.perf_counter() - t0)
    emit({"metric": "utterances/sec (forward) DS-CNN-S", "value": value, "unit": "utterances/sec", "n_gpus": 1,
                      "steps": a.steps, "warmup": max(a.warmup, 3), "ms_per_step": ms / a.steps, "higher_is_better": True,
                      "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic", "impl": "ours",
                      "config": {"workload": f"DS-CNN-S forward (inference), MFCC 49x40 features resident in HBM, batch {n}",
                                 "global_batch": n, "l2": f"inputs rotate over {a.rotate} resident batches; every block streams "
                                                          f"{2 * act / 1e6:.0f} MB of activations (the H100's L2 is 50 MB)",
                                 "exchange": "none (1 GPU)", "forward_flops_per_utt": net.forward_flops,
                                 "pointwise": "fp32 FMA" if os.environ.get("TCR_DSCNN_TC", "2") == "0" else "wgmma 3xTF32"},
                      "fp32_tflops": value * net.forward_flops / 1e12, "roofline": roofline, "kernels": kernels,
                      "gpu_launches": int(sum(k["launches_per_step"] for k in kernels) * a.steps),
                      "e2e": {"value": e2e_v, "unit": "utterances/sec", "h2d_bytes_per_step": n * 49 * 40 * 4,
                              "d2h_bytes_per_step": n * 12 * 4, "steps": esteps,
                              "path": "DsCnn.forward on features copied from pinned host memory, probabilities copied back, every step"}})


_JSON_FD = None


def emit(obj):
    """The ONE JSON line goes to the process's original stdout; everything else any library prints (NCCL's version banner, torch
    warnings) was rerouted to stderr by main()."""
    line = (json.dumps(obj) + "\n").encode()
    if _JSON_FD is None:
        sys.stdout.write(line.decode()); sys.stdout.flush()
    else:
        os.write(_JSON_FD, line)


def main():
    global _JSON_FD
    a = parse_args()
    sys.stdout.flush()
    _JSON_FD = os.dup(1)                # keep the real stdout for the JSON line ...
    os.dup2(2, 1)                       # ... and send fd 1 (C libraries included) to stderr for the rest of the run
    if a.workload == "dscnn":
        return run_dscnn(a)
    if a.workload == "infer":
        return run_infer(a)
    if a.workload == "augment":
        return run_augment(a)
    if a.impl == "reference":
        run_reference(a)
    else:
        run_ours(a)


if __name__ == "__main__":
    main()
