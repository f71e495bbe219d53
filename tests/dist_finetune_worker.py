"""Worker for the two-rank fine-tune + EMA test (tests/test_finetune_ema.py), one rank per GPU under torchrun.

mode dp     : data-parallel partial training (block 2 only) with the weight EMA, Adam, 4 steps on per-rank batches.  The gradient
              exchange is the default one (peer memory) or NCCL with TCR_P2P=0.  Parameters, both slots and the shadow must be
              bit-identical on every rank; the frozen variables, their slots and their shadow entries untouched.
mode syncbn : the same with tcr_comm_set_sync_bn (per-layer kernels, BatchNorm statistics all-reduced), so the truncated
              backward-data chain runs with the SyncBN record exchange.
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import tcresnet_b200  # noqa: E402,F401
from tcresnet_b200.common.model_loader import variables_to_train  # noqa: E402
from tcresnet_b200.engine import Engine  # noqa: E402
from oracle import tcr_oracle as O  # noqa: E402
from parity_cases import perturbed_variables  # noqa: E402


def main():
    mode = sys.argv[1]
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rank, world = dist.get_rank(), dist.get_world_size()
    n = 32
    spec = O.build_spec("TCResNet8", 1.0, 49)
    params, moving = perturbed_variables(spec)
    wav, onehot = O.synthetic_batch(n * world)
    eng = Engine(max_batch=n, dropout_keep_prob=0.5)
    eng.attach_process_group()
    if mode == "syncbn":
        eng.set_sync_bn(True)
    trained = set(eng.set_trainable(variables_to_train("TCResNet8/block2", eng.trainable_names)))
    dev = eng.device
    p = torch.from_numpy(O.flatten_vars(spec, params)).to(dev)
    mv = torch.from_numpy(O.flatten_moving(spec, moving)).to(dev)
    slots, slots2 = eng.new_optimizer_state("adam")
    ema = eng.new_ema(p)
    p0, ema0 = p.clone(), ema.clone()
    x = torch.from_numpy(wav[rank * n:(rank + 1) * n]).to(dev)
    y = torch.from_numpy(onehot[rank * n:(rank + 1) * n]).to(dev)
    for t in range(4):
        opt = dict(kind="adam", beta1=0.9, beta2=0.999, epsilon=1e-8, beta1_power=0.9 ** (t + 1), beta2_power=0.999 ** (t + 1))
        out = eng.train_step(x, y, p, slots, mv, 1e-3, 0.0, 1e-3, dropout_seed=t * world + rank, want_grads=True, optimizer=opt,
                             slots2=slots2, ema=ema, ema_decay=0.9)
    torch.cuda.synchronize()
    tm = torch.zeros(eng.num_trainable, dtype=torch.bool, device=dev)
    for d in eng.table:
        if d["trainable"] and d["name"] in trained:
            tm[d["offset"]:d["offset"] + d["numel"]] = True
    assert torch.equal(p[~tm], p0[~tm]) and torch.equal(ema[~tm], ema0[~tm]), "frozen entries moved"
    assert not torch.any(slots[~tm]) and not torch.any(slots2[~tm]) and not torch.any(out["grads"][~tm])
    assert not torch.equal(p[tm], p0[tm]) and not torch.equal(ema[tm], ema0[tm]) and torch.isfinite(p).all()
    for name, buf in (("params", p), ("slots", slots), ("slots2", slots2), ("ema", ema)):
        gathered = [torch.zeros_like(buf) for _ in range(world)]
        dist.all_gather(gathered, buf)
        assert all(torch.equal(g, gathered[0]) for g in gathered), f"{name} differ between ranks"
    if rank == 0:
        exchange = getattr(eng, "exchange", "none")            # set by attach_process_group when world > 1
        print(f"finetune {mode} exchange={exchange} world={world}: params, slots and shadows bit-identical on every rank")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
