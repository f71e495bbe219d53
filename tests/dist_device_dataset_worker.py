"""Worker for the two-rank --device_dataset test (tests/test_device_dataset.py), one rank per GPU under torchrun.

argv[1]: a split written by test_device_dataset.make_split, large enough that the 12 steps stay inside one epoch.  Runs
train_audio.train with --data_parallel --device_dataset (every rank holds the whole bank; resident-dataset steps with the front-end
ahead and the default gradient exchange), then checks that parameters, slots and moving statistics are bit-identical on every rank,
and that each step of rank r read rows [r n, (r + 1) n) of the one-GPU global batch of the host path: the same positions (hence the
same draws, which are keyed by global position) and the same labels.
"""
import os
import sys
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import tcresnet_b200  # noqa: E402,F401
from tcresnet_b200 import train_audio  # noqa: E402
from tcresnet_b200.datasets.audio_data_wrapper import SingleLabelAudioDataWrapper  # noqa: E402
from test_device_dataset import _args, _wrapper  # noqa: E402

N = 16


def main():
    root = Path(sys.argv[1])
    rows = []                                        # (position, epoch) of every batch this rank read
    take = SingleLabelAudioDataWrapper.next_device_rows

    def recorded(self):
        rows.append(take(self))
        return rows[-1]
    SingleLabelAudioDataWrapper.next_device_rows = recorded
    trainer = train_audio.train(_args(root, extra=f"--device_dataset --data_parallel --batch_size {N}"))
    model = trainer.model
    model.flush_feed()
    torch.cuda.synchronize()
    rank, world = dist.get_rank(), dist.get_world_size()
    assert model.global_step == 12 and len(rows) == 12 and {e for _, e in rows} == {0}, (model.global_step, rows)
    for name, buf in (("params", model.params), ("slots", model.slots), ("moving", model.moving)):
        gathered = [torch.zeros_like(buf) for _ in range(world)]
        dist.all_gather(gathered, buf)
        assert all(torch.equal(g, gathered[0]) for g in gathered), f"{name} differ between ranks"
    host = _wrapper(_args(root, extra=f"--batch_size {N * world}"))          # one GPU, the global batch, host path
    data = model.dataset.device_data
    labels = np.asarray(host.labels)
    for position, epoch in rows:
        idx = host._take_indices()
        assert position == host._cursor - N * world + rank * N, (position, host._cursor)
        _, hot = data.batch(position, epoch, model.dataset.draw_seed, N)
        assert np.array_equal(hot.argmax(1).cpu().numpy(), labels[idx[rank * N:(rank + 1) * N]])
    torch.cuda.synchronize()
    if rank == 0:
        print(f"device dataset world={world} exchange={getattr(model.engine, 'exchange', 'none')}: params, slots and moving "
              f"statistics bit-identical on every rank; rows and labels are the global batch's")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
