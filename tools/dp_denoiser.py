"""N-rank data-parallel DenoisingAutoencoder.fit == the single-process fit at the global batch
(fp32 math, no BatchNorm).
Launch:  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/dp_denoiser.py
Rank 0 prints one JSON line {"world", "train_loss_rel", "test_loss_rel", "weight_rel"}."""
import json
import os
import shutil
import sys
import tempfile

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import golden_utils as gu  # noqa: E402
import atomai_b200 as ab  # noqa: E402
from atomai_b200.models import DenoisingAutoencoder  # noqa: E402
from atomai_b200.parallel import init_distributed  # noqa: E402


def main():
    init_distributed()
    world, rank = dist.get_world_size(), dist.get_rank()
    ab.set_math("fp32")
    B, hw = 4 * world, 64
    clean = gu.images(31, 3 * B, hw, hw)
    noisy = clean + np.random.RandomState(32).normal(0, 0.1, clean.shape).astype(np.float32)
    data = (noisy[:2 * B], clean[:2 * B], noisy[2 * B:], clean[2 * B:])
    kw = dict(training_cycles=5, batch_size=B, swa=False, plot_training_history=False)
    tmp = tempfile.mkdtemp()
    try:
        dp = DenoisingAutoencoder(seed=3)
        dp.fit(*data, filename=os.path.join(tmp, "dp"), **kw)
        assert dp.comm is not None and dp.comm.world == world
        if rank == 0:
            ref = DenoisingAutoencoder(seed=3)
            ref._no_dp = True          # one process, the whole global batch
            ref.fit(*data, filename=os.path.join(tmp, "ref"), **kw)

            def rel(a, b):
                a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
                return float(np.abs(a - b).max() / np.abs(b).max())
            we = wr = 0.0
            sd = ref.net.state_dict()
            for k, v in dp.net.state_dict().items():
                we += float((v.double() - sd[k].double()).pow(2).sum())
                wr += float(sd[k].double().pow(2).sum())
            print(json.dumps({"world": world,
                              "train_loss_rel": rel(dp.loss_acc["train_loss"], ref.loss_acc["train_loss"]),
                              "test_loss_rel": rel(dp.loss_acc["test_loss"], ref.loss_acc["test_loss"]),
                              "weight_rel": (we / wr) ** 0.5}), flush=True)
        dist.barrier()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
