"""N-rank data-parallel dice / focal / IoU == 1-rank values at the global batch (fp32 math).
Launch:  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/dp_seg_objectives.py
Rank 0 prints one JSON line {"world", "dice_loss_rel", "focal_loss_rel", "grad_rel",
"tail_grad_rel_max", "weight_rel", "iou_equal"}."""
import json
import os
import sys
from collections import OrderedDict

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import golden_utils as gu  # noqa: E402
import atomai_b200 as ab  # noqa: E402
from atomai_b200.losses_metrics import IoU, dice_loss, focal_loss  # noqa: E402
from atomai_b200.nets import Unet  # noqa: E402
from atomai_b200.optim import FusedAdam  # noqa: E402
from atomai_b200.parallel import Comm, init_distributed  # noqa: E402


def main():
    init_distributed()
    world, rank = dist.get_world_size(), dist.get_rank()
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    ab.set_math("fp32")
    B, hw = 4 * world, 64
    k = B // world
    x = torch.from_numpy(gu.images(11, B, hw, hw))[:, None].to(dev)
    y = torch.from_numpy(gu.labels(12, B, hw, hw, 3)).to(dev)

    def make():
        net = Unet(nb_classes=3)
        shapes = OrderedDict((n, tuple(v.shape)) for n, v in net.state_dict().items())
        net.load_state_dict({n: torch.from_numpy(v)
                             for n, v in gu.fill_state_dict(shapes, 77).items()})
        return net.to(dev).train()

    comm = Comm(sync_bn=True)
    # dice through the Unet: every rank its slice, SyncBN, summed dice cells, one Adam step with
    # the summed gradients averaged over the ranks (what the trainer does)
    net = make()
    net._comm = comm
    crit = dice_loss()
    crit.comm = comm
    sl = slice(rank * k, (rank + 1) * k)
    logits = net(x[sl])
    loss = crit(logits, y[sl])
    loss.backward()
    grads = OrderedDict()
    for n_, p in net.named_parameters():
        dist.all_reduce(p.grad)
        grads[n_] = p.grad.detach().clone() / world
    opt = FusedAdam(net.parameters(), lr=1e-3)
    opt.grad_scale = 1.0 / world
    opt.step()
    iou_dp = IoU(y[sl], logits.detach(), 3, comm=comm).evaluate()
    ref = make()
    lr_ = dice_loss()(ref(x), y)
    lr_.backward()
    FusedAdam(ref.parameters(), lr=1e-3).step()
    # the same logits evaluated at once: the per-rank confusion counts must add up exactly
    iou_ref = IoU(y, torch.cat(_gather(logits.detach(), world)), 3).evaluate()
    te = tr = we = wr = 0.0
    tail = []
    for (n_, p), (_, q) in zip(ref.named_parameters(), net.named_parameters()):
        e = float((grads[n_].double() - p.grad.double()).pow(2).sum())
        r = float(p.grad.double().pow(2).sum())
        te, tr = te + e, tr + r
        if n_.startswith(("c5.", "c6.", "px.")):
            tail.append((e / (r + 1e-300)) ** 0.5)
        we += float((q.detach().double() - p.detach().double()).pow(2).sum())
        wr += float(p.detach().double().pow(2).sum())
    # focal on 1-channel logits: summed BCE over the ranks
    gen = torch.Generator(device=dev).manual_seed(3)
    z = torch.randn((B, 1, hw, hw), device=dev, generator=gen)
    t = (y[:, None] > 0).float()
    fl = focal_loss()
    fl.comm = comm
    f_dp = fl(z[sl], t[sl])
    f_ref = focal_loss()(z, t)
    out = {"world": world,
           "dice_loss_rel": abs(float(loss) - float(lr_)) / abs(float(lr_)),
           "focal_loss_rel": abs(float(f_dp) - float(f_ref)) / abs(float(f_ref)),
           "grad_rel": (te / tr) ** 0.5, "tail_grad_rel_max": max(tail),
           "weight_rel": (we / wr) ** 0.5, "iou_equal": iou_dp == iou_ref,
           "iou": [iou_dp, iou_ref]}
    if rank == 0:
        print(json.dumps(out), flush=True)
    dist.destroy_process_group()


def _gather(t, world):
    parts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(parts, t.contiguous())
    return parts


if __name__ == "__main__":
    main()
