"""N-rank data-parallel Regressor.fit and Classifier.fit == the single-process fit at the global
batch (fp32 math, SyncBN over the ranks).
Launch:  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/dp_regcls.py
         [--backend gloo]   (gloo: every rank on the process's current GPU, e.g. two ranks on one)
Rank 0 prints one JSON line per model: "step_loss_rel" and "grad_rel" (worst module, relative L2)
of one sharded forward / backward against the single process at the global batch, then, for a
5-cycle fit, "first_loss_rel" (cycle 1), "test_loss_rel", "weight_rel" and "stat_rel"."""
import argparse
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
from atomai_b200.models import Classifier, Regressor  # noqa: E402
from atomai_b200.parallel import init_distributed  # noqa: E402


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / np.abs(b).max())


def module_rel(grads, ref):
    """Worst relative L2 error over modules (parameters grouped by module): a BatchNorm bias in
    front of a convolution that feeds another batch-statistics BatchNorm has an analytic gradient
    of zero, so it is measured together with its weight."""
    groups = {}
    for k in ref:
        m = k.rsplit(".", 1)[0]
        e, r = groups.get(m, (0.0, 0.0))
        groups[m] = (e + float((grads[k].double() - ref[k].double()).pow(2).sum()),
                     r + float(ref[k].double().pow(2).sum()))
    worst = max(groups, key=lambda m: groups[m][0] / max(groups[m][1], 1e-300))
    return (groups[worst][0] / max(groups[worst][1], 1e-300)) ** 0.5, worst


def one_step(make, X, y, comm, rank, world):
    """Gradients of one train-mode step: sharded with SyncBN (comm) or whole (comm None)."""
    model = make()
    net = model.net.train()
    crit = model.criterion
    if comm is not None:
        k = len(X) // world
        X, y = X[rank * k:(rank + 1) * k], y[rank * k:(rank + 1) * k]
        net._comm = comm
    X, y = np.ascontiguousarray(X), np.ascontiguousarray(y)
    loss = crit(net(torch.from_numpy(X).cuda()), torch.from_numpy(y).cuda())
    loss.backward()
    grads = {n: p.grad.detach().clone() for n, p in net.named_parameters()}
    loss = loss.detach().reshape(1).clone()
    if comm is not None:          # the trainer's gradient bucket: sum over ranks, / world
        for g in grads.values():
            dist.all_reduce(g)
            g /= world
        dist.all_reduce(loss)
        loss /= world
    return float(loss), grads


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default=None)
    a = ap.parse_args()
    init_distributed(a.backend)
    world, rank = dist.get_world_size(), dist.get_rank()
    ab.set_math("fp32")
    B, hw = 4 * world, 64
    X = gu.images(41, 3 * B, hw, hw)
    rs = np.random.RandomState(42)
    targets = {"reg": rs.normal(0, 1, (3 * B, 2)).astype(np.float32),
               "cls": (np.arange(3 * B) % 3).astype(np.int64)}
    kw = dict(training_cycles=5, batch_size=B, swa=False, plot_training_history=False)
    tmp = tempfile.mkdtemp()
    try:
        for name, make in (("reg", lambda: Regressor(out_dim=2, seed=3)),
                           ("cls", lambda: Classifier(nb_classes=3, seed=3))):
            y = targets[name]
            data = (X[:2 * B], y[:2 * B], X[2 * B:], y[2 * B:])
            from atomai_b200.parallel import Comm
            l_dp, g_dp = one_step(make, X[:B, None], y[:B], Comm(), rank, world)
            if rank == 0:
                l_ref, g_ref = one_step(make, X[:B, None], y[:B], None, rank, world)
                step = {"step_loss_rel": abs(l_dp - l_ref) / abs(l_ref)}
                step["grad_rel"], step["grad_worst_module"] = module_rel(g_dp, g_ref)
            dist.barrier()
            dp = make()
            dp.fit(*data, filename=os.path.join(tmp, "dp_" + name), **kw)
            assert dp.comm is not None and dp.comm.world == world
            if rank == 0:
                ref = make()
                ref._no_dp = True          # one process, the whole global batch
                ref.fit(*data, filename=os.path.join(tmp, "ref_" + name), **kw)
                we = wr = se = sr = 0.0
                sd = ref.net.state_dict()
                for k, v in dp.net.state_dict().items():
                    if not v.dtype.is_floating_point:
                        assert torch.equal(v, sd[k]), k
                        continue
                    e = float((v.double() - sd[k].double()).pow(2).sum())
                    r = float(sd[k].double().pow(2).sum())
                    if "running_" in k:
                        se, sr = se + e, sr + r
                    else:
                        we, wr = we + e, wr + r
                print(json.dumps({"model": name, "world": world, **step,
                                  "first_loss_rel": rel(dp.loss_acc["train_loss"][:1],
                                                        ref.loss_acc["train_loss"][:1]),
                                  "test_loss_rel": rel(dp.loss_acc["test_loss"],
                                                       ref.loss_acc["test_loss"]),
                                  "weight_rel": (we / wr) ** 0.5,
                                  "stat_rel": (se / sr) ** 0.5}), flush=True)
            dist.barrier()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
