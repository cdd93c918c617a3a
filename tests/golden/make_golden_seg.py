"""
Generates tests/golden/seg_objectives.npz by running the UNMODIFIED reference (AtomAI v0.8.1, CPU
fp32) through oracle/ref_shim.py: dice_loss / focal_loss values and d(logits), IoU values, and
three Adam steps of a Unet trained with each loss.  Run in the build container only:

    python tests/golden/make_golden_seg.py

Inputs come from tests/golden/seg_cases.py (seeded), so only the reference's outputs are stored.
"""
import os
import sys
from collections import OrderedDict

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)

import golden_utils as gu  # noqa: E402
import seg_cases as sc  # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402

aoi = import_reference()
torch.set_num_threads(8)


def loss_and_grad(crit, x, y):
    xt = torch.from_numpy(x).requires_grad_(True)
    loss = crit(xt, torch.from_numpy(y))
    loss.backward()
    return np.float64(loss.item()), xt.grad.numpy().copy()


def adam_case(out, tag, name, crit):
    from test_oracle import CASES, build_case
    from atomai.nets import init_fcnn_model
    c = CASES[name]
    _, sd, _, x, y, _ = build_case(name)
    net, _ = init_fcnn_model(c["model"], c["nb_classes"], **c["cfg"])
    net.load_state_dict(sd)
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    losses = []
    for _ in range(3):
        net.train()
        opt.zero_grad()
        l_ = crit(net(x), y)
        l_.backward()
        opt.step()
        losses.append(l_.item())
    out[f"adam_{tag}/losses"] = np.array(losses, np.float64)
    out[f"adam_{tag}/px_weight"] = net.px.weight.detach().numpy().copy()
    out[f"adam_{tag}/c1_weight"] = net.c1.block[0].weight.detach().numpy().copy()
    print(tag, name, "adam losses", losses)


def main():
    from atomai.losses_metrics import IoU, dice_loss, focal_loss
    out = OrderedDict()
    for name in sc.CASES:
        x, y = sc.case(name)
        out[f"{name}/dice_loss"], out[f"{name}/dice_grad"] = loss_and_grad(dice_loss(), x, y)
        if x.shape[1] == 1:
            out[f"{name}/focal_loss"], out[f"{name}/focal_grad"] = loss_and_grad(focal_loss(), x, y)
        # SegTrainer.accuracy_fn: IoU(y, y_prob, nb_classes).evaluate() (activation truthy)
        out[f"{name}/iou"] = np.float64(IoU(torch.from_numpy(y), torch.from_numpy(x),
                                            x.shape[1]).evaluate())
        print(name, {k.split("/")[1]: float(v) for k, v in out.items()
                     if k.startswith(name + "/") and np.ndim(v) == 0})
    adam_case(out, "dice", sc.ADAM["dice"], dice_loss())
    adam_case(out, "focal", sc.ADAM["focal"], focal_loss())
    np.savez_compressed(os.path.join(HERE, "seg_objectives.npz"), **out)
    print("bytes", os.path.getsize(os.path.join(HERE, "seg_objectives.npz")))


if __name__ == "__main__":
    main()
