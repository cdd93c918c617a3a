"""
Generates tests/golden/*.npz by running the UNMODIFIED reference (/root/reference, AtomAI v0.8.1,
CPU fp32) through oracle/ref_shim.py.  Run in the build container only:

    python tests/golden/make_golden.py

The committed .npz files are what travels to the GPU box; /root/reference does not exist there.
Inputs and weights come from tests/golden/golden_utils.py (seeded numpy RandomState), so only the
reference's OUTPUTS are stored.
"""
import os
import sys
from collections import OrderedDict

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import golden_utils as gu  # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402

aoi = import_reference()
torch.set_num_threads(8)


def load_seeded(net, seed):
    shapes = OrderedDict((k, tuple(v.shape)) for k, v in net.state_dict().items())
    vals = gu.fill_state_dict(shapes, seed)
    net.load_state_dict({k: torch.from_numpy(v) for k, v in vals.items()})
    return net


def fcnn_case(tag, model, nb_classes, seed, n, h, w, logit_stride=1, **kw):
    """eval logits, train logits, loss, grads (sampled), BN running stats after one train fwd."""
    from atomai.nets import init_fcnn_model
    net, meta = init_fcnn_model(model, nb_classes, **kw)
    load_seeded(net, seed)
    x = torch.from_numpy(gu.images(seed + 1, n, h, w))[:, None]
    if nb_classes > 2:
        y = torch.from_numpy(gu.labels(seed + 2, n, h, w, nb_classes))
        crit = torch.nn.CrossEntropyLoss()
    else:
        y = torch.from_numpy((gu.labels(seed + 2, n, h, w, 2) > 0).astype(np.float32))[:, None]
        crit = torch.nn.BCEWithLogitsLoss()
    out = {}
    net.eval()
    with torch.no_grad():
        out["logits_eval"] = net(x).numpy()
    out["logit_stride"] = np.int64(logit_stride)
    net.train()
    net.zero_grad()
    logits = net(x)
    loss = crit(logits, y)
    loss.backward()
    out["logits_train"] = logits.detach().numpy()
    out["loss_train"] = np.float64(loss.item())
    for k, p in net.named_parameters():
        g = p.grad.numpy()
        out["gradnorm/" + k] = np.float64(np.linalg.norm(g.astype(np.float64)))
        out["grad/" + k] = gu.sample_flat(g, 97) if g.size > 4096 else g.copy()
    for k, b in net.named_buffers():
        if "running" in k:
            out["buf/" + k] = b.numpy().copy()
    # three Adam steps (BaseTrainer.train_step semantics, lr 1e-3) -> loss curve + final px weights
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    losses = []
    load_seeded(net, seed)
    for _ in range(3):
        net.train()
        opt.zero_grad()
        l_ = crit(net(x), y)
        l_.backward()
        opt.step()
        losses.append(l_.item())
    out["adam_losses"] = np.array(losses, np.float64)
    last = net.px if hasattr(net, "px") else net.out
    first = net.c1.block[0] if hasattr(net, "c1") else net.net1.res_module[0].c0
    out["adam_px_weight"] = last.weight.detach().numpy().copy()
    out["adam_c1_weight"] = first.weight.detach().numpy().copy()
    if logit_stride > 1:
        out["logits_absmax"] = np.float64(np.abs(out["logits_eval"]).max())
        out["logits_eval"] = gu.sample_flat(out["logits_eval"], logit_stride)
        out["logits_train"] = gu.sample_flat(out["logits_train"], logit_stride)
    np.savez_compressed(os.path.join(HERE, f"{tag}.npz"), **out)
    print(tag, "loss", loss.item(), "adam", losses, "logits absmax", np.abs(out["logits_eval"]).max())


def bfo_case():
    """Real pretrained default 3-class Unet on a crop of the reference's own test image."""
    from atomai.models import load_model
    m = load_model("/root/reference/pretrained/bfo.tar")
    net = m.net.cpu().eval()
    img = np.load("/root/reference/test/predictors/test_data/test_inputimg.npy")
    crop = img[256:384, 320:448].astype(np.float32)
    crop = (crop - crop.min()) / np.ptp(crop)
    with torch.no_grad():
        logits = net(torch.from_numpy(crop)[None, None]).numpy()
    sd = {k: v.cpu().numpy() for k, v in net.state_dict().items()}
    gu.save("bfo_weights.npz", **sd)
    np.savez_compressed(os.path.join(HERE, "bfo_crop.npz"), image=crop, logits=logits)
    print("bfo", logits.shape, np.abs(logits).max())


def bfo_full_case():
    """pretrained/bfo.tar through the reference's whole predict pipeline on its own 1024x1024 test
    image (SURVEY.md 8c(ii)): Segmentor.predict -> softmax output + Locator coordinates (2410 atoms).
    Stores the image (the GPU box has no /root/reference), a strided sample of the eval logits and
    of the softmax output, the coordinates, and how close any pixel's class probability comes to
    the Locator threshold 0.5 (the margin a different arithmetic has before a mask pixel flips)."""
    from atomai.models import load_model
    m = load_model("/root/reference/pretrained/bfo.tar")
    img = np.load("/root/reference/test/predictors/test_data/test_inputimg.npy").astype(np.float32)
    nn_out, coords = m.predict(img)
    net = m.net.cpu().eval()
    x = (img - img.min()) / np.ptp(img)
    with torch.no_grad():
        logits = net(torch.from_numpy(x.astype(np.float32))[None, None]).numpy()
    margin = np.sort(np.abs(nn_out[..., :-1].astype(np.float64) - 0.5).reshape(-1))[:16]
    gu.save("bfo_1024.npz", image=img,
            logits=gu.sample_flat(logits, 61), logits_absmax=np.float64(np.abs(logits).max()),
            nn_output=gu.sample_flat(nn_out, 61), coordinates=coords[0],
            threshold_margins=margin)
    print("bfo_1024", nn_out.shape, coords[0].shape, "closest |p-0.5|:", margin[:4])


def locator_case():
    """Locator.run on a crop of the reference's golden NN output (test/predictors/test_locator.py)."""
    from atomai.predictors import Locator
    nn_out = np.load("/root/reference/test/predictors/test_data/test_nnoutput.npy")
    crop = np.ascontiguousarray(nn_out[:, 300:492, 400:592, :]).astype(np.float32)
    coords = Locator(0.5, 5).run(crop)
    np.savez_compressed(os.path.join(HERE, "locator_crop.npz"), nn_output=crop,
                        coordinates=coords[0])
    print("locator", coords[0].shape)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "locator":
        locator_case()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "big512":
        # BASELINE.json configs[1] geometry (512x512, default 3-class Unet), N = 2
        fcnn_case("unet_default_3c_512", "Unet", 3, 700, 2, 512, 512, logit_stride=61)
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "bfo1024":
        bfo_full_case()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "big":
        fcnn_case("unet_default_3c_128", "Unet", 3, 600, 4, 128, 128, logit_stride=5)
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "resnets":
        fcnn_case("segresnet_default_3c", "SegResNet", 3, 800, 2, 64, 64)
        fcnn_case("segresnet_nobn_1c", "SegResNet", 1, 810, 2, 32, 32, batch_norm=False, nb_filters=16,
                  upsampling="nearest")
        fcnn_case("reshednet_3c", "ResHedNet", 3, 820, 2, 64, 64, nb_filters=16, layers=[2, 2, 2])
        sys.exit(0)
    fcnn_case("unet_default_3c", "Unet", 3, 100, 2, 32, 48)
    fcnn_case("unet_nearest_1c", "Unet", 1, 200, 2, 32, 32, upsampling="nearest", nb_filters=8)
    fcnn_case("unet_dilated_3c", "Unet", 3, 300, 2, 64, 64, with_dilation=True)
    fcnn_case("unet_nobn_3c", "Unet", 3, 400, 2, 32, 32, batch_norm=False, layers=[2, 2, 2, 2])
    fcnn_case("dilnet_default_3c", "dilnet", 3, 500, 2, 32, 32)
    fcnn_case("unet_default_3c_128", "Unet", 3, 600, 4, 128, 128, logit_stride=5)
    bfo_case()
    locator_case()
