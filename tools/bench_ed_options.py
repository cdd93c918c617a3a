"""Cost of ImSpec's encoder_downsampling / 1-D decoder_upsampling and of class conditioning.

  imspec  Im2spec 64 x 64 -> 512 (latent 10, default filters), batch 64: ms per training step
          (forward, MSE, backward, Adam) for encoder_downsampling in {0, 2} x decoder_upsampling in
          {off, on}, with the encoder fc's weight count of each arm
  cvae    VAE and rVAE (conv encoder) on 64 x 64 images, batch 64: ms per training step
          (forward_compute_elbo, backward, Adam) with nb_classes = 0 and nb_classes = 10

Every arm is built and warmed up first; then --rounds rounds run every arm of a group in turn
(alternating), each timing --steps steps between CUDA events.  Reports the median and the spread
of the per-round means.  Prints the card's name and power limit, then one JSON line per arm.

    python tools/bench_ed_options.py [--rounds 5 --steps 20 --warmup 5 --math tf32x3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def imspec_arm(ds, up, batch):
    from atomai_b200.nets import init_imspec_model
    from atomai_b200.optim import FusedAdam
    torch.manual_seed(0)
    net, _ = init_imspec_model((64, 64), (512,), 10, encoder_downsampling=ds, decoder_upsampling=up)
    net = net.cuda().train()
    opt = FusedAdam(list(net.parameters()), lr=1e-4)
    x = torch.rand(batch, 1, 64, 64, device="cuda")
    y = torch.rand(batch, 1, 512, device="cuda")

    def step():
        loss = torch.nn.functional.mse_loss(net(x), y)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
    return step, {"fc_weights": net.encoder.fc.weight.numel()}


def vae_arm(kind, nb_classes, batch):
    from atomai_b200.models import VAE, rVAE
    from atomai_b200.optim import FusedAdam
    cls = VAE if kind == "vae" else rVAE
    m = cls((64, 64), latent_dim=2, nb_classes=nb_classes, conv_encoder=True)
    m.encoder_net.train(); m.decoder_net.train()
    m.dx_prior = 0.1
    opt = FusedAdam(list(m.decoder_net.parameters()) + list(m.encoder_net.parameters()), lr=1e-4)
    g = torch.Generator().manual_seed(0)
    x = torch.rand(batch, 64, 64, generator=g).cuda()
    y = (torch.arange(batch) % nb_classes).cuda() if nb_classes else None

    def step():
        elbo = m.forward_compute_elbo(x, y) if y is not None else m.forward_compute_elbo(x)
        (-elbo).backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
    return step, {}


def timed(step, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        step()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def run_group(group, arms, args):
    built = {}
    for name, make in arms.items():
        step, info = make()
        for _ in range(args.warmup):
            step()
        built[name] = (step, info)
    torch.cuda.synchronize()
    per = {name: [] for name in arms}
    for r in range(args.rounds):
        order = list(arms) if r % 2 == 0 else list(arms)[::-1]
        for name in order:
            per[name].append(timed(built[name][0], args.steps))
    for name, ms in per.items():
        ms = np.array(ms)
        print(json.dumps({"group": group, "arm": name, "batch": args.batch, "math": args.math,
                          "ms_per_step_median": round(float(np.median(ms)), 3),
                          "ms_min": round(float(ms.min()), 3), "ms_max": round(float(ms.max()), 3),
                          **built[name][1]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--math", default="tf32x3", choices=["fp32", "tf32", "tf32x3"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ed_options needs a CUDA device")
    import atomai_b200 as ab
    ab.set_math(args.math)
    print("card:", card(), flush=True)
    b = args.batch
    run_group("imspec", {f"ds{ds}_up{int(up)}": (lambda ds=ds, up=up: imspec_arm(ds, up, b))
                         for ds in (0, 2) for up in (False, True)}, args)
    for kind in ("vae", "rvae"):
        run_group(kind, {f"nb_classes{k}": (lambda k=k: vae_arm(kind, k, b)) for k in (0, 10)}, args)


if __name__ == "__main__":
    main()
