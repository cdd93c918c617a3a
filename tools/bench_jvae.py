"""Train-step cost of jrVAE against rVAE, and of the fused joint-latent kernels alone.

  step     jrVAE((64, 64), latent_dim=2, discrete_dim=[10], conv_encoder=True) and the same rVAE,
           batch 100, in one process: the two arms alternate for --rounds rounds of --steps train
           steps each (forward, backward, fused Adam, the ELBO read back as train_epoch does), timed
           with CUDA events after --warmup steps per arm; median, min and max ms per step
  latent   joint_latent forward + backward (B = 100, 5 continuous columns, one head of 10) with
           CUDA events over many calls, and the same block as the reference's torch expressions
           (oracle/jvae_ref.py, fp32) for comparison

Prints one JSON line per measurement, starting with the card's name and power limit.

    python tools/bench_jvae.py [--rounds 5 --steps 20 --warmup 5]
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
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def make(kind):
    from atomai_b200.models import jrVAE, rVAE
    if kind == "jrVAE":
        m = jrVAE((64, 64), latent_dim=2, discrete_dim=[10], conv_encoder=True)
    else:
        m = rVAE((64, 64), latent_dim=2, conv_encoder=True)
    return m


def step(m, x):
    elbo = m.forward_compute_elbo(x)
    (-elbo).backward()
    m.optim.step()
    m.optim.zero_grad(set_to_none=True)
    return elbo.item()


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    import atomai_b200 as ab
    import golden_utils as gu
    from atomai_b200.losses_metrics.vi_losses import joint_latent
    from oracle import jvae_ref
    print(json.dumps({"card": card(), "math": "tf32"}), flush=True)
    ab.set_math("tf32")
    dev = torch.device("cuda:0")
    X = gu.images(7, 100, 64, 64)
    x = torch.from_numpy(X).to(dev)
    arms = {}
    for kind in ("rVAE", "jrVAE"):
        m = make(kind)
        m.compile_trainer((X, None), training_cycles=1, batch_size=100)
        m.dx_prior = 0.1
        m.encoder_net.train(); m.decoder_net.train()
        for _ in range(args.warmup):
            step(m, x)
        arms[kind] = (m, [])
    for _ in range(args.rounds):
        for kind, (m, res) in arms.items():
            res.append(timed(lambda: step(m, x), args.steps))
    for kind, (_, res) in arms.items():
        print(json.dumps({"what": "train_step", "model": kind, "batch": 100, "steps": args.steps,
                          "rounds": args.rounds, "median_ms": round(float(np.median(res)), 3),
                          "min_ms": round(min(res), 3), "max_ms": round(max(res), 3)}), flush=True)

    B, heads, Dc = 100, [10], 5
    mu = torch.randn(B, Dc, device=dev, requires_grad=True)
    ls = (0.5 * torch.randn(B, Dc, device=dev)).requires_grad_(True)
    lg = torch.randn(B, 10, device=dev, requires_grad=True)
    eps, u = torch.randn(B, Dc, device=dev), torch.rand(B, 10, device=dev)

    def fused():
        a, zdec, phi, dx, kl = joint_latent(mu, ls, lg, heads, 0.67, eps, coord=3)
        (zdec.sum() + phi.sum() + dx.sum() + kl.sum()).backward()

    def torch_ref():
        a, zdec, phi, dx, kc, kd = jvae_ref.joint_latent(mu, ls, lg, heads, 0.67, eps, u, 3)
        (zdec.sum() + phi.sum() + dx.sum() + kc + kd).backward()

    for name, fn in (("fused", fused), ("torch_expressions", torch_ref)):
        for _ in range(20):
            fn()
        ms = [timed(fn, 200) for _ in range(args.rounds)]
        print(json.dumps({"what": "joint_latent_fwd_bwd", "impl": name, "B": B, "heads": heads,
                          "median_us": round(1e3 * float(np.median(ms)), 2),
                          "min_us": round(1e3 * min(ms), 2), "max_us": round(1e3 * max(ms), 2)}),
              flush=True)


if __name__ == "__main__":
    main()
