"""Fit-cycle cost of the default DenoisingAutoencoder, per-layer convolution times, and the same
network in torch / cuDNN for comparison.

  cycle    DenoisingAutoencoder() (default config, tf32x3 math), batch 32 at 256x256 and 512x512:
           one fit cycle = BaseTrainer.train_step (forward, MSE, backward, fused Adam, loss read
           back) + test_step (eval forward + loss on a second batch).  The arms (two sizes x native
           / torch) alternate for --rounds rounds of --steps cycles each, timed with CUDA events
           after --warmup cycles per arm; median, min and max ms per cycle
  torch    the same cycle with oracle/dae_ref.py in fp32 on the same GPU: cuDNN convolutions with
           TF32 off, torch autograd, torch.optim.Adam
  layers   one native training step at batch 32 x 256x256 with ops.PROFILE on (a separate pass, the
           per-launch events slow the host): kernel family, algorithmic FLOPs and bytes, time of
           every convolution launch (forward, weight gradient, data gradient) by layer

Prints one JSON line per measurement, starting with the card's name and power limit.

    python tools/bench_denoiser.py [--rounds 5 --steps 10 --warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
from collections import OrderedDict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

BATCH = 32


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def data(hw, dev):
    import golden_utils as gu
    # golden_utils.images costs O(h * w) per blob: tile 64 x 64 images up to hw x hw
    clean = torch.from_numpy(np.tile(gu.images(hw, 2 * BATCH, 64, 64), (1, hw // 64, hw // 64)))[:, None]
    noisy = clean + 0.1 * torch.randn(clean.shape, generator=torch.Generator().manual_seed(hw))
    return noisy[:BATCH].to(dev), clean[:BATCH].to(dev), noisy[BATCH:].to(dev), clean[BATCH:].to(dev)


def native_arm(hw, dev):
    from atomai_b200.models import DenoisingAutoencoder
    from atomai_b200.optim import FusedAdam
    m = DenoisingAutoencoder()
    m.optimizer = FusedAdam(list(m.net.parameters()), lr=1e-3)
    m.criterion = m.get_loss_fn("mse")
    x, y, xt, yt = data(hw, dev)

    def cycle():
        m.train_step(x, y)
        m.test_step(xt, yt)
    return cycle


def torch_arm(hw, dev):
    from atomai_b200.models import DenoisingAutoencoder
    from oracle import dae_ref
    sd = OrderedDict((k, torch.nn.Parameter(v.detach().clone().to(dev)))
                     for k, v in DenoisingAutoencoder().net.state_dict().items())
    opt = torch.optim.Adam(list(sd.values()), lr=1e-3)
    x, y, xt, yt = data(hw, dev)
    mse = torch.nn.functional.mse_loss

    def cycle():
        opt.zero_grad(set_to_none=True)
        loss = mse(dae_ref.dae_forward(x, sd, {}, training=True), y)
        loss.backward()
        opt.step()
        loss.item()
        with torch.no_grad():
            mse(dae_ref.dae_forward(xt, sd, {}), yt).item()
    return cycle


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def layer_table(dev):
    """Per-launch rows of one native training step (batch 32, 256x256)."""
    from atomai_b200 import ops
    from atomai_b200.models import DenoisingAutoencoder
    from atomai_b200.optim import FusedAdam
    m = DenoisingAutoencoder()
    m.criterion = m.get_loss_fn("mse")
    m.optimizer = FusedAdam(list(m.net.parameters()), lr=1e-3)
    x, y, _, _ = data(256, dev)
    for _ in range(3):
        m.train_step(x, y)
    names = [n for n, mod in m.net.named_modules() if isinstance(mod, torch.nn.Conv2d)]
    shapes = {n: tuple(mod.weight.shape) for n, mod in m.net.named_modules()
              if isinstance(mod, torch.nn.Conv2d)}
    labels = [(n, "fwd") for n in names]
    for n in reversed(names):              # backward: weight gradient, then data gradient
        labels.append((n, "wgrad"))
        if n != names[0]:                  # the network input needs no gradient
            labels.append((n, "dgrad"))
    ops.PROFILE = []
    try:
        m.train_step(x, y)
        torch.cuda.synchronize()
        prof = list(ops.PROFILE)
    finally:
        ops.PROFILE = None
    assert len(prof) == len(labels), (len(prof), len(labels))
    rows = []
    for (layer, what), (kern, fl, by, e0, e1) in zip(labels, prof):
        ms = e0.elapsed_time(e1)
        rows.append({"what": "layer", "layer": layer, "weight": list(shapes[layer]), "pass": what,
                     "kernel": kern, "gflop": round(fl / 1e9, 3), "mbytes": round(by / 1e6, 2),
                     "us": round(1e3 * ms, 1), "tflops": round(fl / (ms * 1e-3) / 1e12, 2)})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    import atomai_b200 as ab
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    ab.set_math("tf32x3")
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card(), "math": ab.get_math(), "torch_arm": "fp32, TF32 off"}),
          flush=True)
    arms = OrderedDict()
    for hw in (256, 512):
        for impl, make in (("native", native_arm), ("torch_cudnn_fp32", torch_arm)):
            fn = make(hw, dev)
            for _ in range(args.warmup):
                fn()
            torch.cuda.synchronize()
            arms[(impl, hw)] = (fn, [])
    for _ in range(args.rounds):
        for fn, res in arms.values():
            res.append(timed(fn, args.steps))
    for (impl, hw), (_, res) in arms.items():
        print(json.dumps({"what": "fit_cycle", "impl": impl, "batch": BATCH, "hw": hw,
                          "steps": args.steps, "rounds": args.rounds,
                          "median_ms": round(float(np.median(res)), 2),
                          "min_ms": round(min(res), 2), "max_ms": round(max(res), 2)}), flush=True)
    arms.clear()
    torch.cuda.empty_cache()
    rows = layer_table(dev)
    for r in rows:
        print(json.dumps(r), flush=True)
    tot = sum(r["us"] for r in rows)
    print(json.dumps({"what": "layer_total", "launches": len(rows), "us": round(tot, 1)}), flush=True)


if __name__ == "__main__":
    main()
