"""
Regressor / Classifier (MobileNetV2) training step: native sm_90a path vs the same network as
torch.nn.functional calls (oracle/regcls_ref.py) on cuDNN in fp32, on the same GPU, in
alternating rounds.  One step = forward + loss + backward + Adam.  Prints one JSON line per
(model, size) with the median ms of each arm.
    python tools/bench_regcls.py [--batch 64] [--sizes 64 128] [--rounds 5] [--steps 10]
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
import atomai_b200 as ab  # noqa: E402
from atomai_b200.losses_metrics import MSELoss, NLLLoss  # noqa: E402
from atomai_b200.nets import ClassifierNet, RegressorNet  # noqa: E402
from atomai_b200.optim import FusedAdam  # noqa: E402
from oracle import regcls_ref  # noqa: E402


def card():
    """'name, power limit, max SM clock' of the current GPU, read alongside the measurement."""
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                        "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--sizes", type=int, nargs="+", default=[64, 128])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--math", default="tf32x3")
    a = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda")
    gpu = card()
    ab.set_math(a.math)
    for kind in ("reg", "cls"):
        for hw in a.sizes:
            torch.manual_seed(0)
            net = (RegressorNet(1, 2) if kind == "reg" else ClassifierNet(1, 4, "mobilenet")).to(dev)
            x = torch.rand(a.batch, 1, hw, hw, device=dev)
            y = torch.randn(a.batch, 2, device=dev) if kind == "reg" else \
                torch.randint(0, 4, (a.batch,), device=dev)
            crit = MSELoss() if kind == "reg" else NLLLoss()
            opt = FusedAdam(net.parameters(), lr=1e-3)

            def native():
                opt.zero_grad()
                crit(net(x), y).backward()
                opt.step()

            params = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point and
                                                         "running_" not in k)
                      for k, v in net.state_dict().items()}
            leaves = [v for v in params.values() if v.requires_grad]
            topt = torch.optim.Adam(leaves, lr=1e-3)

            def torch_arm():
                topt.zero_grad()
                out = regcls_ref.forward(kind, x, params, True, {})
                regcls_ref.loss(kind, out, y).backward()
                topt.step()

            for f in (native, torch_arm):
                timed(f, 3)
            tn, tt = [], []
            for _ in range(a.rounds):
                tn.append(timed(native, a.steps))
                tt.append(timed(torch_arm, a.steps))
            print(json.dumps({"model": kind, "hw": hw, "batch": a.batch, "math": a.math,
                              "native_ms": round(float(np.median(tn)), 3),
                              "torch_cudnn_fp32_ms": round(float(np.median(tt)), 3),
                              "native_rounds": [round(t, 3) for t in tn],
                              "torch_rounds": [round(t, 3) for t in tt],
                              "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
