"""Cost of the Reconstructor's predictive mean and of one training step.

  predict  the mean over every pixel of a 256^2 and a 512^2 grid from N = 10 % of the pixels
           (RBF and Matern-2.5): the fused Gram-times-vector kernel (atomai_b200_gram_matvec)
           against the materialised route, cross-Gram row batches through atomai_b200_gram
           (tf32x3) and a GEMV on the library's GEMM kernel; the two arms alternate, CUDA events
  fit      one Reconstructor training step (fp32 Gram + adjoint, float64 Cholesky, Adam) at N =
           10 % of a 256^2 and a 512^2 grid, host clock after a synchronise

Prints one JSON line per measurement, starting with the card's name and power limit.

    python tools/bench_reconstructor.py [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def event_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def problem(side, seed=0):
    rs = np.random.RandomState(seed)
    n = side * side // 10
    idx = rs.choice(side * side, n, replace=False)
    x = np.stack([idx // side, idx % side], 1).astype(np.float32)
    full = np.indices((side, side)).reshape(2, -1).T.astype(np.float32)
    y = (np.cos(x[:, 0] / 5.0) * np.sin(x[:, 1] / 7.0) + 1.5).astype(np.float32)
    return x, y, full


def bench_predict(side, kind, reps, dev):
    from atomai_b200 import ops
    x, _, full = problem(side)
    c = full.mean(0)
    xt = torch.from_numpy(x - c).to(dev).contiguous()
    xq = torch.from_numpy(full - c).to(dev).contiguous()
    n, nq = len(x), len(full)
    inv_ls = torch.tensor([1 / 6.0, 1 / 9.0], device=dev)
    alpha = torch.randn(n, device=dev, dtype=torch.float64)
    alpha32 = alpha.float()
    out = torch.empty(nq, device=dev, dtype=torch.float64)
    k = {"rbf": 0, "matern": 1}[kind]
    rows = max(16, min(nq, (1 << 30) // (4 * n)) // 16 * 16)      # <= 1 GiB of cross-Gram
    ldk = -(-n // 4) * 4
    kbuf = torch.empty((rows, ldk), device=dev, dtype=torch.float32)
    mat_out = torch.empty((nq, 1), device=dev, dtype=torch.float32)

    def fused():
        ops.gram_matvec(xq, xt, inv_ls, alpha, 0.0, 1.0, k, out)

    def materialised():
        for r0 in range(0, nq, rows):
            r = min(rows, nq - r0)
            kb = kbuf[:r, :n]
            ops.gram(xq[r0:r0 + r], xt, inv_ls, 1.0, k, kb, ops.MATH_TF32X3)
            ops.gemm(kb, ldk, 1, alpha32, 1, 1, mat_out[r0:r0 + r], 1, r, 1, n)

    fused()
    materialised()
    torch.cuda.synchronize()
    diff = float((mat_out[:, 0].double() - out).abs().max() / alpha.abs().sum())
    tf, tm = [], []
    for _ in range(reps):
        tf.append(event_ms(fused))
        tm.append(event_ms(materialised))
    pairs = nq * n
    return dict(bench="predict", grid=f"{side}x{side}", kind=kind, n_train=n, n_query=nq,
                fused_ms=float(np.median(tf)), materialised_ms=float(np.median(tm)),
                fused_runs_ms=[round(t, 3) for t in tf], materialised_runs_ms=[round(t, 3) for t in tm],
                fused_gpairs_per_s=pairs / (np.median(tf) * 1e-3) / 1e9,
                materialised_row_batch=rows, max_diff_over_sum_abs_alpha=diff)


def bench_fit(side, reps, dev):
    from atomai_b200.models import Reconstructor
    from atomai_b200.utils import get_lengthscale_constraints
    x, y, full = problem(side)
    rec = Reconstructor(device=str(dev))
    rec.compile_trainer(x, y, 1, lengthscale_constraints=get_lengthscale_constraints(full))
    rec.train_step()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        rec.train_step()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return dict(bench="fit_step", grid=f"{side}x{side}", n_train=len(x),
                step_ms=float(np.median(ts)), runs_ms=[round(t, 2) for t in ts])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sides", type=int, nargs="+", default=[256, 512])
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_reconstructor needs a CUDA device"
    import __graft_entry__ as g
    g.build()
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card()}), flush=True)
    for side in a.sides:
        for kind in ("rbf", "matern"):
            print(json.dumps(bench_predict(side, kind, a.reps, dev)), flush=True)
    for side in a.sides:
        print(json.dumps(bench_fit(side, max(2, a.reps // 2), dev)), flush=True)


if __name__ == "__main__":
    main()
