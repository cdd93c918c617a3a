"""Cost of the segmentation objectives on the benchmark workload (default 3-class Unet, 32 x 512^2
images per batch, tf32x3, device-resident data, deferred loss read-back).

Fit cycles (one train + one test mini-batch) are timed with CUDA events for four arms in one
process, alternating between them round by round: ce, dice, ce + compute_accuracy (IoU on both
steps), dice + compute_accuracy.  Then each new kernel is timed alone at the same size.  Prints
one JSON line per measurement, starting with the card's name and power limit.

    python tools/bench_seg_objectives.py [--rounds 5 --steps 10 --warmup 3]
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


def kernel_ms(fn, iters=50):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--hw", type=int, default=512)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    import atomai_b200 as ab
    from atomai_b200 import ops
    from atomai_b200.models import Segmentor
    print(json.dumps({"card": card()}), flush=True)
    ab.set_math("tf32x3")
    rs = np.random.RandomState(0)
    B, hw = args.batch, args.hw
    X = rs.rand(2 * B, hw, hw).astype(np.float32)
    y = rs.randint(0, 3, (2 * B, hw, hw)).astype(np.int64)
    Xt = rs.rand(B, hw, hw).astype(np.float32)
    yt = rs.randint(0, 3, (B, hw, hw)).astype(np.int64)
    cycles = args.warmup + args.rounds * args.steps + 2
    arms = {"ce": ("ce", False), "dice": ("dice", False), "ce+iou": ("ce", True),
            "dice+iou": ("dice", True)}
    trainers, pos = {}, {}
    for name, (loss, acc) in arms.items():
        m = Segmentor("Unet", nb_classes=3, seed=1)
        m.compile_trainer((X, y, Xt, yt), loss=loss, training_cycles=cycles, batch_size=B,
                          compute_accuracy=acc, memory_alloc=64, plot_training_history=False,
                          sync_host=False, filename="/tmp/bench_seg_objectives")
        for e in range(args.warmup):
            m.step(e)
        trainers[name], pos[name] = m, args.warmup
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for name, m in trainers.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                m.step(pos[name])
                pos[name] += 1
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.steps)
    base = float(np.median(times["ce"]))
    for name in arms:
        med = float(np.median(times[name]))
        print(json.dumps({"arm": name, "cycle_ms_median": round(med, 3),
                          "cycle_ms_min": round(min(times[name]), 3),
                          "cycle_ms_max": round(max(times[name]), 3),
                          "vs_ce_pct": round(100 * (med - base) / base, 2)}), flush=True)
    del trainers
    torch.cuda.empty_cache()

    # the new kernels alone at the benchmark size (NHWC logits as the network leaves them)
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(1)
    l3 = torch.randn((B, hw, hw, 3), device=dev, generator=gen)
    lab = torch.randint(0, 3, (B, hw, hw), device=dev, generator=gen)
    l1 = torch.randn((B, hw, hw, 1), device=dev, generator=gen)
    t1 = (torch.rand((B, 1, hw, hw), device=dev, generator=gen) > 0.5).float()
    K = 3 * hw
    cells = torch.empty(2 * K, device=dev, dtype=torch.float64)
    coef = torch.empty(2 * K, device=dev)
    loss = torch.empty(1, device=dev)
    d3 = torch.empty_like(l3)
    counts = torch.zeros(9, device=dev, dtype=torch.int64)
    acc = torch.zeros(1, device=dev, dtype=torch.float64)
    fac = torch.empty(1, device=dev)
    d1 = torch.empty_like(l1)
    npix = B * hw * hw
    rows = [
        ("dice_sums", lambda: ops.dice_sums(l3, lab, cells), npix * (12 + 8)),
        ("dice_finalize", lambda: ops.dice_finalize(cells, 1e-7, loss, coef), 0),
        ("dice_bwd", lambda: ops.dice_bwd(l3, lab, coef, d3), npix * (12 + 8 + 12)),
        ("iou_hist", lambda: ops.iou_hist(l3, lab, 0.5, counts), npix * (12 + 8)),
        ("iou_finalize", lambda: ops.iou_finalize(counts, 3, loss), 0),
        ("focal_bce_sum", lambda: ops.pointwise_loss(l1, t1, 1, acc), npix * 8),
        ("focal_finalize", lambda: ops.focal_finalize(acc, npix, 0.5, 2.0, loss, fac), 0),
        ("focal_bce_bwd", lambda: ops.pointwise_loss(l1, t1, 1, None, d1, 1.0 / npix, fac),
         npix * 12),
    ]
    for name, fn, nbytes in rows:
        ms = kernel_ms(fn)
        rec = {"kernel": name, "ms": round(ms, 4), "shape": [B, 3 if "focal" not in name else 1,
                                                             hw, hw]}
        if nbytes:
            rec["GB_per_s"] = round(nbytes / ms / 1e6, 1)
            rec["share_of_3.35TB_s"] = round(nbytes / ms / 1e6 / 3350, 3)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
