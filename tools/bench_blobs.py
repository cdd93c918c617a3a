"""Cost of filter_cells / filter_cells_ on the GPU (csrc/blobs.cu).

  kernel  device time of each pass (local, merge, roots, write) from torch.profiler's CUDA
          activities over --iters calls, and CUDA-event ms of the whole filter (one C call, four
          launches) averaged over --iters calls after a warm-up, with the bytes model below and
          the rate it gives against the H100 SXM's 3.35 TB/s
  e2e     wall time of the public call ending in a device synchronise, median of --iters calls:
          numpy in / numpy out and CUDA in / CUDA out; and the host restatement
          (oracle/blobs_ref.py: threshold, scipy.ndimage.label, np.bincount, frame by frame) once
          in the same run, with a flag for exact equality of the outputs
Bytes model per pixel, with s the input's and o the output's element size: local s + 8 (pixels
read; labels and counts written); merge 64 B per tile edge pair (two labels on each side of its
32-pixel top and left edges); roots 4 (the counts read; tile roots also climb to their root,
which hits in cache); write 4 + o (labels read, output written; the counts read at the roots and
the label rewrites of pixels whose tile root moved are left out).  So the model is a lower bound.
Workloads: 100 frames of 1024² float32 at fill 0.4 with blob_thresh 20 (a movie of small
particles); 8 frames of 2048² at fill 0.59, near the square lattice's site-percolation threshold,
where the largest components are fractal and span many tiles; one 4096² frame at fill 0.59
through filter_cells_.  Prints the card's name and power limit, then one JSON line per measurement.

    python tools/bench_blobs.py [--iters 10]
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
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import blobs_cases as bc  # noqa: E402
from atomai_b200 import ops, utils  # noqa: E402
from oracle import blobs_ref  # noqa: E402

PEAK = 3.35e12
PASSES = ("blob_local", "blob_merge", "blob_roots", "blob_write")


def _emit(**kw):
    print(json.dumps(kw), flush=True)


def _events(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def _wall(fn, iters):
    fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    return float(np.median(t))


def _pass_ms(fn, iters):
    """mean device ms per call of each pass, from a profiled run of its own"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    ms = dict.fromkeys(PASSES, 0.0)
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        for p in PASSES:
            if f"{p}_kernel" in e.key:
                ms[p] += us / 1e3 / iters
    return ms


def run(tag, host, iters, im_thresh, blob_thresh, single=False):
    n, h, w = host.shape
    dev = torch.from_numpy(host).cuda()
    out_dtype = torch.int32 if single else dev.dtype
    labels = torch.empty(dev.shape, dtype=torch.int32, device="cuda")
    counts = torch.empty_like(labels)
    out = torch.empty(dev.shape, dtype=out_dtype, device="cuda")
    filt = lambda: ops.blob_filter(dev, im_thresh, blob_thresh, False, labels, counts, out)
    npix = n * h * w
    tiles = n * -(-h // 32) * -(-w // 32)
    s, o = dev.element_size(), out.element_size()
    model = {"blob_local": npix * (s + 8), "blob_merge": tiles * 64, "blob_roots": npix * 4,
             "blob_write": npix * (4 + o)}
    for p, ms in _pass_ms(filt, iters).items():
        _emit(workload=tag, measure=f"{p}_kernel", ms=round(ms, 4), bytes=model[p],
              gbps=round(model[p] / ms / 1e6, 1) if ms else None)
    total = sum(model.values())
    ms = _events(filt, iters)
    _emit(workload=tag, measure="filter_total", ms=round(ms, 4), bytes=total,
          bytes_per_pixel=round(total / npix, 2), gbps=round(total / ms / 1e6, 1),
          share_of_peak=round(total / ms / 1e-3 / PEAK, 3),
          gpix_per_s=round(npix / ms / 1e6, 2))
    if single:
        np_call = lambda: utils.filter_cells_(host[0], im_thresh, blob_thresh)
        cu_call = lambda: utils.filter_cells_(dev[0], im_thresh, blob_thresh)
    else:
        np_call = lambda: utils.filter_cells(host, im_thresh, blob_thresh)
        cu_call = lambda: utils.filter_cells(dev, im_thresh, blob_thresh)
    _emit(workload=tag, measure="wall_numpy", ms=round(_wall(np_call, iters) * 1e3, 2))
    _emit(workload=tag, measure="wall_cuda", ms=round(_wall(cu_call, iters) * 1e3, 2))
    t0 = time.perf_counter()
    ref = blobs_ref.filter_frame(host[0], im_thresh, blob_thresh) if single else \
        blobs_ref.filter_stack(host, im_thresh, blob_thresh)
    host_s = time.perf_counter() - t0
    _emit(workload=tag, measure="oracle_host", ms=round(host_s * 1e3, 1),
          equal=bool(np.array_equal(np_call(), ref)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"card: {q}", flush=True)
    run("stack_100x1024_fill0.4", bc.stack(100, 1024, 1024, 1, 0.4), a.iters, 0.6, 20)
    run("stack_8x2048_fill0.59", bc.stack(8, 2048, 2048, 2, 0.59), a.iters, 0.41, 20)
    run("frame_4096_fill0.59", bc.stack(1, 4096, 4096, 3, 0.59), a.iters, 0.41, 20, single=True)


if __name__ == "__main__":
    main()
