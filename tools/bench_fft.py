"""Cost of FFTmask / FFTsub on the GPU (csrc/fft.cu).

  kernel  device time of each pass from torch.profiler's CUDA activities over --iters calls:
          twiddle / chirp tables, the two row passes (rows), the plain transpose (transpose) and
          the fused store (store_mask, store_sub), and FFTsub's extremes and normalisation; and
          CUDA-event ms of the whole C call averaged over --iters calls after a warm-up, with the
          bytes model below and its rate against the H100 SXM's 3.35 TB/s of HBM3
  e2e     wall time of the public call ending in a device synchronise, median of --iters calls:
          numpy in / numpy out and CUDA in / CUDA out; and scipy.fftpack's restatement on the
          host (the reference's own calls) once in the same run, with whether it agrees with the
          GPU within the test bounds of tests/golden/fft_cases.py
Bytes model of an (h, w) float64 image, N = h w, complex double = 16 B: row pass 1 reads the
image (8 N) and writes 16 N; the transpose and row pass 2 each read and write 16 N; FFTmask's
store reads 16 N and writes F2 and F3 (32 N); FFTsub's first pass reads its spectrum (16 N), its
store reads 16 N and the image (8 N) and writes the difference (8 N), its normalisation reads
8 N and writes 8 N.  The tables and tile extremes are left out.
Workloads: 1024², 2048², 4096², 8192² (radix-2), 1000² and 4093² (Bluestein) float64 images,
maskratio 10.  Prints the card's name and power limit, then one JSON line per measurement.

    python tools/bench_fft.py [--iters 10]
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

import fft_cases as fc  # noqa: E402
from atomai_b200 import ops, utils  # noqa: E402
from atomai_b200.utils import img as imgmod  # noqa: E402

PEAK = 3.35e12
SIZES = ((1024, 1024), (2048, 2048), (4096, 4096), (8192, 8192), (1000, 1000), (4093, 4093))


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


def _pass_name(key):
    for k, n in (("fft_twiddle", "tables"), ("fft_chirp", "tables"), ("fft_rows", "rows"),
                 ("fft_minmax", "minmax"), ("fft_normalise", "normalise")):
        if k in key:
            return n
    if "fft_transpose" in key:
        return {"<0>": "transpose", "<1>": "store_mask", "<2>": "store_sub"}.get(
            next((t for t in ("<0>", "<1>", "<2>") if t in key), ""), "transpose")
    return None


def _pass_ms(fn, iters):
    """mean device ms per call of each pass, from a profiled run of its own"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    ms = {}
    for e in prof.key_averages():
        p = _pass_name(e.key)
        if p is None:
            continue
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        ms[p] = ms.get(p, 0.0) + us / 1e3 / iters
    return {k: round(v, 4) for k, v in ms.items()}


def _fftpack(x):
    """the reference's FFTmask and FFTsub, atomai/utils/img.py:455-486, on the host"""
    from scipy import fftpack
    F2 = fftpack.fftshift(fftpack.fft2(x))
    F3 = F2.copy()
    l, m = int(x.shape[0] / 10), int(x.shape[0] / 2)
    y, xx = np.ogrid[1:2 * l + 1, 1:2 * l + 1]
    mask = (xx - l) * (xx - l) + (y - l) * (y - l) <= l * l
    F3[m - l:m + l, m - l:m + l] = F3[m - l:m + l, m - l:m + l] * (1 - mask)
    rec = np.real(fftpack.ifft2(fftpack.ifftshift(F3)))
    d = np.abs(x - rec)
    d = d - np.amin(d)
    return F2, F3, d / np.amax(d)


def run(h, w, iters):
    tag = f"{h}x{w}"
    x = fc.image(h, w, 1)
    dev = torch.from_numpy(x).cuda()
    N = h * w
    f2 = torch.empty((h, w), dtype=torch.complex128, device="cuda")
    f3 = torch.empty_like(f2)
    r0, c0, l = imgmod._mask_box((h, w), 10)
    out = torch.empty((h, w), dtype=torch.float64, device="cuda")
    mask = lambda: ops.fft2_mask(dev, r0, c0, l, f2, f3)
    sub = lambda: ops.fft2_sub(dev, f3, out)
    for name, fn, nbytes in (("FFTmask", mask, (8 + 16 + 32 + 32 + 16 + 32) * N),
                             ("FFTsub", sub, (16 + 16 + 32 + 32 + 16 + 8 + 8 + 8 + 8) * N)):
        _emit(workload=tag, call=name, measure="passes_ms", **_pass_ms(fn, iters))
        ms = _events(fn, iters)
        _emit(workload=tag, call=name, measure="c_call", ms=round(ms, 4), bytes=nbytes,
              gbps=round(nbytes / ms / 1e6, 1), share_of_peak=round(nbytes / ms / 1e-3 / PEAK, 3))
    _emit(workload=tag, measure="wall_numpy_ms",
          FFTmask=round(_wall(lambda: utils.FFTmask(x), iters) * 1e3, 2),
          FFTsub=round(_wall(lambda: utils.FFTsub(x, f3.cpu().numpy()), iters) * 1e3, 2))
    _emit(workload=tag, measure="wall_cuda_ms",
          FFTmask=round(_wall(lambda: utils.FFTmask(dev), iters) * 1e3, 2),
          FFTsub=round(_wall(lambda: utils.FFTsub(dev, f3), iters) * 1e3, 2))
    t0 = time.perf_counter()
    R2, R3, Rd = _fftpack(x)
    host_s = time.perf_counter() - t0
    G2, G3 = utils.FFTmask(x)
    Gd = utils.FFTsub(x, R3)
    ok_mask = bool(np.linalg.norm(G2 - R2) <= fc.spectrum_tol(R2, False)
                   and np.linalg.norm(G3 - R3) <= fc.spectrum_tol(R3, False))
    from oracle import fft_ref
    _, raw = fft_ref.fftsub(x, R3, raw=True)
    tol = fc.sub_tol(x, R3, raw, False)
    ok_sub = bool(tol is not None and np.abs(Gd - Rd).max() <= tol)
    _emit(workload=tag, measure="fftpack_host", ms=round(host_s * 1e3, 1),
          FFTmask_within_bound=ok_mask, FFTsub_within_bound=ok_sub)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"card: {q}", flush=True)
    for h, w in SIZES:
        run(h, w, a.iters)


if __name__ == "__main__":
    main()
