"""Cost of the PCA / NMF / FastICA passes of atomai_b200.stat (csrc/decomp.cu).

  kernel  per workload: CUDA-event ms of each pass, averaged over --iters, with the bytes and flops
          of the model below, achieved GB/s and GFLOP/s, and the larger of the HBM and FP32 (FP64
          for the FastICA step) bounds over the measured time (3.35 TB/s, 67 / 34 TFLOP/s, H100
          SXM data sheet); the float64 eigensolve of the Gram is reported on its own line
  e2e     wall time of PCA(k).fit, NMF(k, max_iter=20, tol=0).fit and FastICA(k, max_iter=20).fit
          against sklearn's (default solvers) on the host for the same matrix, once each
          ("not measured" when sklearn is not installed); the sklearn runs are skipped above
          --sk-max-n rows

Model (N rows, d features, k components; one FMA = 2 flops; bytes are the least traffic, one read
of X and one write of each output):
  gram       4 N d bytes, N d (d + 64) flops (upper-triangle 64 x 64 tiles of the d x d Gram)
  project    4 N d + 4 N k bytes, 2 N d k flops
  nmf_w      4 N d + 8 N k bytes (W read and written), 2 N d k + 2 N k^2 flops
  accum WtX  4 N d + 4 N k bytes, 2 N d k flops (atomai_b200_stat_accum, FFMA kernel)
  nmf_h      16 k d bytes, 2 d k^2 flops
  ica_step   4 N k bytes, 4 N k^2 float64 flops
Workloads: stacks of 32 x 32 x 3 windows (d = 3072) at N = 2e4 and 1e5 with k = 10, and a
hyperspectral 65536 x 1024 matrix with k = 4.  Prints the card's name and power limit, then one
JSON line per measurement.

    python tools/bench_decomp.py [--iters 20 --sk-max-n 70000]
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

HBM, FP32, FP64 = 3.35e12, 67e12, 34e12
WORKLOADS = {"stack_2e4": (20000, 3072, 10), "stack_1e5": (100000, 3072, 10),
             "hyper_65536x1024": (65536, 1024, 4)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def data(N, d, seed=0):
    """non-negative mixture of 10 smooth patterns with noise (usable by all three estimators)"""
    rs = np.random.RandomState(seed)
    t = np.linspace(0, 1, d, dtype=np.float32)
    P = np.stack([np.exp(-((t - c) / 0.1) ** 2) for c in rs.rand(10)]).astype(np.float32)
    W = rs.exponential(1.0, (N, 10)).astype(np.float32)
    return W @ P + 0.05 * np.abs(rs.randn(N, d)).astype(np.float32)


def timed(fn, iters):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def report(tag, name, ms, nbytes, flops, peak):
    bound = max(nbytes / HBM, flops / peak)
    print(json.dumps({"workload": tag, "pass": name, "ms": round(ms, 4),
                      "GBps": round(nbytes / ms / 1e6, 1), "GFLOPs": round(flops / ms / 1e6, 1),
                      "bound": "HBM" if nbytes / HBM >= flops / peak else
                      ("FP64" if peak == FP64 else "FP32"),
                      "share_of_bound": round(bound * 1e3 / ms, 3)}), flush=True)


def bench_kernels(tag, Xd, k, iters):
    from atomai_b200 import _C, ops
    N, d = Xd.shape
    dev = Xd.device
    mu = Xd.mean(0).contiguous()
    G = torch.empty(d, d, dtype=torch.float64, device=dev)
    report(tag, "gram", timed(lambda: ops.decomp_gram(Xd, mu, G, False), iters),
           4 * N * d, N * d * (d + 64), FP32)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.linalg.eigh(G)
    e0.record()
    torch.linalg.eigh(G)
    e1.record()
    torch.cuda.synchronize()
    print(json.dumps({"workload": tag, "pass": f"eigh float64 {d} x {d}",
                      "ms": round(e0.elapsed_time(e1), 2)}), flush=True)
    rs = np.random.RandomState(1)
    H = torch.from_numpy(rs.rand(k, d).astype(np.float32)).to(dev)
    W = torch.from_numpy(rs.rand(N, k).astype(np.float32)).to(dev)
    out = torch.empty(N, k, device=dev)
    report(tag, f"project k={k}", timed(lambda: ops.decomp_project(Xd, mu, H, out), iters),
           4 * N * d + 4 * N * k, 2 * N * d * k, FP32)
    HHt = (H.double() @ H.double().T).contiguous()
    wout = torch.empty(k * k + 1, dtype=torch.float64, device=dev)
    W0 = W.clone()
    report(tag, f"nmf_w k={k}", timed(lambda: (W.copy_(W0), ops.decomp_nmf_w(Xd, H, HHt, W, wout)),
                                      iters), 4 * N * d + 8 * N * k, 2 * N * d * k + 2 * N * k * k,
           FP32)
    WtX = torch.empty(k, d, dtype=torch.float64, device=dev)
    report(tag, f"accum WtX k={k}",
           timed(lambda: ops.stat_accum(Xd, None, k, WtX, resp=W, math=_C.MATH_FP32), iters),
           4 * N * d + 4 * N * k, 2 * N * d * k, FP32)
    hout = torch.empty_like(wout)
    WtW = wout[:k * k].view(k, k)
    H0 = H.clone()
    report(tag, f"nmf_h k={k}", timed(lambda: (H.copy_(H0), ops.decomp_nmf_h(WtX, WtW, H, hout)),
                                      iters), 16 * k * d, 2 * d * k * k, FP32)
    X1 = torch.from_numpy(rs.laplace(size=(N, k)).astype(np.float32)).to(dev)
    Wi = torch.from_numpy(np.linalg.qr(rs.randn(k, k))[0]).to(dev)
    iout = torch.empty(k * k + k, dtype=torch.float64, device=dev)
    report(tag, f"ica_step k={k}", timed(lambda: ops.decomp_ica_step(X1, Wi, iout), iters),
           4 * N * k, 4 * N * k * k, FP64)


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def bench_e2e(tag, X, k, sk_max_n):
    import warnings
    from atomai_b200 import stat
    warnings.simplefilter("ignore")
    ours = {"PCA": lambda: stat.PCA(k).fit(X),
            "NMF": lambda: stat.NMF(k, max_iter=20, tol=0.0, random_state=0).fit(X),
            "FastICA": lambda: stat.FastICA(k, max_iter=20, random_state=0).fit(X)}
    try:
        from sklearn import decomposition as skd
    except ImportError:
        skd = None
    for name, fn in ours.items():
        fn()                                           # warm-up: module load, eigensolver setup
        rec = {"workload": tag, "e2e": name, "native_s": round(wall(fn), 4)}
        if skd is None or X.shape[0] > sk_max_n:
            rec["sklearn_s"] = "not measured"
        else:
            sk = {"PCA": lambda: skd.PCA(k).fit(X),
                  "NMF": lambda: skd.NMF(k, max_iter=20, tol=0.0, random_state=0).fit(X),
                  "FastICA": lambda: skd.FastICA(k, max_iter=20, random_state=0).fit(X)}[name]
            t = time.perf_counter()
            sk()
            rec["sklearn_s"] = round(time.perf_counter() - t, 3)
        print(json.dumps(rec), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--sk-max-n", type=int, default=70000)
    ap.add_argument("--workloads", nargs="*", default=list(WORKLOADS))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_decomp needs a CUDA device")
    print("card:", card(), flush=True)
    for tag in a.workloads:
        N, d, k = WORKLOADS[tag]
        X = data(N, d)
        Xd = torch.from_numpy(X).cuda()
        bench_kernels(tag, Xd, k, a.iters)
        del Xd
        bench_e2e(tag, X, k, a.sk_max_n)


if __name__ == "__main__":
    main()
