"""Cost of the Gaussian-mixture / k-means passes of atomai_b200.stat.

  iter  per case (N sub-images of 32 x 32 x 3, K components, diag): CUDA-event ms of one EM
        iteration (E-step pass + M-step pass + parameter update) and of one Lloyd iteration
        (assignment pass + centre sums + update), averaged over --iters; bytes and flops per
        iteration from the model below, achieved GB/s, and the larger of the HBM and FP32-FMA
        bounds (3.35 TB/s, 67 TFLOP/s, H100 SXM data sheet) over the measured time
  e2e   wall time of GaussianMixture(K, 'diag').fit_predict against sklearn's on the host for the
        same stack, alternating over --rounds ("not measured" when sklearn is not installed)

Model per EM iteration: 2 reads of X (4 N d bytes each) + N K responsibilities written and read;
2 N d K (E: a x + b x^2) + 2 N d K (M: r x, r x^2) FMAs = 8 N d K flops.  Per Lloyd iteration:
2 reads of X, N d K (assign) + N d K (sums) FMAs = 4 N d K flops (the one-hot weights of the sums
count as FMAs).
Prints the card's name and power limit, then one JSON line per measurement.

    python tools/bench_imlocal.py [--iters 20 --rounds 3]
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

HBM, FMA = 3.35e12, 67e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def stack(N, seed=0, K=10, d=32 * 32 * 3):
    rs = np.random.RandomState(seed)
    centres = rs.rand(K, d).astype(np.float32)
    return centres[rs.randint(0, K, N)] + 0.3 * rs.randn(N, d).astype(np.float32)


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


def bench_iter(X, K, iters):
    from atomai_b200 import ops
    from atomai_b200.stat.mixture import _Centred
    N, d = X.shape
    dev = X.device
    data = _Centred(X)
    mu = data.mu
    lab = torch.randint(0, K, (N,), dtype=torch.int32, device=dev)
    sx = torch.empty(K, d, dtype=torch.float64, device=dev)
    sxx, nk = torch.empty_like(sx), torch.empty(K, dtype=torch.float64, device=dev)
    P = [torch.empty(K, d, device=dev), torch.empty(K, d, device=dev), torch.empty(K, device=dev),
         torch.empty(K, d, device=dev), torch.empty(K, d, device=dev), torch.empty(K, device=dev)]
    means, covs, weights, A, B, cst = P
    ops.stat_accum(X, mu, K, sx, sxx, nk, labels=lab)
    ops.stat_gmm_params(sx, sxx, nk, N, 0, 1e-6, 1, *P)
    resp = torch.empty(N, K, device=dev)
    out = torch.empty(1, dtype=torch.float64, device=dev)

    def em():
        ops.stat_estep(X, mu, ops.STAT_GMM, A, B, cst, out, resp=resp)
        ops.stat_accum(X, mu, K, sx, sxx, nk, resp=resp)
        ops.stat_gmm_params(sx, sxx, nk, N, 0, 1e-6, 0, *P)

    c = torch.empty(K, d, device=dev).copy_(X[:K] - mu)
    c2 = torch.empty_like(c)
    Ak, ck = torch.empty(K, d, device=dev), torch.empty(K, device=dev)
    status = torch.zeros(2, dtype=torch.float64, device=dev)
    ops.stat_kmeans_centres(c, Ak, ck)

    def lloyd():
        ops.stat_estep(X, mu, ops.STAT_KMEANS, Ak, None, ck, out, labels=lab, changes=status[:1])
        ops.stat_accum(X, mu, K, sx, nk=nk, labels=lab)
        ops.stat_kmeans_centres(c2, Ak, ck, sx=sx, nk=nk, c_old=c, shift=status[1:])

    rows = []
    for name, fn, nbytes, flops in (
            ("em_iter", em, 2 * 4 * N * d + 2 * 4 * N * K, 8 * N * d * K),
            ("lloyd_iter", lloyd, 2 * 4 * N * d + 3 * 4 * N, 4 * N * d * K)):
        ms = timed(fn, iters)
        s = ms * 1e-3
        bound = max(nbytes / HBM, flops / FMA)
        rows.append({"case": name, "N": N, "d": d, "K": K, "ms": round(ms, 4),
                     "bytes": nbytes, "flops": flops, "GB_s": round(nbytes / s / 1e9, 1),
                     "bound_over_time": round(bound / s, 3),
                     "bound_by": "hbm" if nbytes / HBM > flops / FMA else "fp32_fma"})
    return rows


def bench_e2e(Xh, K, rounds):
    from atomai_b200 import stat
    try:
        from sklearn.mixture import GaussianMixture as SkGMM
    except ImportError:
        SkGMM = None
    nat, sk = [], []
    for _ in range(rounds):
        Xd = torch.from_numpy(Xh).cuda()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        g = stat.GaussianMixture(K, covariance_type="diag", random_state=1)
        g.fit_predict(Xd)
        torch.cuda.synchronize()
        nat.append(time.perf_counter() - t0)
        if SkGMM is not None:
            t0 = time.perf_counter()
            SkGMM(K, covariance_type="diag", random_state=1).fit_predict(Xh)
            sk.append(time.perf_counter() - t0)
    return {"case": "gmm_fit_predict", "N": Xh.shape[0], "d": Xh.shape[1], "K": K,
            "native_s": [round(t, 3) for t in nat], "native_n_iter": g.n_iter_,
            "sklearn_s": [round(t, 3) for t in sk] if sk else "not measured"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sizes", type=int, nargs="+", default=[20000, 100000])
    ap.add_argument("--ks", type=int, nargs="+", default=[5, 10, 20])
    ap.add_argument("--e2e-size", type=int, default=20000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_imlocal needs a CUDA device"
    print(json.dumps({"card": card()}), flush=True)
    for N in args.sizes:
        X = torch.from_numpy(stack(N)).cuda()
        for K in args.ks:
            for row in bench_iter(X, K, args.iters):
                print(json.dumps(row), flush=True)
        del X
    Xh = stack(args.e2e_size)
    for K in args.ks:
        print(json.dumps(bench_e2e(Xh, K, args.rounds)), flush=True)


if __name__ == "__main__":
    main()
