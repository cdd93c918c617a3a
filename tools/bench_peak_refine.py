"""Cost of the 2-D Gaussian peak refinement (atomai_b200_peak_refine) on the reference's 1024 x 1024
test frame (tests/golden/bfo_1024.npz, 2410 atoms).

  kernel   CUDA events over many launches: the frame at d = 4 and d = 6, and a 16-frame stack of it
           (38560 atoms, d = 4), inputs already on the device
  predict  Segmentor.predict(refine=True) against refine=False with the pretrained bfo weights on
           the frame (fp32 math), host clock after a synchronise
  scipy    the CPU oracle (scipy curve_fit's lmdif, one fit per atom) on the same host, d = 4

Prints one JSON line per measurement, starting with the card's name and power limit.

    python tools/bench_peak_refine.py [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def kernel_ms(fn, iters):
    for _ in range(2):
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
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    import atomai_b200 as ab
    import golden_utils as gu
    import refine_cases as rc
    from atomai_b200 import ops
    from atomai_b200.models import Segmentor
    from atomai_b200.utils.coords import _window_origins
    from oracle import refine_ref as ref
    print(json.dumps({"card": card()}), flush=True)
    dev = torch.device("cuda:0")
    frame, xy = rc.bfo_frame()

    def table(nframes, d):
        org = _window_origins(frame.shape, xy, d)
        t = np.concatenate([np.stack([np.full(len(xy), f), org[:, 0], org[:, 1],
                                      np.full(len(xy), d)], 1) for f in range(nframes)])
        return torch.from_numpy(t.astype(np.int32)).to(dev)

    for nframes, d in ((1, 4), (1, 6), (16, 4)):
        stack = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(
            frame, (nframes,) + frame.shape))).to(dev)
        atoms = table(nframes, d)
        popt = torch.empty((len(atoms), 7), dtype=torch.float64, device=dev)
        info = torch.empty(len(atoms), dtype=torch.int32, device=dev)
        nfev = torch.empty(len(atoms), dtype=torch.int32, device=dev)
        ms = kernel_ms(lambda: ops.peak_refine(stack, atoms, d, popt, info, nfev), args.iters)
        print(json.dumps({"what": "kernel", "frames": nframes, "d": d, "atoms": len(atoms),
                          "ms": round(ms, 3), "us_per_atom": round(1e3 * ms / len(atoms), 4),
                          "median_nfev": float(nfev.float().median()),
                          "maxfev_hits": int((info == 5).sum())}), flush=True)

    ab.set_math("fp32")
    w = gu.load("bfo_weights.npz")
    img = gu.load("bfo_1024.npz")["image"]
    m = Segmentor("Unet", nb_classes=3)
    m.net.load_state_dict({k: torch.from_numpy(w[k]) for k in w.files})
    for refine in (False, True):   # warm-up
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            m.predict(img, refine=refine, d=4, verbose=False)
    for refine in (False, True):
        times = []
        for _ in range(5):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                m.predict(img, refine=refine, d=4, verbose=False)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        med = float(np.median(times))
        print(json.dumps({"what": "predict", "refine": refine, "median_s": round(med, 4)}),
              flush=True)

    t0 = time.perf_counter()
    ref.peak_refinement(frame, xy, 4)
    print(json.dumps({"what": "scipy_oracle", "d": 4, "atoms": len(xy),
                      "s": round(time.perf_counter() - t0, 3)}), flush=True)


if __name__ == "__main__":
    main()
