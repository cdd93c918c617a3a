"""A/B of the weight-gradient kernel between two library builds in one process: on every
tensor-core layer shape of the default Unet at the bench workload (batch 32 x 512^2, the layer
table of tools/bench_layers.py), CUDA-event time of `atomai_b200_conv_wgrad` per build and the
difference of the two dW on the same seeded inputs.

usage: ab_wgrad.py BASE_LIB [NEW_LIB] [--math tf32|tf32x3] [--reps R]
  BASE_LIB, NEW_LIB: paths of libatomai_b200.so builds (NEW_LIB defaults to this tree's)."""
import argparse
import ctypes as C
import os
import sys
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from atomai_b200 import _C, ops
from atomai_b200.ops import Source
from tools.bench_layers import LAYERS, N

ap = argparse.ArgumentParser()
ap.add_argument("base")
ap.add_argument("new", nargs="?", default=_C.LIB_PATH)
ap.add_argument("--math", default="tf32", choices=["tf32", "tf32x3"])
ap.add_argument("--reps", type=int, default=20)
args = ap.parse_args()
MATH = {"tf32": ops.MATH_TF32, "tf32x3": ops.MATH_TF32X3}[args.math]


def load(path):
    lib = C.CDLL(os.path.abspath(path))
    lib.atomai_b200_conv_wgrad.restype = C.c_int
    lib.atomai_b200_conv_wgrad.argtypes = [C.POINTER(_C.Conv), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.atomai_b200_last_error.restype = C.c_char_p
    return lib


libs = {"base": load(args.base), "new": load(args.new)}


def wgrad(lib, d, dy, dw):
    if lib.atomai_b200_conv_wgrad(C.byref(d), dy.data_ptr(), dy.shape[3], dw.data_ptr(),
                                  torch.cuda.current_stream().cuda_stream):
        raise RuntimeError(lib.atomai_b200_last_error().decode())


def timeit(fn, reps):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


dev = "cuda"
print(f"{torch.cuda.get_device_name()}  math={args.math}  batch {N}  reps {args.reps}", flush=True)
print(f"{'layer':5s} {'shape':>20s} | {'base ms':>8s} {'new ms':>8s} {'new/base':>8s} | "
      f"{'max |d|':>9s} {'max |d|/max|dW|':>15s} {'identical':>9s}")
tot = {"base": 0.0, "new": 0.0}
for name, hh, cins, cout, ks, pool in LAYERS:
    g = torch.Generator(device=dev).manual_seed(zlib.crc32(name.encode()))
    srcs = []
    for ci in cins:
        s = 2 * hh if pool else hh
        x = torch.rand(N, s, s, ci, device=dev, generator=g)
        srcs.append(Source(x, torch.rand(ci, device=dev, generator=g) + 0.5,
                           torch.rand(ci, device=dev, generator=g), pool))
    cin = sum(cins)
    d = ops.conv_desc(srcs, N, hh, hh, cout, (ks, ks), 1, 1.0, MATH)
    dy = torch.randn(N, hh, hh, cout, device=dev, generator=g)
    out, ms = {}, {}
    for k, lib in libs.items():
        dw = torch.zeros(cout, cin, ks, ks, device=dev)
        wgrad(lib, d, dy, dw)
        out[k] = dw.clone()
        ms[k] = timeit(lambda: wgrad(lib, d, dy, dw), args.reps)
        tot[k] += ms[k]
    diff = float((out["new"] - out["base"]).abs().max())
    rel = diff / max(float(out["base"].abs().max()), 1e-30)
    same = torch.equal(out["new"].view(torch.int32), out["base"].view(torch.int32))
    print(f"{name:5s} {f'{hh}^2 {cin}->{cout} k{ks}':>20s} | {ms['base']:8.3f} {ms['new']:8.3f} "
          f"{ms['new'] / ms['base']:8.3f} | {diff:9.3g} {rel:15.3g} {str(same):>9s}", flush=True)
print(f"total ms: base {tot['base']:.3f}  new {tot['new']:.3f}  new/base {tot['new'] / tot['base']:.3f}")
