"""Per-layer CUDA-event timing of the three conv kernels (fwd, dgrad, wgrad) on the tensor-core
layer shapes of the default Unet at the bench workload (batch 32 x 512^2).  usage: bench_layers.py [fwd] [dgrad] [wgrad] [--math tf32|tf32x3]"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from atomai_b200 import ops
from atomai_b200.ops import Source
N = 32
LAYERS = [  # name, H, [cins], cout, ks, pool   (default Unet: nb_filters 16, layers [1, 2, 2, 3])
    ("c2.0", 256, [16], 32, 3, True), ("c2.1", 256, [32], 32, 3, False),
    ("c3.0", 128, [32], 64, 3, True), ("c3.1", 128, [64], 64, 3, False),
    ("bn.0", 64, [64], 128, 3, True), ("bn.1", 64, [128], 128, 3, False), ("bn.2", 64, [128], 128, 3, False),
    ("u1", 64, [128], 64, 1, False), ("c4.0", 128, [64, 64], 64, 3, False), ("c4.1", 128, [64], 64, 3, False),
    ("u2", 128, [64], 32, 1, False), ("c5.0", 256, [32, 32], 32, 3, False), ("c5.1", 256, [32], 32, 3, False),
    ("u3", 256, [32], 16, 1, False), ("c6.0", 512, [16, 16], 16, 3, False),
]
args = sys.argv[1:]
MATH = ops.MATH_TF32
if "--math" in args:
    i = args.index("--math")
    MATH = {"tf32": MATH, "tf32x3": ops.MATH_TF32X3, "fp32": ops.MATH_FP32}[args[i + 1]]
    del args[i:i + 2]
which = args or ["fwd", "dgrad", "wgrad"]
dev = "cuda"
def timeit(fn, reps=5):
    for _ in range(2): fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps
tot = {k: 0.0 for k in which}
for name, hh, cins, cout, ks, pool in LAYERS:
    srcs = []
    for ci in cins:
        s = 2 * hh if pool else hh
        x = torch.rand(N, s, s, ci, device=dev)
        srcs.append(Source(x, torch.rand(ci, device=dev) + 0.5, torch.rand(ci, device=dev), pool))
    cin = sum(cins)
    w = torch.randn(cout, cin, ks, ks, device=dev) * 0.05
    b = torch.randn(cout, device=dev) * 0.1
    out = torch.empty(N, hh, hh, cout, device=dev)
    st = torch.zeros(2 * cout, device=dev, dtype=torch.float64)
    d = ops.conv_desc(srcs, N, hh, hh, cout, (ks, ks), 1, 0.01, MATH)
    row = [f"{name:5s} {hh:3d}^2 {cin:3d}->{cout:3d} k{ks}"]
    gb_f = 4.0 * N * hh * hh * (cin * (4 if pool else 1) + cout) / 1e9
    if "fwd" in which:
        wp = ops.prep_weights(w, ops.WMODE_FWD, MATH)
        ms = timeit(lambda: ops.conv_fwd(d, wp, b, out, st)); tot["fwd"] += ms
        row.append(f"fwd {ms*1e3:7.1f} us ({gb_f/ms*1e3:5.0f} GB/s)")
    dy = torch.randn(N, hh, hh, cout, device=dev)
    if "dgrad" in which and not pool:
        dd = ops.conv_desc([Source(dy)], N, hh, hh, cin, (ks, ks), 1, 1.0, MATH, act=ops.ACT_LRELU)
        wd = ops.prep_weights(w, ops.WMODE_DGRAD, MATH)
        dx = torch.empty(N, hh, hh, cin, device=dev)
        ms = timeit(lambda: ops.conv_fwd(dd, wd, None, dx, None)); tot["dgrad"] += ms
        row.append(f"dgrad {ms*1e3:7.1f} us")
    if "wgrad" in which:
        dw = torch.zeros(cout, cin, ks, ks, device=dev)
        ms = timeit(lambda: ops.conv_wgrad(d, dy, dw)); tot["wgrad"] += ms
        row.append(f"wgrad {ms*1e3:7.1f} us ({gb_f/ms*1e3:5.0f} GB/s)")
    print(" | ".join(row), flush=True)
    del srcs, out, dy
print("totals ms:", {k: round(v, 3) for k, v in tot.items()})
