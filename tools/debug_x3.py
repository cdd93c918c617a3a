"""Per-kernel accuracy of the tensor-core paths (tf32 / tf32x3) against float64 on layer shapes."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from atomai_b200 import ops
from atomai_b200.ops import Source

dev = "cuda"
torch.manual_seed(0)


def rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30))


for (N, H, W, cin, cout, ks) in [(2, 16, 16, 64, 64, 3), (2, 16, 16, 64, 128, 3), (2, 16, 16, 128, 64, 3), (2, 8, 8, 128, 128, 3), (2, 8, 8, 64, 128, 3), (2, 8, 8, 128, 64, 1), (2, 16, 16, 32, 64, 3),
                                  (2, 64, 64, 16, 16, 3), (2, 64, 64, 32, 16, 3), (2, 32, 32, 64, 64, 3),
                                  (2, 16, 16, 128, 128, 3), (2, 32, 32, 128, 64, 1), (4, 128, 128, 32, 32, 3)]:
    x = torch.randn(N, H, W, cin, device=dev)
    sc = torch.rand(cin, device=dev) + 0.5
    sh = torch.randn(cin, device=dev) * 0.3
    w = torch.randn(cout, cin, ks, ks, device=dev) * 0.1
    dy = torch.randn(N, H, W, cout, device=dev)
    xa = (x * sc + sh).double().permute(0, 3, 1, 2)
    ref_y = F.conv2d(xa, w.double(), padding=ks // 2).permute(0, 2, 3, 1)
    xa_ = xa.detach().requires_grad_(True)
    wd = w.double().requires_grad_(True)
    (F.conv2d(xa_, wd, padding=ks // 2).permute(0, 2, 3, 1) * dy.double()).sum().backward()
    ref_dw, ref_dx = wd.grad, xa_.grad.permute(0, 2, 3, 1)
    line = f"{N}x{H}x{W} {cin}->{cout} k{ks}:"
    for name, math in (("fp32", ops.MATH_FP32), ("tf32", ops.MATH_TF32), ("x3", ops.MATH_TF32X3)):
        d = ops.conv_desc([Source(x, sc, sh)], N, H, W, cout, (ks, ks), 1, 1.0, math)
        y = torch.empty(N, H, W, cout, device=dev)
        ops.conv_fwd(d, ops.prep_weights(w, ops.WMODE_FWD, math), None, y, None)
        dw = torch.zeros_like(w)
        ops.conv_wgrad(d, dy, dw)
        dd = ops.conv_desc([Source(dy)], N, H, W, cin, (ks, ks), 1, 1.0, math)
        dx = torch.empty(N, H, W, cin, device=dev)
        ops.conv_fwd(dd, ops.prep_weights(w, ops.WMODE_DGRAD, math), None, dx, None)
        line += f"  [{name}] fwd {rel(y, ref_y):.1e} wgrad {rel(dw, ref_dw):.1e} dgrad {rel(dx, ref_dx):.1e}"
    print(line, flush=True)
