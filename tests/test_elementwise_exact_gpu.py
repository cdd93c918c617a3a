"""Exact and float64 parity of the memory-bound kernels around the convolutions (elementwise.cu,
resnet.cu, the non-convolution kernels of mobilenet.cu, and vae.cu's GEMM, Linear and coord_latent
kernels), driven through the C ABI (`atomai_b200.ops`).

Layout control.  Every NHWC operand is placed in a NaN-filled buffer (class Slot): pixel stride
ld = C + pad and an optional start offset of one float, so each case decides which dispatch path
runs.  The predicates are mirrored here (vec_ok for elementwise.cu, res_vec_ok for resnet.cu's
affine_res_act) and each case id names the path it must take ("f4" or "scalar").  The shape grid
covers C in {1, 3, 5} (scalar only), {12, 24, 48} (float4 with the division branch of ChanIdx<4>),
{4, 16, 32, 1024} (float4, shift branch), C = 32 with ld = 33 (scalar), odd H and W, h or w = 1
for the resamplers, N = 1, and launches large enough for the grid-stride loops to go round more
than once (ab_grid caps the grid at 8 x SMs CTAs in elementwise.cu).

(a) Exact tier.  Small integers, BN scales in +-{0.5, 1, 2}, shifts on a 0.5 grid, LeakyReLU
    slope 0.25, resize factors 2 and 4 and the bilinear x2 weights 1/4 and 3/4: every product and
    partial sum is exact (float atomics and the ordered double sums included), so the result must
    be bitwise equal to the float64 reference.  Each case asserts that precondition: the sum of
    |terms| in units of the value grid stays below 2^24.  Max-pool ties (first maximum wins, as in
    ATen) and ReLU6 inputs exactly on 0 and 6 (mask 0, as in hardtanh_backward) are reached here.
(b) Normal tier.  randn data, per element |y - y64| <= k 2^-24 sum|terms|, k the number of
    roundings in the kernel's expression (inputs that the kernel receives rounded to fp32, such as
    BatchNorm statistics, count as roundings).  The __expf / __logf losses get explicit budgets
    (see ce_budget / bce_budget), with logits of +-80 to reach the max-subtraction and log1p paths.
    Largest |y - y64| / bound observed on the first run (H100 80GB HBM3, 700 W power limit):
    about 1.0 for the single-rounding kernels (affine, add_slice, pool backward, affine_relu6,
    where the bound is one rounding), 0.75 avgpool_bwd, 0.62 affine_res_act, 0.54 dilated_sum,
    0.53 upsample, 0.48 resize, 0.47 log_softmax_bwd, 0.39 bn_finalize, 0.37 bn_act_bwd,
    0.36 linear, 0.22 coord_latent forward, 0.14 gemm, and at most 0.03 for every sum over pixels
    (BatchNorm sums, dbias, losses, coord_latent backward).
(c) Float4 against scalar.  The W = 4 and W = 1 instances of every per-element kernel are bitwise
    identical on the same data.
(d) Sentinels.  Pad channels and the guard floats around each buffer still hold NaN bits after
    every call; every non-accumulating output is NaN-filled first; accumulating outputs start
    from non-zero values.
(e) Reproducibility.  Every ordered reduction is bitwise identical across two launches (the float
    atomics of resize_bwd, split-K gemm, the skinny Linear forward and coord_latent_bwd are
    exempt).
(f) Host-side refusals raise NativeError from argument checks before any launch.
(g) Dispatch coverage: torch.profiler confirms that both instances (<4> and <1>) of every dual-path
    kernel were launched.
"""
import ctypes as C
import itertools
import math
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from atomai_b200 import _C, ops
from atomai_b200.ops import ACT_LRELU, ACT_TANH

LIMIT = 2 ** 24
U = 2.0 ** -24
NAN_BITS = 0x7FC00000

gpu = pytest.mark.gpu


# ----------------------------------------------------------------------------- values
def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def ints(g, shape, amp=3, zero=0.2):
    v = torch.randint(-amp, amp + 1, shape, generator=g).double()
    return torch.where(torch.rand(shape, generator=g) < zero, torch.zeros_like(v), v)


def normal(g, shape):
    return torch.randn(shape, generator=g, dtype=torch.float32).double()


def vals(g, shape, data, amp=3):
    return ints(g, shape, amp) if data == "int" else normal(g, shape)


def bn_scale(g, C, data):
    if data == "int":
        return torch.tensor([0.5, 1.0, 2.0])[torch.randint(0, 3, (C,), generator=g)] * \
            (torch.randint(0, 2, (C,), generator=g).double() * 2 - 1)
    return normal(g, (C,))


def bn_shift(g, C, data):
    if data == "int":
        return torch.randint(-4, 5, (C,), generator=g).double() * 0.5
    return normal(g, (C,))


def grid_of(*ts):
    """Largest power of two 2^-e (e >= 0) that divides every value of the tensors."""
    for e in range(0, 60):
        s = 2.0 ** e
        if all(bool(torch.all(torch.frac(t.double() * s) == 0)) for t in ts if t is not None):
            return 2.0 ** -e
    raise AssertionError("values are not on a binary grid")


def exact_case(mag, unit, what):
    """The exact-tier precondition: every partial sum is a multiple of `unit` below 2^24 units."""
    m = float(mag.max()) if mag.numel() else 0.0
    assert m / unit < LIMIT, f"{what}: not an exact case (max sum|terms| {m}, grid {unit})"


def first_mismatch(got, ref):
    got, ref = got.double(), ref.double()
    bad = ~(got == ref)
    n = int(bad.sum())
    if n == 0:
        return None
    idx = tuple(int(i) for i in bad.nonzero()[0])
    return (f"{n}/{bad.numel()} elements differ, first at {idx}: got {float(got[idx])!r}, "
            f"want {float(ref[idx])!r}")


def expect(got, ref, mag, k, data, what, unit=None):
    """data == "int": bitwise equal to the float64 reference (after checking the exact-case
    precondition with grid `unit`); otherwise |got - ref| <= k 2^-24 mag per element."""
    got, ref, mag = got.double(), ref.double(), mag.double()
    if data == "int":
        if unit is not None:
            exact_case(mag, unit, what)
        msg = first_mismatch(got, ref)
        assert msg is None, f"{what}: {msg}"
        return 0.0
    err = (got - ref).abs()
    bound = k * U * mag
    bad = ~(err <= bound)
    if bool(bad.any()):
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.numel()} elements outside "
                             f"{k} 2^-24 sum|terms|, first at {idx}: got {float(got[idx])!r}, "
                             f"want {float(ref[idx])!r}, bound {float(bound[idx])!r}")
    return float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0


def same_bits(a, b, what):
    a, b = a.contiguous(), b.contiguous()
    assert a.dtype == b.dtype and a.shape == b.shape
    ia = a.view(torch.int32 if a.dtype == torch.float32 else torch.int64)
    ib = b.view(ia.dtype)
    bad = ia != ib
    if bool(bad.any()):
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} elements differ in their bits, first at "
                             f"{idx}: {float(a[idx])!r} vs {float(b[idx])!r}")


# ----------------------------------------------------------------------------- layout control
LAYOUTS = {"dense": (0, 0), "ld4": (4, 0), "ld1": (1, 0), "off1": (0, 1)}


class Slot:
    """An NHWC (N, H, W, C) tensor inside a NaN-filled flat float32 buffer: pixel stride
    ld = C + pad, data starting `off` floats in (off = 1 gives a 4-byte-misaligned pointer), and
    four guard floats after it."""

    def __init__(self, shape, dev, lay="dense", values=None):
        pad, off = LAYOUTS[lay] if isinstance(lay, str) else lay
        N, H, W, Cc = shape
        n = N * H * W * (Cc + pad)
        self.flat = torch.full((off + n + 4,), float("nan"), device=dev)
        self.t = self.flat[off:off + n].view(N, H, W, Cc + pad)[..., :Cc]
        mask = torch.zeros(off + n + 4, dtype=torch.bool, device=dev)
        mask[off:off + n].view(N, H, W, Cc + pad)[..., :Cc] = True
        self.mask = mask
        if values is not None:
            self.t.copy_(values.to(dev))
            assert torch.equal(self.t.double(), values.to(dev).double()), "values not fp32-exact"

    def intact(self):
        rest = self.flat[~self.mask].view(torch.int32)
        return bool(torch.all(rest == NAN_BITS))


def assert_intact(what, *slots):
    for i, s in enumerate(slots):
        assert s.intact(), f"{what}: wrote outside the tensor (pad channels / guards of operand {i})"


def nan_like(t):
    return torch.full_like(t, float("nan"))


def vec_ok(C, tensors, lds, total4):
    """elementwise.cu vec_ok: C % 4 == 0, < 2^31 float4 items, 16-byte pointers, lds % 4 == 0."""
    return (C % 4 == 0 and total4 < 2 ** 31 and
            all(t is None or t.data_ptr() % 16 == 0 for t in tensors) and
            all(ld % 4 == 0 for ld in lds))


def res_vec_ok(C, a, y, scale, shift, res):
    """resnet.cu affine_res_act's vec_ok call: < 2^31 float4 items, the operands' pointers and
    pixel strides as in vec_ok."""
    npix = a.shape[0] * a.shape[1] * a.shape[2]
    lds = [ops._ld(a), ops._ld(y)] + ([] if res is None else [ops._ld(res)])
    return vec_ok(C, (a, y, scale, shift, res), lds, npix * C // 4)


def exp_vec(C, lay):
    pad, off = LAYOUTS[lay]
    return C % 4 == 0 and pad % 4 == 0 and off == 0


def path_cases(shapes, layouts=("dense", "ld4", "ld1", "off1"), max_scalar_c=None):
    """(shape, layout) pairs, named by the path they must take (max_scalar_c: the largest C the
    scalar path accepts)."""
    out = []
    for s in shapes:
        for lay in layouts:
            if s[3] % 4 and lay == "ld4":
                continue
            if max_scalar_c is not None and s[3] > max_scalar_c and not exp_vec(s[3], lay):
                continue
            out.append(pytest.param(s, lay, id=f"{'x'.join(map(str, s))}-{lay}-"
                                               f"{'f4' if exp_vec(s[3], lay) else 'scalar'}"))
    return out


# (N, H, W, C): H, W are the output size for the pool, the input size for the upsampling
EW_SHAPES = [(2, 5, 7, 1), (1, 3, 5, 3), (2, 4, 7, 5), (2, 3, 5, 12), (1, 5, 9, 24), (2, 3, 7, 48),
             (2, 6, 8, 4), (1, 5, 7, 16), (2, 3, 5, 32), (1, 3, 3, 1024)]
UP_SHAPES = EW_SHAPES + [(2, 1, 6, 12), (1, 7, 1, 3), (1, 1, 1, 32), (2, 1, 5, 4)]
BIG = (2, 128, 128, 64)
DATA = ("int", "randn")


def _f(x):
    return None if x is None else x.float()


def _d(x, dev):
    return None if x is None else x.float().to(dev)


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ----------------------------------------------------------------------------- float64 references
def interp_matrix(n, f, bilinear, dev="cpu"):
    """(n f, n) matrix of F.interpolate(size = n f, align_corners=False) along one axis."""
    M = torch.zeros(n * f, n, dtype=torch.float64)
    for o in range(n * f):
        if not bilinear:
            M[o, o // f] = 1.0
            continue
        s = max((o + 0.5) / f - 0.5, 0.0)
        i0 = int(math.floor(s))
        i1 = min(i0 + 1, n - 1)
        lam = s - i0
        M[o, i0] += 1.0 - lam
        M[o, i1] += lam
    return M.to(dev)


def resize_ref(x, f, bilinear=True):
    """NHWC float64 resize by the integer factor f (bilinear align_corners=False or nearest)."""
    Mh = interp_matrix(x.shape[1], f, bilinear, dev=x.device)
    Mw = interp_matrix(x.shape[2], f, bilinear, dev=x.device)
    return torch.einsum("oh,nhwc,pw->nopc", Mh, x, Mw)


def resize_adj_ref(dy, h, w, f, bilinear=True):
    Mh = interp_matrix(h, f, bilinear, dev=dy.device)
    Mw = interp_matrix(w, f, bilinear, dev=dy.device)
    return torch.einsum("oh,nopc,pw->nhwc", Mh, dy, Mw)


def pool_ref(x):
    """2x2 max pool of an NHWC tensor: (values, window index of the first maximum)."""
    N, H, W, Cc = x.shape
    win = x.view(N, H // 2, 2, W // 2, 2, Cc).permute(0, 1, 3, 5, 2, 4).reshape(N, H // 2, W // 2, Cc, 4)
    v, i = win.max(-1)
    first = (win == v.unsqueeze(-1)).double().argmax(-1)   # first of equal maxima
    return v, first


def unpool_ref(dp, first, H, W):
    N, Ho, Wo, Cc = dp.shape
    win = torch.zeros(N, Ho, Wo, Cc, 4, dtype=dp.dtype, device=dp.device)
    win.scatter_(-1, first.unsqueeze(-1), dp.unsqueeze(-1))
    return win.view(N, Ho, Wo, Cc, 2, 2).permute(0, 1, 4, 2, 5, 3).reshape(N, H, W, Cc)


def adam_ref(p, g, m, v, step, lr, b1, b2, eps, wd, gs=1.0, bc=None):
    """One step of torch.optim.Adam (L2 weight decay added to the gradient) in float64; bc:
    (1 - b1^step, 1 - b2^step) if given, else computed in float64."""
    bc1, bc2 = bc if bc is not None else (1 - b1 ** step, 1 - b2 ** step)
    gi = g * gs + wd * p
    m = b1 * m + (1 - b1) * gi
    v = b2 * v + (1 - b2) * gi * gi
    p = p - lr / bc1 * m / (v.sqrt() / math.sqrt(bc2) + eps)
    return p, m, v


def coord_grid(H, W, dev):
    """imcoordgrid: (HW, 2) float64, x = linspace(-1, 1, H) slowest, y = linspace(1, -1, W)."""
    gx = torch.linspace(-1, 1, H, dtype=torch.float64, device=dev) if H > 1 else \
        torch.full((1,), -1.0, dtype=torch.float64, device=dev)
    gy = torch.linspace(1, -1, W, dtype=torch.float64, device=dev) if W > 1 else \
        torch.full((1,), 1.0, dtype=torch.float64, device=dev)
    return torch.stack([gx.repeat_interleave(W), gy.repeat(H)], 1)


# ============================================================================= CPU reference checks
def test_references_match_torch():
    """The float64 helpers above against torch's own float64 operators on random data."""
    g = _gen("refs")
    for (n, h, w, c), f, bil in itertools.product([(2, 5, 7, 3), (1, 1, 4, 2), (1, 3, 1, 1)],
                                                  (2, 3, 4), (True, False)):
        x = torch.randn(n, h, w, c, generator=g, dtype=torch.float64)
        mode = dict(mode="bilinear", align_corners=False) if bil else dict(mode="nearest")
        xr = x.permute(0, 3, 1, 2).clone().requires_grad_(True)
        y = F.interpolate(xr, size=(h * f, w * f), **mode)
        assert torch.allclose(resize_ref(x, f, bil), y.permute(0, 2, 3, 1), atol=1e-12, rtol=0)
        dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
        y.backward(dy)
        got = resize_adj_ref(dy.permute(0, 2, 3, 1), h, w, f, bil)
        assert torch.allclose(got, xr.grad.permute(0, 2, 3, 1), atol=1e-12, rtol=0)
    # max pool with ties (integers): values and the first-maximum gradient routing
    x = torch.randint(-2, 3, (2, 6, 10, 5), generator=g).double()
    xr = x.permute(0, 3, 1, 2).clone().requires_grad_(True)
    y = F.max_pool2d(xr, 2, 2)
    v, first = pool_ref(x)
    assert torch.equal(v, y.detach().permute(0, 2, 3, 1))
    dp = torch.randn(y.shape, generator=g, dtype=torch.float64)
    y.backward(dp)
    assert torch.equal(unpool_ref(dp.permute(0, 2, 3, 1), first, 6, 10), xr.grad.permute(0, 2, 3, 1))
    assert int((first > 0).sum()) > 0 and bool((x.view(2, 3, 2, 5, 2, 5) == 2).any())
    # Adam recurrence
    for wd, gs in ((0.0, 1.0), (0.01, 0.5)):
        p0 = torch.randn(50, generator=g, dtype=torch.float64)
        grads = [torch.randn(50, generator=g, dtype=torch.float64) for _ in range(5)]
        p = p0.clone().requires_grad_(True)
        opt = torch.optim.Adam([p], lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=wd)
        q, m, vv = p0.clone(), torch.zeros(50, dtype=torch.float64), torch.zeros(50, dtype=torch.float64)
        for s, gr in enumerate(grads, 1):
            p.grad = gr * gs
            opt.step()
            q, m, vv = adam_ref(q, gr, m, vv, s, 1e-2, 0.9, 0.999, 1e-8, wd, gs)
            assert torch.allclose(q, p.detach(), atol=1e-13, rtol=0), (wd, gs, s)


def test_vec_predicates():
    """The Python mirrors of the dispatch predicates agree with the layout names."""
    for c, lay in itertools.product((1, 3, 4, 12, 32), LAYOUTS):
        pad, off = LAYOUTS[lay]
        buf = torch.zeros(off + 64 * (c + pad) + 4)   # CPU: data_ptr alignment as on the device
        t = buf[off:off + 64 * (c + pad)]
        ok = vec_ok(c, [t], [c + pad], 64 * c // 4) if buf.data_ptr() % 16 == 0 else None
        if ok is not None:
            assert ok == exp_vec(c, lay), (c, lay)


# ============================================================================= elementwise.cu
@gpu
@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("shape,lay", path_cases(EW_SHAPES) + path_cases([BIG], ("dense", "ld1")))
def test_affine(cuda, shape, lay, data):
    run_affine(cuda, shape, lay, data)
    if lay == "dense":
        run_affine(cuda, shape, lay, data, aff=False)
        run_affine(cuda, shape, lay, data, nchw=True)


def run_affine(dev, shape, lay, data, aff=True, nchw=False):
    g = _gen("affine", shape, data)
    N, H, W, Cc = shape
    a = vals(g, shape, data).to(dev)
    sc, sh = (bn_scale(g, Cc, data).to(dev), bn_shift(g, Cc, data).to(dev)) if aff else (None, None)
    ref = a * sc + sh if aff else a
    mag = (a * sc).abs() + sh.abs() if aff else a.abs()
    A = Slot(shape, dev, lay, a)
    what = f"affine {shape} {lay} {data} aff={aff} nchw={nchw}"
    if nchw:
        y = torch.full((N, Cc, H, W), float("nan"), device=dev)
        ops.affine(A.t, _f(sc), _f(sh), y, out_nchw=True)
        got = y.permute(0, 2, 3, 1)
        Y = None
    else:
        Y = Slot(shape, dev, lay)
        assert vec_ok(Cc, [A.t, Y.t, sc, sh], [ops._ld(A.t), ops._ld(Y.t)], N * H * W * Cc // 4) == \
            exp_vec(Cc, lay), what
        ops.affine(A.t, _f(sc), _f(sh), Y.t)
        got = Y.t
    torch.cuda.synchronize()
    expect(got, ref, mag, 1, data, what, grid_of(a) * 0.5)
    assert_intact(what, A, *( [Y] if Y else []))
    return got.clone()


@gpu
@pytest.mark.parametrize("shape", [s for s in EW_SHAPES + [BIG] if s[3] % 4 == 0],
                         ids=lambda s: "x".join(map(str, s)))
def test_float4_matches_scalar(cuda, shape):
    """Same data through the float4 and the scalar path: bitwise identical outputs."""
    for name, fn in (("affine", lambda lay: [run_affine(cuda, shape, lay, "randn")]),
                     ("add_slice", lambda lay: [run_add_slice(cuda, shape, lay, "randn", True)]),
                     ("pool fwd/bwd", lambda lay: run_pool(cuda, shape, lay, "randn")),
                     ("upsample bilinear fwd/bwd", lambda lay: run_upsample(cuda, shape, lay, "randn", True)),
                     ("upsample nearest fwd/bwd", lambda lay: run_upsample(cuda, shape, lay, "randn", False)),
                     ("affine_res_act", lambda lay: [run_affine_res_act(cuda, shape, lay, "randn", True, True)])):
        for f4, sc in zip(fn("dense"), fn("ld1")):
            same_bits(f4, sc, f"{name}: float4 vs scalar {shape}")
    if shape[3] <= 256:
        for combo in ((True, True, True, ACT_LRELU, True), (True, True, False, ACT_TANH, False),
                      (False, False, True, ACT_LRELU, True)):
            f4 = run_bn_act_bwd(cuda, shape, "dense", "randn", *combo)[0]
            sc = run_bn_act_bwd(cuda, shape, "ld1", "randn", *combo)[0]
            same_bits(f4, sc, f"bn_act_bwd dpre float4 vs scalar {shape} {combo}")


@gpu
@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("shape,lay", path_cases(EW_SHAPES) + path_cases([BIG], ("dense", "ld1")))
def test_add_slice(cuda, shape, lay, data):
    run_add_slice(cuda, shape, lay, data, False)
    run_add_slice(cuda, shape, lay, data, True)


def run_add_slice(dev, shape, lay, data, accumulate):
    g = _gen("add_slice", shape, data)
    s = vals(g, shape, data).to(dev)
    prior = vals(g, shape, data).to(dev)
    S = Slot(shape, dev, lay, s)
    D = Slot(shape, dev, lay, prior if accumulate else None)
    ops.add_slice(S.t, D.t, accumulate)
    torch.cuda.synchronize()
    what = f"add_slice {shape} {lay} {data} acc={accumulate}"
    ref = s + prior if accumulate else s
    expect(D.t, ref, s.abs() + (prior.abs() if accumulate else 0), 1, data, what, 1.0)
    assert_intact(what, S, D)
    return D.t.clone()


# ----------------------------------------------------------------------------- pooling
@gpu
@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("shape,lay", path_cases(EW_SHAPES) + path_cases([(2, 96, 96, 64)], ("dense", "ld1")))
def test_pool(cuda, shape, lay, data):
    run_pool(cuda, shape, lay, data)
    run_pool(cuda, shape, lay, data, aff=False, accumulate=False)
    if ops.pool_bwd_stats_ok(shape[3]) and exp_vec(shape[3], lay):
        run_pool(cuda, shape, lay, data, stats=True)
        run_pool(cuda, shape, lay, data, aff=False, accumulate=False, stats=True)


def run_pool(dev, shape, lay, data, aff=True, accumulate=True, stats=False):
    """shape: the pooled (N, Ho, Wo, C).  Forward and backward (optionally with the fused
    BatchNorm-backward statistics of the full-resolution gradient)."""
    g = _gen("pool", shape, data)
    N, Ho, Wo, Cc = shape
    full = (N, 2 * Ho, 2 * Wo, Cc)
    a = vals(g, full, data, amp=2).to(dev)
    sc, sh = (bn_scale(g, Cc, data).to(dev), bn_shift(g, Cc, data).to(dev)) if aff else (None, None)
    dp = vals(g, shape, data).to(dev)
    prior = vals(g, full, data).to(dev) if accumulate else torch.zeros(full, dtype=torch.float64, device=dev)
    what = f"pool {shape} {lay} {data} aff={aff} acc={accumulate} stats={stats}"
    A = Slot(full, dev, lay, a)
    Y = Slot(shape, dev, lay)
    ops.pool_fwd(A.t, _f(sc), _f(sh), Y.t)
    af = (a * sc + sh).float().double() if aff else a     # fmaf: one rounding, as compared
    ref_y, first = pool_ref(af)
    torch.cuda.synchronize()
    expect(Y.t, ref_y, ref_y.abs(), 1, data, what + " fwd", 1.0 / 16)
    DP = Slot(shape, dev, lay, dp)
    DF = Slot(full, dev, lay, prior if accumulate else None)
    mean = invstd = sums = None
    if stats:
        mean = bn_shift(g, Cc, data).to(dev)
        invstd = (bn_scale(g, Cc, data).abs() if data == "int" else normal(g, (Cc,)).abs() + 0.5).to(dev)
        sums0 = ints(g, (2 * Cc,), 5).to(dev)
        sums = sums0.clone()
    ops.pool_bwd(DP.t, A.t, _f(sc), _f(sh), DF.t, accumulate, _f(mean), _f(invstd), sums)
    torch.cuda.synchronize()
    ref_df = prior + unpool_ref(dp, first, 2 * Ho, 2 * Wo)
    expect(DF.t, ref_df, ref_df.abs() + prior.abs(), 1, data, what + " bwd", 1.0)
    assert_intact(what, A, Y, DP, DF)
    if stats:
        t = DF.t.double()       # the fp32 gradient the statistics are formed from
        xh = (a - mean) * invstd
        red = t.reshape(-1, Cc)
        s1 = sums0[:Cc] + red.sum(0)
        s2 = sums0[Cc:] + (red * xh.reshape(-1, Cc)).sum(0)
        # per channel: fp32 per-thread sums, a CTA sum of 256/C4 rows, an ordered double sum
        k = N * 4 * Ho * Wo + 260    # per-thread fp32 sums, a CTA sum, the ordered double sum
        m1 = red.abs().sum(0)
        m2 = (red * xh.reshape(-1, Cc)).abs().sum(0) + \
            (red.abs() * ((a.abs() + mean.abs()) * invstd).reshape(-1, Cc)).sum(0) * 4 / max(k, 1)
        unit2 = grid_of(t) * grid_of(xh) if data == "int" else None
        expect(sums[:Cc] - sums0[:Cc], s1 - sums0[:Cc], m1, k, data, what + " sum dy", 1.0)
        expect(sums[Cc:] - sums0[Cc:], s2 - sums0[Cc:], m2, k, data, what + " sum dy*xh", unit2)
        sums_b = sums0.clone()
        DF2 = Slot(full, dev, lay, prior if accumulate else None)
        ops.pool_bwd(DP.t, A.t, _f(sc), _f(sh), DF2.t, accumulate, _f(mean), _f(invstd), sums_b)
        torch.cuda.synchronize()
        same_bits(sums, sums_b, what + " statistics reproducible")
    return Y.t.clone(), DF.t.clone()


# ----------------------------------------------------------------------------- x2 upsampling
@gpu
@pytest.mark.parametrize("bilinear", (True, False), ids=("bilinear", "nearest"))
@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("shape,lay", path_cases(UP_SHAPES) + path_cases([BIG], ("dense", "ld1")))
def test_upsample(cuda, shape, lay, data, bilinear):
    run_upsample(cuda, shape, lay, data, bilinear)


def run_upsample(dev, shape, lay, data, bilinear):
    """shape: the low-resolution (N, h, w, C)."""
    g = _gen("upsample", shape, data)
    N, h, w, Cc = shape
    hi = (N, 2 * h, 2 * w, Cc)
    x = vals(g, shape, data).to(dev)
    dy = vals(g, hi, data).to(dev)
    what = f"upsample {'bilinear' if bilinear else 'nearest'} {shape} {lay} {data}"
    X = Slot(shape, dev, lay, x)
    Y = Slot(hi, dev, lay)
    ops.upsample_fwd(X.t, Y.t, bilinear)
    DY = Slot(hi, dev, lay, dy)
    DX = Slot(shape, dev, lay)
    ops.upsample_bwd(DY.t, DX.t, bilinear)
    torch.cuda.synchronize()
    ref = resize_ref(x, 2, bilinear)
    # (1-lh)((1-lw)a + lw b) + lh(...): 3 roundings per level, 2 levels + final add
    expect(Y.t, ref, resize_ref(x.abs(), 2, bilinear), 6, data, what + " fwd", 1.0 / 16)
    ref_dx = resize_adj_ref(dy, h, w, 2, bilinear)
    expect(DX.t, ref_dx, resize_adj_ref(dy.abs(), h, w, 2, bilinear), 10, data, what + " bwd", 1.0 / 16)
    assert_intact(what, X, Y, DY, DX)
    return Y.t.clone(), DX.t.clone()


# ----------------------------------------------------------------------------- BatchNorm
BN_SHAPES = [(1, 3, 5, 1), (1, 3, 5, 3), (2, 3, 5, 5), (2, 3, 5, 12), (1, 5, 9, 24), (2, 3, 7, 48),
             (2, 4, 6, 4), (1, 5, 7, 16), (2, 3, 5, 32), (1, 3, 3, 1024), (2, 3, 3, 255),
             (2, 3, 3, 256), (1, 2, 2, 64)]


@gpu
@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("shape,lay", path_cases(BN_SHAPES, max_scalar_c=256) +
                         path_cases([BIG], ("dense", "ld1")))
def test_bn_bwd_reduce(cuda, shape, lay, data):
    g = _gen("bn_bwd_reduce", shape, data)
    N, H, W, Cc = shape
    dy, a = vals(g, shape, data).to(cuda), vals(g, shape, data).to(cuda)
    mean = bn_shift(g, Cc, data).to(cuda)
    invstd = (bn_scale(g, Cc, "int").abs() if data == "int" else normal(g, (Cc,)).abs() + 0.5).to(cuda)
    sums0 = ints(g, (2 * Cc,), 5).to(cuda)
    DY, A = Slot(shape, cuda, lay, dy), Slot(shape, cuda, lay, a)
    runs = []
    for _ in range(2):
        s = sums0.clone()
        ops.bn_bwd_reduce(DY.t, A.t, _f(mean), _f(invstd), s)
        runs.append(s)
    torch.cuda.synchronize()
    what = f"bn_bwd_reduce {shape} {lay} {data}"
    same_bits(runs[0], runs[1], what + " reproducible")
    xh = (a - mean) * invstd
    d2, x2 = dy.reshape(-1, Cc), xh.reshape(-1, Cc)
    npix = N * H * W
    k = npix + 256 + 8          # sequential per-thread fp32 sums, a CTA sum, the ordered double sum
    got = runs[0] - sums0
    expect(got[:Cc], d2.sum(0), d2.abs().sum(0), k, data, what + " sum dy", 1.0)
    m2 = (d2 * x2).abs().sum(0) + (d2.abs() * ((a.abs() + mean.abs()) * invstd).reshape(-1, Cc)).sum(0) * 3 / k
    expect(got[Cc:], (d2 * x2).sum(0), m2, k, data, what + " sum dy*xh", grid_of(dy) * grid_of(xh))
    assert_intact(what, DY, A)


BN_ACT_COMBOS = list(itertools.product((True, False), (True, False), (True, False),
                                       (ACT_LRELU, ACT_TANH), (True, False)))


@gpu
@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("shape,lay", path_cases(BN_SHAPES, max_scalar_c=256) +
                         path_cases([BIG], ("dense", "ld1")))
def test_bn_act_bwd(cuda, shape, lay, data):
    """Every combination of BN on/off, extra on/off, dy present/None, LeakyReLU/tanh, dbias."""
    combos = BN_ACT_COMBOS if shape != BIG else BN_ACT_COMBOS[:2]
    for bn, extra, has_dy, act, dbias in combos:
        run_bn_act_bwd(cuda, shape, lay, data, bn, extra, has_dy, act, dbias)


def run_bn_act_bwd(dev, shape, lay, data, bn, extra, has_dy, act, dbias):
    g = _gen("bn_act_bwd", shape, data, bn, extra, has_dy, act)
    N, H, W, Cc = shape
    npix = N * H * W
    slope = 0.25 if data == "int" else 0.1
    amp = 1 if npix > 4096 else 3          # keeps the large case's dbias sums exact
    what = (f"bn_act_bwd {shape} {lay} {data} bn={bn} extra={extra} dy={has_dy} "
            f"act={'tanh' if act == ACT_TANH else 'lrelu'} dbias={dbias}")
    if act == ACT_TANH:
        a = (ints(g, shape, 1) if data == "int" else torch.tanh(normal(g, shape)).float().double())
    else:
        a = vals(g, shape, data, amp)
    a = a.to(dev)
    dy = vals(g, shape, data, amp).to(dev) if has_dy else torch.zeros(shape, dtype=torch.float64, device=dev)
    ex = vals(g, shape, data, amp).to(dev) if extra else torch.zeros(shape, dtype=torch.float64, device=dev)
    gamma = bn_scale(g, Cc, data).to(dev)
    if data == "int":
        # formula reference on exact operands: mean / invstd / sums chosen on the grid
        mean = bn_shift(g, Cc, data).to(dev)
        invstd = bn_scale(g, Cc, "int").abs().to(dev)
        count = 64.0
        k1 = (ints(g, (Cc,), 2) * 0.5).to(dev)
        k2 = (ints(g, (Cc,), 2) * 0.5).to(dev)
        sums = torch.cat([k1, k2]) * count
        scale = gamma
    else:
        # the statistics of `a` as BatchNorm2d would use them (fp32-rounded where the kernel
        # receives fp32), and the BN-backward sums of dy
        a2 = a.reshape(-1, Cc)
        mean64 = a2.mean(0)
        var = a2.var(0, unbiased=False)
        inv64 = 1.0 / torch.sqrt(var + 1e-5)
        mean, invstd = mean64.float().double(), inv64.float().double()
        scale = (gamma * invstd).float().double()
        count = float(npix)
        xh_k = (a - mean) * invstd
        sums = torch.cat([dy.reshape(-1, Cc).sum(0), (dy * xh_k).reshape(-1, Cc).sum(0)])
        k1, k2 = sums[:Cc] / count, sums[Cc:] / count
    if not bn:
        k1 = k2 = torch.zeros(Cc, dtype=torch.float64, device=dev)
    dact = (1 - a * a) if act == ACT_TANH else torch.where(a > 0, torch.ones_like(a), torch.full_like(a, slope))
    if data == "int" or not bn:
        gb = scale * (dy - k1 - (a - mean) * invstd * k2) if bn else dy
        ref = (gb + ex) * dact + ex
    else:
        # autograd through act and BatchNorm2d: L = <dy, BN(a)> + <ex, a> + <ex, pre>, a = act(pre)
        pre = (torch.atanh(a) if act == ACT_TANH else torch.where(a > 0, a, a / slope)).clone().requires_grad_(True)
        av = torch.tanh(pre) if act == ACT_TANH else F.leaky_relu(pre, slope)
        bnout = F.batch_norm(av.permute(0, 3, 1, 2), None, None, gamma, None, training=True, eps=1e-5)
        L = (bnout.permute(0, 2, 3, 1) * dy).sum() + (ex * av).sum() + (ex * pre).sum()
        L.backward()
        ref = pre.grad
    xhm = (a.abs() + mean.abs()) * invstd.abs()
    gm = scale.abs() * (dy.abs() + k1.abs() + xhm * k2.abs()) if bn else dy.abs()
    mag = (gm + ex.abs()) * (dact.abs() + (2 * a.abs() * a.abs() if act == ACT_TANH else 0)) + ex.abs()
    # roundings: mean, invstd, scale, k1, k2 as fp32 inputs; a - m, * is, * k2, g - k1, - , * sc,
    # + ex, * act', + ex; tanh's 1 - a*a: 2 more
    k = 18 if bn else 5
    A = Slot(shape, dev, lay, a)
    DY = Slot(shape, dev, lay, dy) if has_dy else None
    EX = Slot(shape, dev, lay, ex) if extra else None
    D = Slot(shape, dev, lay)
    db0 = ints(g, (Cc,), 5).to(dev)
    dbs = []
    for _ in range(2 if dbias else 1):
        db = db0.clone() if dbias else None
        ops.bn_act_bwd(DY.t if DY else None, A.t, _f(mean) if bn else None, _f(invstd) if bn else None,
                       _f(scale) if bn else None, sums if bn else None, count,
                       EX.t if EX else None, act, slope, D.t, db)
        dbs.append(db)
    torch.cuda.synchronize()
    got = D.t.clone()
    expect(got, ref, mag, k, data, what, 1.0 / 1024 if data == "int" else None)
    if dbias:
        same_bits(dbs[0], dbs[1], what + " dbias reproducible")
        d2 = got.double().reshape(-1, Cc)
        kd = npix + 256 + 8
        expect(dbs[0] - db0, d2.sum(0), d2.abs().sum(0), kd, data, what + " dbias",
               grid_of(d2) if data == "int" else None)
    assert_intact(what, *[s for s in (A, DY, EX, D) if s is not None])
    return got, (dbs[0] if dbias else None)


@gpu
def test_bn_finalize(cuda):
    g = _gen("bn_finalize")
    for Cc, count, training, affine, running, momentum in (
            (7, 1.0, True, True, True, 0.1), (33, 48.0, True, True, True, 0.25),
            (33, 1000.0, True, False, True, 0.1), (5, 10.0, True, True, False, 0.1),
            (300, 7.0, False, True, True, 0.1), (8, 3.0, False, False, True, 0.1)):
        what = f"bn_finalize C={Cc} count={count} training={training} affine={affine}"
        x = normal(g, (int(max(count, 1)) if count < 100 else 100, Cc)) + 0.5
        stats = torch.cat([x.sum(0) * count / x.shape[0], (x * x).sum(0) * count / x.shape[0]]).to(cuda)
        gamma = normal(g, (Cc,)).float().to(cuda) if affine else None
        beta = normal(g, (Cc,)).float().to(cuda) if affine else None
        rm0, rv0 = normal(g, (Cc,)).float().to(cuda), (normal(g, (Cc,)).abs() + 0.1).float().to(cuda)
        rm, rv = (rm0.clone(), rv0.clone()) if running else (None, None)
        outs = [torch.full((Cc,), float("nan"), device=cuda) for _ in range(4)]
        eps = 1e-5
        ops.bn_finalize(stats, count, gamma, beta, rm, rv, momentum, eps, training, outs[0], outs[1],
                        outs[2], outs[3])
        torch.cuda.synchronize()
        m = stats[:Cc] / count
        vb = (stats[Cc:] / count - m * m).clamp_min(0)
        if training:
            mean, var = m.float().double(), vb.float().double()
        else:
            mean, var = rm0.double(), rv0.double()
        invstd = 1.0 / torch.sqrt(var + eps)
        gm = gamma.double() if affine else torch.ones_like(mean)
        bt = beta.double() if affine else torch.zeros_like(mean)
        expect(outs[2], mean, mean.abs() + (m.abs() if training else 0), 1, "randn", what + " mean")
        expect(outs[3], invstd, invstd, 4, "randn", what + " invstd")
        expect(outs[0], gm * invstd, (gm * invstd).abs(), 6, "randn", what + " scale")
        expect(outs[1], bt - mean * gm * invstd, bt.abs() + (mean * gm * invstd).abs(), 10, "randn",
               what + " shift")
        if running and training:
            unb = vb * count / (count - 1) if count > 1 else vb
            erm = (1 - momentum) * rm0.double() + momentum * mean
            erv = (1 - momentum) * rv0.double() + momentum * unb
            expect(rm, erm, erm.abs() + rm0.double().abs() + mean.abs(), 4, "randn", what + " running_mean")
            expect(rv, erv, erv.abs() + rv0.double().abs() + unb.abs(), 5, "randn", what + " running_var")
        elif running:
            assert torch.equal(rm, rm0) and torch.equal(rv, rv0), what + ": eval changed running stats"


# ----------------------------------------------------------------------------- DilatedBlock sum
@gpu
@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("shape", [(2, 3, 5, 3), (1, 4, 6, 16), BIG], ids=lambda s: "x".join(map(str, s)))
def test_dilated_sum(cuda, shape, data):
    """Sum over every sub-module output of the DilatedBlock (conv output, LeakyReLU output and,
    with BatchNorm, the BN output) for 1 to 8 layers."""
    g = _gen("dilated", shape, data)
    Cc = shape[3]
    slope = 0.25 if data == "int" else 0.1
    layers_all = []
    for _ in range(8):
        pre = vals(g, shape, data).to(cuda)
        a = F.leaky_relu(pre, slope)
        if data != "int":
            a = a.float().double()
            pre = torch.where(a > 0, a, a / slope)
        layers_all.append((pre, a, bn_scale(g, Cc, data).to(cuda), bn_shift(g, Cc, data).to(cuda)))
    for nl, bn in itertools.product(range(1, 9) if shape != BIG else (1, 8), (False, True)):
        ls = layers_all[:nl]
        out = torch.full(shape, float("nan"), device=cuda)
        ops.dilated_sum([a.float() for _, a, _, _ in ls], [_f(s) if bn else None for *_, s, _ in ls],
                        [_f(t) if bn else None for *_, t in ls], slope, out)
        torch.cuda.synchronize()
        ref = sum(pre + a + (a * s + t if bn else 0) for pre, a, s, t in ls)
        mag = sum(pre.abs() + a.abs() + ((a * s).abs() + t.abs() if bn else 0) for pre, a, s, t in ls)
        expect(out, ref, mag, 4 * nl, data, f"dilated_sum {shape} {data} layers={nl} bn={bn}", 1.0 / 8)


# ----------------------------------------------------------------------------- losses
def ce_budget(l, y):
    """Per-pixel bound of ce_kernel's loss term and per-element bound of its gradient, with
    __expf / __logf: ex2.approx after x*log2(e) (relative error (2 + |x|) 2^-23 for x = l - m),
    __logf absolute error <= 2^-21 on [1, C], C-term fp32 sums."""
    m = l.max(-1, keepdim=True).values
    e = torch.exp(l - m)
    s = e.sum(-1, keepdim=True)
    C_ = l.shape[-1]
    rel_e = (2 + (l - m).abs()) * 2 ** -23
    ds = (e * rel_e).sum(-1, keepdim=True) + C_ * U * s
    lse = m + torch.log(s)
    ly = l.gather(-1, y.unsqueeze(-1))
    loss_b = 2 ** -21 + ds / s + 4 * U * (m.abs() + lse.abs() + ly.abs())
    pr = e / s
    grad_b = pr * (rel_e + ds / s + 4 * U) + 2 * U
    return loss_b.squeeze(-1), grad_b


@gpu
@pytest.mark.parametrize("shape,lay", [pytest.param((2, 5, 7, 3), "dense", id="2x5x7x3-dense"),
                                       pytest.param((1, 3, 5, 12), "ld1", id="1x3x5x12-ld1"),
                                       pytest.param((2, 96, 96, 4), "ld4", id="2x96x96x4-ld4")])
def test_ce(cuda, shape, lay):
    g = _gen("ce", shape)
    N, H, W, Cc = shape
    l = (normal(g, shape) * 3).float().double()
    l.view(-1)[::7] = 80.0
    l.view(-1)[3::11] = -80.0
    l = l.to(cuda)
    y = torch.randint(0, Cc, (N, H, W), generator=g).to(cuda)
    L = Slot(shape, cuda, lay, l)
    gscale = 0.75
    outs = []
    for _ in range(2):
        loss = torch.full((1,), 2.5, dtype=torch.float64, device=cuda)
        D = Slot(shape, cuda, lay)
        ops.ce_fwd_bwd(L.t, y, loss, D.t, gscale)
        outs.append((loss, D))
    torch.cuda.synchronize()
    what = f"ce {shape} {lay}"
    same_bits(outs[0][0], outs[1][0], what + " loss reproducible")
    same_bits(outs[0][1].t, outs[1][1].t, what + " dlogits reproducible")
    lp = torch.log_softmax(l, -1)
    per = -lp.gather(-1, y.unsqueeze(-1)).squeeze(-1)
    lb, gb = ce_budget(l, y)
    npix = N * H * W
    iters = -(-npix // (min(-(-npix // 256), 8 * sm_count()) * 256))
    tot_b = float(lb.sum()) + (iters + 12) * U * float(per.abs().sum())
    err = abs(float(outs[0][0]) - 2.5 - float(per.sum()))
    assert err <= tot_b, f"{what}: loss error {err} > budget {tot_b}"
    ref_d = (lp.exp() - F.one_hot(y, Cc).double()) * gscale
    err_d = (outs[0][1].t.double() - ref_d).abs()
    assert bool((err_d <= gb * gscale).all()), f"{what}: dlogits {float((err_d / (gb * gscale)).max())} x budget"
    assert_intact(what, L, outs[0][1])


def bce_budget(x, t):
    e = torch.exp(-x.abs())
    rel_e = (2 + x.abs()) * 2 ** -23
    loss_b = 4 * U * (x.clamp_min(0) + (x * t).abs() + torch.log1p(e)) + e * rel_e + 2 * U * torch.log1p(e)
    sig = torch.sigmoid(x)
    grad_b = sig * ((2 + x.abs()) * 2 ** -23 + 4 * U) + 2 * U * (sig - t).abs()
    return loss_b, grad_b


@gpu
@pytest.mark.parametrize("n", (1, 1000, 600_000))
@pytest.mark.parametrize("kind,data", [(0, "int"), (0, "randn"), (1, "randn")],
                         ids=("mse-int", "mse-randn", "bce-randn"))
def test_pointwise_loss_and_sqerr(cuda, n, kind, data):
    """BCE uses __expf / __logf: normal tier only."""
    g = _gen("pointwise", n, kind, data)
    x = vals(g, (n,), data)
    if kind == 1:
        x = x * 4
        x[::5] = 80.0
        x[2::7] = -80.0
    t = vals(g, (n,), data) if kind == 0 else torch.rand(n, generator=g).double().float().double()
    x, t = x.to(cuda), t.to(cuda)
    gscale = 0.5
    what = f"pointwise kind={kind} n={n} {data}"
    runs = []
    for _ in range(2):
        loss = torch.full((1,), 1.5, dtype=torch.float64, device=cuda)
        d = torch.full((n,), float("nan"), device=cuda)
        ops.pointwise_loss(x.float(), t.float(), kind, loss, d, gscale)
        runs.append((loss, d))
    torch.cuda.synchronize()
    same_bits(runs[0][0], runs[1][0], what + " loss reproducible")
    iters = -(-n // (min(-(-n // 256), 8 * sm_count()) * 256))
    if kind == 0:
        dd = x - t
        per, ref_d = dd * dd, 2 * dd * gscale
        expect(runs[0][0] - 1.5, per.sum().view(1), per.abs().sum().view(1), iters + 12, data,
               what + " loss", grid_of(dd) ** 2 if data == "int" else None)
        expect(runs[0][1], ref_d, 2 * dd.abs() * gscale, 3, data, what + " dpred", 1.0 / 4)
    else:
        per = F.binary_cross_entropy_with_logits(x, t, reduction="none")
        lb, gb = bce_budget(x, t)
        tot_b = float(lb.sum()) + (iters + 12) * U * float(per.abs().sum())
        err = abs(float(runs[0][0]) - 1.5 - float(per.sum()))
        assert err <= tot_b, f"{what}: loss error {err} > budget {tot_b}"
        err_d = (runs[0][1].double() - (torch.sigmoid(x) - t) * gscale).abs()
        assert bool((err_d <= gb * gscale + 1e-30).all()), f"{what}: dpred outside its budget"
    # sqerr_reduce: 0.5 sum (xhat - x)^2 and dxhat = (xhat - x) gscale
    sq = []
    for _ in range(2):
        out = torch.full((1,), -2.0, dtype=torch.float64, device=cuda)
        dx = torch.full((n,), float("nan"), device=cuda)
        ops.sqerr_reduce(t.float(), x.float(), out, dx, gscale)
        sq.append((out, dx))
    torch.cuda.synchronize()
    same_bits(sq[0][0], sq[1][0], what + " sqerr reproducible")
    dd = x - t
    expect(sq[0][0] + 2.0, (0.5 * dd * dd).sum().view(1), (0.5 * dd * dd).sum().view(1), iters + 12,
           data, what + " sqerr", grid_of(dd) ** 2 / 2 if data == "int" else None)
    expect(sq[0][1], dd * gscale, dd.abs() * gscale, 2, data, what + " sqerr dxhat", 1.0 / 2)


# ----------------------------------------------------------------------------- Adam
@gpu
@pytest.mark.parametrize("wd,gs", [(0.0, 1.0), (0.01, 1.0), (0.0, 0.25), (0.05, 2.0)])
def test_adam_multi(cuda, wd, gs):
    g = _gen("adam", wd, gs)
    sizes = (1, 1000, 70_001)
    # the kernel receives fp32 hyper-parameters
    lr, b1, b2, eps, wd, gs = (float(np.float32(v)) for v in (1e-2, 0.9, 0.999, 1e-8, wd, gs))
    ps = [normal(g, (n,)).float().to(cuda) for n in sizes]
    gr = [torch.zeros(n, device=cuda) for n in sizes]
    ms = [torch.zeros(n, device=cuda) for n in sizes]
    vs = [torch.zeros(n, device=cuda) for n in sizes]
    tab = torch.tensor([[p.data_ptr(), q.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel()]
                        for p, q, m, v in zip(ps, gr, ms, vs)], dtype=torch.int64, device=cuda)
    for step in range(1, 6):
        for q in gr:
            q.copy_(normal(g, q.shape))
        before = [(p.double(), m.double(), v.double()) for p, m, v in zip(ps, ms, vs)]
        ops.adam_multi(tab, len(ps), max(sizes), lr, b1, b2, eps, wd, step, gs)
        torch.cuda.synchronize()
        # the host computes the bias corrections in fp32 with powf
        bc1 = float(np.float32(1) - np.power(np.float32(b1), np.float32(step)))
        bc2 = float(np.float32(1) - np.power(np.float32(b2), np.float32(step)))
        for (p0, m0, v0), p, q, m, v in zip(before, ps, gr, ms, vs):
            what = f"adam n={p.numel()} step={step} wd={wd} gs={gs}"
            q64 = q.double()
            gim = (q64 * gs).abs() + (wd * p0).abs()
            _, m64, v64 = adam_ref(p0, q64, m0, v0, step, lr, b1, b2, eps, wd, gs, (bc1, bc2))
            # g*gs, fma(wd, p, .), b1*m, (1-b1)*g, + (1 - b1 is exact in fp32)
            expect(m, m64, b1 * m0.abs() + (1 - b1) * gim, 8, "randn", what + " exp_avg")
            expect(v, v64, b2 * v0.abs() + (1 - b2) * gim * gim, 10, "randn", what + " exp_avg_sq")
            # the parameter from the kernel's own (m, v): roundings of lr/bc1, sqrt, /sqrt(bc2),
            # + eps, m/denom, step*, p - u
            mk, vk = m.double(), v.double()
            u = lr / bc1 * mk / (vk.sqrt() / math.sqrt(bc2) + eps)
            expect(p, p0 - u, p0.abs() + 8 * u.abs(), 8, "randn", what + " param")


# ----------------------------------------------------------------------------- transpose
@gpu
@pytest.mark.parametrize("N,R,Cc", [(1, 1, 1), (2, 33, 17), (3, 64, 32), (1, 5, 100)])
def test_transpose(cuda, N, R, Cc):
    x = torch.randn(N, R, Cc, device=cuda)
    y = torch.full((N, Cc, R), float("nan"), device=cuda)
    ops.transpose(x, y, N, R, Cc)
    torch.cuda.synchronize()
    assert torch.equal(y, x.transpose(1, 2))


# ============================================================================= resnet.cu
@gpu
@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("shape,lay", path_cases(EW_SHAPES) + path_cases([BIG], ("dense", "ld1")))
def test_affine_res_act(cuda, shape, lay, data):
    for aff, res in ((True, True), (True, False), (False, True), (False, False)):
        run_affine_res_act(cuda, shape, lay, data, aff, res)
    run_lrelu_mask_bwd(cuda, shape, lay, data)


def run_affine_res_act(dev, shape, lay, data, aff, res):
    g = _gen("affine_res_act", shape, data)
    Cc = shape[3]
    slope = 0.25 if data == "int" else 0.1
    a = vals(g, shape, data).to(dev)
    r = vals(g, shape, data).to(dev)
    sc, sh = (bn_scale(g, Cc, data).to(dev), bn_shift(g, Cc, data).to(dev)) if aff else (None, None)
    A, Y = Slot(shape, dev, lay, a), Slot(shape, dev, lay)
    R = Slot(shape, dev, lay, r) if res else None
    what = f"affine_res_act {shape} {lay} {data} aff={aff} res={res}"
    assert res_vec_ok(Cc, A.t, Y.t, sc, sh, R.t if R else None) == exp_vec(Cc, lay), what
    ops.affine_res_act(A.t, _f(sc), _f(sh), R.t if R else None, slope, Y.t)
    torch.cuda.synchronize()
    v = (a * sc + sh if aff else a) + (r if res else 0)
    mag = ((a * sc).abs() + sh.abs() if aff else a.abs()) + (r.abs() if res else 0)
    expect(Y.t, F.leaky_relu(v, slope), mag, 3, data, what, 1.0 / 8)
    assert_intact(what, *[s for s in (A, Y, R) if s is not None])
    return Y.t.clone()


def run_lrelu_mask_bwd(dev, shape, lay, data):
    g = _gen("lrelu_mask_bwd", shape, data)
    slope = 0.25 if data == "int" else 0.1
    dy, y = vals(g, shape, data).to(dev), vals(g, shape, data).to(dev)
    DY, Y, G = Slot(shape, dev, lay, dy), Slot(shape, dev, lay, y), Slot(shape, dev, lay)
    ops.lrelu_mask_bwd(DY.t, Y.t, slope, G.t)
    torch.cuda.synchronize()
    what = f"lrelu_mask_bwd {shape} {lay} {data}"
    expect(G.t, torch.where(y > 0, dy, dy * slope), dy.abs(), 1, data, what, 1.0 / 4)
    assert_intact(what, DY, Y, G)


RESIZE_SHAPES = [(2, 3, 5, 1), (1, 1, 4, 3), (2, 4, 1, 2), (1, 1, 1, 5), (2, 3, 3, 4), (1, 5, 7, 16),
                 (2, 96, 96, 3)]


@gpu
@pytest.mark.parametrize("bilinear", (True, False), ids=("bilinear", "nearest"))
@pytest.mark.parametrize("f,data", [(2, "int"), (4, "int"), (2, "randn"), (3, "randn")])
@pytest.mark.parametrize("shape", RESIZE_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("lay", ("dense", "ld1"))
def test_resize(cuda, shape, f, data, bilinear, lay):
    g = _gen("resize", shape, f, data)
    N, h, w, Cc = shape
    hi = (N, h * f, w * f, Cc)
    x, dy = vals(g, shape, data).to(cuda), vals(g, hi, data).to(cuda)
    X, Y, DY = Slot(shape, cuda, lay, x), Slot(hi, cuda, lay), Slot(hi, cuda, lay, dy)
    DX = Slot(shape, cuda, lay, torch.zeros(shape, dtype=torch.float64))    # the kernel adds
    ops.resize_fwd(X.t, Y.t, f, bilinear)
    ops.resize_bwd(DY.t, DX.t, f, bilinear)
    torch.cuda.synchronize()
    what = f"resize x{f} {'bilinear' if bilinear else 'nearest'} {shape} {lay} {data}"
    # bil_src forms the source coordinate with 1/f in fp32 (ATen: in/out): for f = 3 an error of
    # up to 3 2^-24 (|s| + 1) in the weight, and a source index that may move to the neighbour
    # (weight ~1 - 2^-22 instead of 0), so the magnitude takes the 3x3 neighbourhood maximum
    kc = 6 if f in (2, 4) else 6 + 6 * (max(h, w) + 1)
    xm = x.abs() if f in (2, 4) else \
        F.max_pool2d(x.abs().permute(0, 3, 1, 2), 3, 1, 1).permute(0, 2, 3, 1)
    expect(Y.t, resize_ref(x, f, bilinear), resize_ref(xm, f, bilinear), kc, data, what + " fwd",
           1.0 / 64)
    # adjoint: float atomics in any order, up to (f + 1)^2 contributions per element
    dym = dy.abs() if f in (2, 4) else \
        F.max_pool2d(dy.abs().permute(0, 3, 1, 2), 2 * f + 1, 1, f).permute(0, 2, 3, 1)
    expect(DX.t, resize_adj_ref(dy, h, w, f, bilinear), resize_adj_ref(dym, h, w, f, bilinear),
           kc + 3 * (2 * f) ** 2, data, what + " bwd", 1.0 / 64)
    assert_intact(what, X, Y, DY, DX)


# ============================================================================= mobilenet.cu
@gpu
@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("pooled", (False, True), ids=("dense", "pooled"))
@pytest.mark.parametrize("shape,lay", [pytest.param(s, l, id=f"{'x'.join(map(str, s))}-{l}")
                                       for s, l in [((2, 4, 4, 3), "dense"), ((1, 4, 4, 32), "ld1"),
                                                    ((2, 2, 8, 40), "off1"), ((2, 4, 4, 96), "dense"),
                                                    ((3, 16, 16, 64), "ld4"), (BIG, "dense")]])
def test_relu6_bwd_reduce(cuda, shape, lay, pooled, data):
    """g = dy * [0 < a*scale + shift < 6] and the BN-backward sums of g; pooled: dy is the (N, C)
    gradient of AdaptiveAvgPool2d(1), spread over H*W.  Integer data lands exactly on 0 and 6."""
    g = _gen("relu6", shape, pooled, data)
    N, H, W, Cc = shape
    a = (ints(g, shape, 4) + 2 if data == "int" else (normal(g, shape) * 3 + 2).float().double()).to(cuda)
    sc = (torch.ones(Cc).double() if data == "int" else normal(g, (Cc,))).to(cuda)
    sc[: Cc // 2] = bn_scale(g, Cc // 2, data).to(cuda)
    sh = (torch.zeros(Cc).double() if data == "int" else normal(g, (Cc,))).to(cuda)
    mean = bn_shift(g, Cc, data).to(cuda)
    invstd = (bn_scale(g, Cc, "int").abs() if data == "int" else normal(g, (Cc,)).abs() + 0.5).to(cuda)
    dshape = (N, 1, 1, Cc) if pooled else shape
    dy = vals(g, dshape, data).to(cuda)
    # reference: autograd through AdaptiveAvgPool2d(1) and hardtanh(0, 6)
    y = (a * sc + sh).float().double().requires_grad_(True)   # the fp32 fmaf the mask is read from
    out = F.hardtanh(y, 0.0, 6.0)
    if pooled:
        (F.adaptive_avg_pool2d(out.permute(0, 3, 1, 2), 1).permute(0, 2, 3, 1) * dy).sum().backward()
    else:
        (out * dy).sum().backward()
    ref_g = y.grad
    if data == "int":
        assert bool(((y == 0) | (y == 6)).any()), "no ReLU6 boundary hit"
    A, G, DY = Slot(shape, cuda, lay, a), Slot(shape, cuda, lay), Slot(dshape, cuda, "dense", dy)
    sums0 = ints(g, (2 * Cc,), 5).to(cuda)
    runs = []
    for _ in range(2):
        s = sums0.clone()
        ops.relu6_bwd_reduce(DY.t, A.t, _f(sc), _f(sh), _f(mean), _f(invstd), G.t, s, pooled)
        runs.append(s)
    torch.cuda.synchronize()
    what = f"relu6_bwd_reduce {shape} {lay} pooled={pooled} {data}"
    same_bits(runs[0], runs[1], what + " reproducible")
    expect(G.t, ref_g, ref_g.abs(), 2, data, what + " g", 1.0 / 64)
    gk = G.t.double().reshape(-1, Cc)
    xh = ((a - mean) * invstd).reshape(-1, Cc)
    k = N * H * W + 64
    expect(runs[0][:Cc] - sums0[:Cc], gk.sum(0), gk.abs().sum(0), k, data, what + " sum g", 1.0 / 64)
    m2 = (gk * xh).abs().sum(0) + (gk.abs() * ((a.abs() + mean.abs()) * invstd).reshape(-1, Cc)).sum(0) * 3 / k
    expect(runs[0][Cc:] - sums0[Cc:], (gk * xh).sum(0), m2, k, data, what + " sum g*xh",
           grid_of(gk) * grid_of(xh) if data == "int" else None)
    assert_intact(what, A, G, DY)


@gpu
@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("shape,lay", path_cases([(2, 3, 5, 3), (1, 4, 4, 32), (2, 7, 7, 96), BIG],
                                                 ("dense", "ld1")))
def test_mobilenet_elementwise(cuda, shape, lay, data):
    """affine_relu6 (inputs exactly on 0 and 6 included) and avgpool_bwd."""
    g = _gen("mbv2 ew", shape, data)
    N, H, W, Cc = shape
    a = (ints(g, shape, 4) + 2 if data == "int" else (normal(g, shape) * 3).float().double()).to(cuda)
    sc, sh = bn_scale(g, Cc, data).to(cuda), bn_shift(g, Cc, data).to(cuda)
    A, Y = Slot(shape, cuda, lay, a), Slot(shape, cuda, lay)
    ops.affine_relu6(A.t, _f(sc), _f(sh), Y.t)
    dy = vals(g, (N, Cc), data).to(cuda)
    G = Slot(shape, cuda, lay)
    ops.avgpool_bwd(dy.float(), G.t)
    torch.cuda.synchronize()
    what = f"mobilenet {shape} {lay} {data}"
    expect(Y.t, (a * sc + sh).clamp(0, 6), (a * sc).abs() + sh.abs(), 1, data, what + " affine_relu6", 1.0 / 4)
    HW = H * W
    ref = (dy / HW).view(N, 1, 1, Cc).expand(shape)
    # 1/HW in fp32, then one product: exact for HW a power of two on the integer grid
    d_int = "int" if data == "int" and HW & (HW - 1) == 0 else "randn"
    expect(G.t, ref, ref.abs(), 2, d_int, what + " avgpool_bwd", 1.0 / HW)
    assert_intact(what, A, Y, G)


@gpu
@pytest.mark.parametrize("B,Cc", [(1, 1), (3, 10), (7, 33), (5, 100), (2000, 3)])
def test_log_softmax_bwd(cuda, B, Cc):
    g = _gen("log_softmax_bwd", B, Cc)
    x = normal(g, (B, Cc)) * 4
    y = torch.log_softmax(x, -1).float().to(cuda)
    dy = normal(g, (B, Cc)).float().to(cuda)
    dx = torch.full((B, Cc), float("nan"), device=cuda)
    ops.log_softmax_bwd(y, dy, dx)
    torch.cuda.synchronize()
    y64, d64 = y.double(), dy.double()
    s = d64.sum(-1, keepdim=True)
    ref = d64 - y64.exp() * s
    # expf (2 ulp), the C-term warp sum, product and difference
    mag = d64.abs() + y64.exp() * (d64.abs().sum(-1, keepdim=True) * (Cc + 2) + s.abs() * 4)
    expect(dx, ref, mag, 2, "randn", f"log_softmax_bwd B={B} C={Cc}")


# ============================================================================= vae.cu
GEMM_MNK = [(1, 1, 1), (15, 16, 17), (16, 17, 15), (17, 15, 16), (63, 64, 65), (64, 65, 63),
            (65, 63, 64), (200, 17, 1), (1, 200, 64), (17, 1, 200), (64, 64, 200), (65, 65, 0),
            (15, 200, 200), (200, 1, 17)]
GEMM_EPI = [("id", ACT_LRELU, 1.0), ("relu", ACT_LRELU, 0.0), ("lrelu", ACT_LRELU, 0.25),
            ("tanh", ACT_TANH, 1.0)]


def gemm_strides(pat, M, N, K):
    """(A shape, a_sm, a_sk, B shape, b_sk, b_sn, to-matrix functions) of the callers' patterns:
    NN (coord_latent's dz = sb Wz, gp.py's W z2), NT (Linear forward, x W^T),
    TN (Linear / coord_latent weight gradients, gp.py's W^T z1)."""
    if pat == "NN":
        return (M, K), K, 1, (K, N), N, 1, (lambda a: a), (lambda b: b)
    if pat == "NT":
        return (M, K), K, 1, (N, K), 1, K, (lambda a: a), (lambda b: b.t())
    return (K, M), 1, M, (K, N), N, 1, (lambda a: a.t()), (lambda b: b)


@gpu
@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("pat", ("NN", "NT", "TN"))
@pytest.mark.parametrize("M,N,K", GEMM_MNK, ids=lambda v: str(v))
def test_gemm(cuda, M, N, K, pat, data):
    g = _gen("gemm", M, N, K, pat, data)
    ash, a_sm, a_sk, bsh, b_sk, b_sn, am, bm = gemm_strides(pat, M, N, K)
    A, B = vals(g, ash, data).to(cuda), vals(g, bsh, data).to(cuda)
    bias = vals(g, (N,), data).to(cuda)
    prior = vals(g, (M, N), data).to(cuda)
    Af, Bf = A.float(), B.float()
    A64, B64 = am(A), bm(B)
    prod = A64 @ B64
    pmag = A64.abs() @ B64.abs()
    c_sm = N + 3
    for (ename, act, slope), has_bias, acc, split in itertools.product(GEMM_EPI, (True, False),
                                                                       (False, True), (1, 2, 4, 8)):
        kps = max(16, -(-(-(-K // split)) // 16) * 16)      # as atomai_b200_gemm rounds it
        eff_split = max(1, -(-K // kps))
        if eff_split > 1 and not (act == ACT_LRELU and slope == 1.0):
            continue                          # refused (test_refusals)
        if data == "int" and act == ACT_TANH:
            continue
        what = f"gemm {pat} M={M} N={N} K={K} {ename} bias={has_bias} acc={acc} split={split}->{eff_split} {data}"
        buf = torch.full((M * c_sm + 4,), float("nan"), device=cuda)
        Cv = buf[:M * c_sm].view(M, c_sm)[:, :N]
        if acc:
            Cv.copy_(prior)
        ops.gemm(Af, a_sm, a_sk, Bf, b_sk, b_sn, Cv, c_sm, M, N, K, bias.float() if has_bias else None,
                 act, slope, acc, split)
        torch.cuda.synchronize()
        z = prod + (bias if has_bias else 0)
        zm = pmag + (bias.abs() if has_bias else 0)
        if act == ACT_TANH:
            ref, mag = torch.tanh(z), zm + 1
        else:
            ref, mag = torch.where(z > 0, z, z * slope), zm
        if acc:
            ref, mag = ref + prior, mag + prior.abs()
        # K fma per partial sum, <= 8 split-K atomics, bias, epilogue, accumulate; tanhf 2 ulp
        expect(Cv, ref, mag, K + 12 + (2 if act == ACT_TANH else 0), data, what, 1.0 / 4)
        mask = torch.ones_like(buf, dtype=torch.bool)
        mask[:M * c_sm].view(M, c_sm)[:, :N] = False
        assert bool(torch.all(buf[mask].view(torch.int32) == NAN_BITS)), what + ": wrote outside C"


@gpu
def test_gemm_split_k_accumulate_keeps_bias(cuda):
    """accumulate = 1 means C += A.B + bias whatever the effective K split (regression: the split-K
    epilogue used to drop the bias when accumulating)."""
    M, N, K = 33, 70, 512
    g = _gen("gemm split acc")
    A, B, bias, prior = ints(g, (M, K), 2), ints(g, (K, N), 2), ints(g, (N,), 5), ints(g, (M, N), 5)
    ref = (prior + A @ B + bias).to(cuda)
    for split in (1, 2, 8):
        Cm = prior.float().to(cuda)
        ops.gemm(A.float().to(cuda), K, 1, B.float().to(cuda), N, 1, Cm, N, M, N, K,
                 bias.float().to(cuda), ACT_LRELU, 1.0, True, split)
        torch.cuda.synchronize()
        msg = first_mismatch(Cm, ref)
        assert msg is None, f"split_k={split}: {msg}"


LINEAR_CASES = [(B, K, O) for B in (1, 5, 768) for K in (4096, 8196) for O in (1, 8, 9, 16)] + \
               [(5, 1000, 5), (3, 4096, 17), (4, 4099, 8), (100, 200, 40)]


def skinny(B, K, O):
    return 1 <= O <= 16 and K % 4 == 0 and K >= 4096 and B >= 1


@gpu
@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("B,K,O", LINEAR_CASES, ids=lambda v: str(v))
def test_linear(cuda, B, K, O, data):
    g = _gen("linear", B, K, O, data)
    x, w, b = vals(g, (B, K), data, 2).to(cuda), vals(g, (O, K), data, 2).to(cuda), vals(g, (O,), data).to(cuda)
    dy = vals(g, (B, O), data).to(cuda)
    what = f"linear B={B} K={K} O={O} {data} {'skinny' if skinny(B, K, O) else 'general'}"
    y = torch.full((B, O), float("nan"), device=cuda)
    ops.linear_fwd(x.float(), w.float(), b.float(), y)
    torch.cuda.synchronize()
    expect(y, x @ w.t() + b, x.abs() @ w.abs().t() + b.abs(), K + 4, data, what + " fwd", 1.0)
    for with_dx, with_dw in ((True, True), (False, True), (True, False)):
        dx = torch.full((B, K), float("nan"), device=cuda) if with_dx else None
        dw = torch.full((O, K), float("nan"), device=cuda) if with_dw else None
        db = torch.full((O,), float("nan"), device=cuda)
        ops.linear_bwd(x.float(), w.float(), dy.float(), dx, dw, db)
        torch.cuda.synchronize()
        w_ = f"{what} bwd dx={with_dx} dw={with_dw}"
        if with_dx:
            expect(dx, dy @ w, dy.abs() @ w.abs(), O + 4, data, w_ + " dx", 1.0)
        if with_dw:
            expect(dw, dy.t() @ x, dy.abs().t() @ x.abs(), B + 4, data, w_ + " dw", 1.0)
        expect(db, dy.sum(0), dy.abs().sum(0), B + 4, data, w_ + " db", 1.0)


COORD_CASES = [(2, 3, 5, 4, 1), (1, 9, 17, 0, 100), (3, 5, 1, 2, 128), (2, 1, 9, 3, 129),
               (1, 17, 9, 6, 512), (2, 2, 3, 0, 7)]


@gpu
@pytest.mark.parametrize("tanh_act,data", [(False, "int"), (False, "randn"), (True, "randn")],
                         ids=("id-int", "id-randn", "tanh-randn"))
@pytest.mark.parametrize("B,H,W,zdim,hid", COORD_CASES, ids=lambda v: str(v))
def test_coord_latent(cuda, B, H, W, zdim, hid, tanh_act, data):
    """rVAE's first decoder layer: h0 = act(Wc (R(phi) g + dx) + bc + Wz z) on imcoordgrid, and
    the backward sums (dwc, dbc, sb, dphi, ddx) against float64 autograd.  Exact tier: grid sizes
    with H - 1, W - 1 powers of two (or 1) and phi = 0, so every coordinate is dyadic."""
    for with_phi, with_dx in ((True, True), (False, False), (True, False), (False, True)):
        run_coord_latent(cuda, B, H, W, zdim, hid, tanh_act, data, with_phi, with_dx)


def run_coord_latent(dev, B, H, W, zdim, hid, tanh_act, data, with_phi, with_dx):
    g = _gen("coord", B, H, W, zdim, hid, data)
    what = f"coord_latent B={B} {H}x{W} z={zdim} hid={hid} tanh={tanh_act} phi={with_phi} dx={with_dx} {data}"
    if data == "int":
        assert all(n == 1 or (n - 1) & (n - 2) == 0 for n in (H, W)), "grid not dyadic"
    z = vals(g, (B, zdim), data).to(dev) if zdim else None
    phi = (torch.zeros(B) if data == "int" else normal(g, (B,))).double().to(dev) if with_phi else None
    dxy = (ints(g, (B, 2), 2) * 0.5 if data == "int" else normal(g, (B, 2))).to(dev) if with_dx else None
    wc, bc = vals(g, (hid, 2), data, 2).to(dev), vals(g, (hid,), data).to(dev)
    wz = vals(g, (hid, zdim), data).to(dev) if zdim else None
    dpre = vals(g, (B, H, W, hid), data, 2).to(dev)
    grid = coord_grid(H, W, dev)
    # float64 reference with autograd for the backward
    lv = {k: v.clone().requires_grad_(True) for k, v in (("wc", wc), ("bc", bc), ("phi", phi), ("dx", dxy))
          if v is not None}
    ph = lv["phi"] if phi is not None else torch.zeros(B, dtype=torch.float64, device=dev)
    c, s = torch.cos(ph), torch.sin(ph)
    gx, gy = grid[:, 0], grid[:, 1]
    X = gx[None] * c[:, None] - gy[None] * s[:, None]
    Y = gx[None] * s[:, None] + gy[None] * c[:, None]
    if dxy is not None:
        X, Y = X + lv["dx"][:, :1], Y + lv["dx"][:, 1:]
    hz = lv["bc"][None] + (z @ wz.t() if zdim else 0)
    sb_leaf = torch.zeros(B, hid, dtype=torch.float64, device=dev, requires_grad=True)
    pre = X[..., None] * lv["wc"][:, 0] + Y[..., None] * lv["wc"][:, 1] + (hz + sb_leaf)[:, None, :]
    ref_h = torch.tanh(pre) if tanh_act else pre
    (pre * dpre.view(B, H * W, hid)).sum().backward()
    mag_xy = grid.abs().sum(1)[None] + (dxy.abs().sum(1, keepdim=True) if dxy is not None else 0)   # (B, HW)
    hzm = bc.abs()[None] + (z.abs() @ wz.abs().t() if zdim else 0)
    mag = mag_xy[..., None] * wc.abs().sum(1) + hzm[:, None, :] + (1 if tanh_act else 0)
    h0 = torch.full((B, H, W, hid), float("nan"), device=dev)
    keep = [_f(z), _f(phi), _f(dxy), wc.float(), bc.float(), _f(wz)]
    d = ops.coord_latent_desc(B, H, W, keep[0], keep[1], keep[2], keep[3], keep[4], keep[5], tanh_act)
    ops.coord_latent_fwd(d, h0)
    torch.cuda.synchronize()
    expect(h0.view(B, H * W, hid), ref_h.detach(), mag, zdim + 12, data, what + " fwd", 1.0 / 64)
    # backward: every output accumulates into a non-zero prior
    pri = {k: ints(g, sh, 3).to(dev) for k, sh in
           (("dwc", (hid, 2)), ("dbc", (hid,)), ("sb", (B, hid)), ("dphi", (B,)), ("ddx", (B, 2)))}
    outs = {k: v.float() for k, v in pri.items()}
    dpf = dpre.float()
    ops.coord_latent_bwd(d, dpf, outs["dwc"], outs["dbc"], outs["sb"],
                         outs["dphi"] if with_phi else None, outs["ddx"] if with_dx else None)
    torch.cuda.synchronize()
    HW = H * W
    # per-thread sums over a pixel chunk and the hidden lanes, a 128-thread CTA sum, atomics
    k = B * HW + hid + 160
    ad = dpre.abs().view(B, HW, hid)
    refs = {"dwc": (lv["wc"].grad, torch.stack([(ad * mag_xy[..., None]).sum((0, 1))] * 2, 1)),
            "dbc": (lv["bc"].grad, ad.sum((0, 1))),
            "sb": (sb_leaf.grad, ad.sum(1))}
    dmag = (ad * wc.abs().sum(1)).sum(-1)                       # (B, HW)
    if with_phi:
        refs["dphi"] = (lv["phi"].grad, (dmag * grid.abs().sum(1)[None]).sum(1))
    if with_dx:
        refs["ddx"] = (lv["dx"].grad, dmag.sum(1, keepdim=True).expand(B, 2))
    for name, (r, m) in refs.items():
        expect(outs[name].double() - pri[name], r, m + 1e-300, k, data, f"{what} {name}", 1.0 / 8)
    if not with_phi:
        assert torch.equal(outs["dphi"].double(), pri["dphi"]), what + ": dphi written though NULL"


# ============================================================================= host-side refusals
@gpu
def test_refusals(cuda):
    """Unsupported arguments are refused by the host-side checks, before any launch."""
    dev = cuda
    z = lambda *s: torch.zeros(*s, device=dev)
    err = _C.NativeError
    for Cc in (257, 1028):
        a = z(1, 2, 2, Cc)
        with pytest.raises(err, match="bn_bwd_reduce"):
            ops.bn_bwd_reduce(a, a, z(Cc), z(Cc), torch.zeros(2 * Cc, dtype=torch.float64, device=dev))
        with pytest.raises(err, match="bn_lrelu_bwd"):
            ops.bn_act_bwd(a, a, None, None, None, None, 1.0, None, ACT_LRELU, 0.1, z(1, 2, 2, Cc), None)
    for Cc in (12, 5):                      # C/4 not a power of two; no float4 path at all
        dp, full = z(1, 2, 2, Cc), z(1, 4, 4, Cc)
        with pytest.raises(err, match="pool2x2_bwd_bn"):
            ops.pool_bwd(dp, full, None, None, full, False, z(Cc), z(Cc),
                         torch.zeros(2 * Cc, dtype=torch.float64, device=dev))
    with pytest.raises(err, match="split-K"):
        ops.gemm(z(8, 256), 256, 1, z(256, 8), 8, 1, z(8, 8), 8, 8, 8, 256, None, ACT_TANH, 1.0,
                 False, 4)
    a = z(1, 2, 2, 4)
    for layers, slope in (([], 0.1), ([a] * 9, 0.1), ([a], 0.0)):
        with pytest.raises(err, match="dilated_sum"):
            ops.dilated_sum(layers, [None] * len(layers), [None] * len(layers), slope, z(1, 2, 2, 4))
    for slope in (0.0, -0.1):
        with pytest.raises(err, match="lrelu_mask_bwd"):
            ops.lrelu_mask_bwd(a, a, slope, z(1, 2, 2, 4))
    with pytest.raises(err, match="hid=513"):
        ops.coord_latent_fwd(ops.coord_latent_desc(1, 2, 2, None, None, None, z(513, 2), z(513),
                                                   None, False), z(1, 2, 2, 513))
    with pytest.raises(err, match="scale and shift"):
        ops.affine_res_act(a, z(4), None, None, 0.1, z(1, 2, 2, 4))
    torch.cuda.synchronize()


@gpu
def test_dilated_sum_rejects_strided_views(cuda):
    buf = torch.zeros(1, 2, 2, 8, device=cuda)
    with pytest.raises(AssertionError):
        ops.dilated_sum([buf[..., :4]], [None], [None], 0.1, torch.zeros(1, 2, 2, 4, device=cuda))
    with pytest.raises(AssertionError):
        ops.dilated_sum([torch.zeros(1, 2, 2, 4, device=cuda)], [None], [None], 0.1, buf[..., :4])


# ============================================================================= dispatch coverage
@gpu
def test_dispatch_coverage_by_width(cuda):
    """Both instances (W = 4 and W = 1) of every dual-path kernel (and the special kernels) are
    launched by the cases above; a dispatch rule that changes later shows up here."""
    from torch.profiler import ProfilerActivity, profile
    dev = cuda
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for lay in ("dense", "ld1"):
            run_affine(dev, (2, 3, 5, 12), lay, "int")
            run_add_slice(dev, (2, 3, 5, 12), lay, "int", True)
            run_pool(dev, (2, 3, 5, 16), lay, "int")
            run_upsample(dev, (2, 3, 5, 12), lay, "int", True)
            run_bn_act_bwd(dev, (2, 3, 5, 12), lay, "int", True, True, True, ACT_LRELU, True)
            run_affine_res_act(dev, (2, 3, 5, 12), lay, "int", True, True)
        run_pool(dev, (2, 3, 5, 16), "dense", "int", stats=True)
        for Cc in (12, 5):
            s = torch.zeros(2 * Cc, dtype=torch.float64, device=dev)
            a = torch.zeros(1, 2, 2, Cc, device=dev)
            ops.bn_bwd_reduce(a, a, torch.zeros(Cc, device=dev), torch.ones(Cc, device=dev), s)
        x = torch.ones(5, 4096, device=dev)
        for O in (8, 16):
            w = torch.ones(O, 4096, device=dev)
            y = torch.empty(5, O, device=dev)
            ops.linear_fwd(x, w, torch.zeros(O, device=dev), y)
            ops.linear_bwd(x, w, torch.ones(5, O, device=dev), torch.empty_like(x), torch.empty_like(w),
                           torch.empty(O, device=dev))
        ops.gemm(torch.ones(4, 512, device=dev), 512, 1, torch.ones(512, 4, device=dev), 4, 1,
                 torch.empty(4, 4, device=dev), 4, 4, 4, 512, None, ACT_LRELU, 1.0, False, 4)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    text = "\n".join(sorted(set(names)))

    def launched(pat):
        return any(pat in n for n in names)

    for k in ("affine_kernel<4>", "affine_kernel<1>", "add_slice_kernel<4>", "add_slice_kernel<1>",
              "pool_fwd_kernel<4>", "pool_fwd_kernel<1>", "pool_bwd_kernel<4, true>",
              "pool_bwd_kernel<4, false>", "pool_bwd_kernel<1, false>", "upsample_fwd_kernel<4>",
              "upsample_fwd_kernel<1>", "upsample_bwd_kernel<4>", "upsample_bwd_kernel<1>",
              "bn_bwd_reduce_kernel<4>", "bn_bwd_reduce_kernel<1>", "bn_lrelu_bwd_kernel<4>",
              "bn_lrelu_bwd_kernel<1>", "affine_res_act_kernel<4>", "affine_res_act_kernel<1>",
              "skinny_fwd_kernel", "skinny_bwd_kernel<8>", "skinny_bwd_kernel<16>", "gemm_kernel",
              "bias_fill_kernel"):
        assert launched(k), f"{k} was not launched; kernels seen:\n{text}"
