"""Exact and float64 parity of the convolution kernels (conv_tc, wgrad_tc and the exact-fp32 SIMT
kernels), driven through the C ABI (`atomai_b200.ops`).

(a) Exact arithmetic.  Inputs, weights and biases are small integers (BN scales in +-{0.5, 1, 2},
    shifts on a 0.5 grid, LeakyReLU slope 1 or 0.25, bilinear weights 1/4 and 3/4), so every
    product and partial sum the kernels form is exactly representable: RN-to-TF32, the bf16
    correction planes (whose low parts are 0), the tensor core's truncating fp32 accumulation,
    FFMA, float atomics and the ordered double sums are all exact.  The output must then be
    bitwise equal to a float64 reference in fp32, tf32 and tf32x3 under every tile plan.  Each
    case asserts that precondition itself: conv(|x|, |w|) + |b|, in units of the value grid,
    stays below 2^24 (and the BN statistics' fp32 partials likewise).
(b) Correction terms (tf32x3).  x = i + k 2^-16 (i in {-1, 0, 1}, |k| <= 15) rounds to exactly i
    in TF32 and leaves an exact bf16/TF32 low part; tf32x3 must again be bitwise equal to float64,
    and tf32 must differ.  Repeated with the low parts on the weights, for the data gradient, and
    for wgrad_tc with low parts on dy only and on x only (lo * lo is dropped by design).
(c) Rounding on normal data, per element against the arithmetic model
    |y - y64| <= c(K) (conv(|x|, |w|) + |b|),  c = (K+2) 2^-24 (fp32),
    2^-10 + (K+2) 2^-23 (tf32), 2^-18 + (K+2) 2^-23 (tf32x3); tf32x3 at least 8x more accurate than
    tf32 (norm-wise) for K >= 72; every launch bitwise reproducible (outputs, BN statistics and
    weight gradients are ordered sums in every kernel, the exact-fp32 ones included).

PLAN_MATRIX forces every conv_tc plan variant through the plan hooks; tests/test_conv_plan.py
checks on a CPU that each entry still produces the plan it names.
"""
import os
import re
import tempfile
import zlib
from dataclasses import dataclass
from types import SimpleNamespace
from typing import List, Tuple

import pytest
import torch
import torch.nn.functional as F

from atomai_b200 import _C, ops
from atomai_b200.ops import Source

FP32, TF32, TF32X3 = ops.MATH_FP32, ops.MATH_TF32, ops.MATH_TF32X3
MATH_NAMES = {FP32: "fp32", TF32: "tf32", TF32X3: "tf32x3"}
LIMIT = 2 ** 24


# ----------------------------------------------------------------------------- layer description
@dataclass
class S:
    """One input source: C channels, optional BN affine, on-load transform (ops.SRC_*), and `pad`
    extra channels in the buffer (pixel stride ld = C + pad, filled with NaN)."""
    C: int
    tr: int = ops.SRC_PLAIN
    aff: bool = False
    pad: int = 0

    def __repr__(self):
        t = ["", "pool", "bil", "near"][self.tr]
        return f"{self.C}" + (f"+{t}" if t else "") + ("+aff" if self.aff else "") + \
            (f"+ld{self.C + self.pad}" if self.pad else "")


@dataclass
class Layer:
    srcs: List[S]
    cout: int
    H: int
    W: int
    N: int = 2
    ks: Tuple[int, int] = (3, 3)
    dil: int = 1

    def __post_init__(self):
        self.srcs = [s if isinstance(s, S) else S(s) for s in self.srcs]
        if isinstance(self.ks, int):
            self.ks = (self.ks, self.ks)

    @property
    def ctot(self):
        return sum(s.C for s in self.srcs)

    @property
    def taps(self):
        return self.ks[0] * self.ks[1]

    @property
    def pad(self):
        return (self.dil * (self.ks[0] // 2), self.dil * (self.ks[1] // 2))

    def __repr__(self):
        return (f"N{self.N} {self.H}x{self.W} {self.srcs}->{self.cout} k{self.ks[0]}x{self.ks[1]} "
                f"d{self.dil}")


def L(srcs, cout, H, W, **kw):
    return Layer(list(srcs), cout, H, W, **kw)


# ----------------------------------------------------------------------------- plan matrix
# (id, environment, layer, math, plan the environment must produce).  Every conv_tc variant:
# resident / streamed weights, sub-tiles 1 and 2, KC 8/16/32, operand rings n_a = 2 (one stage
# per pipeline) and 4, the smallest weight ring, TMA and register-staged loaders, every consumer
# instantiation (nn x sub), second launches of 16 and 80 channels.
def _p(resident, sub, KC, n_a, n_b, tma):
    return dict(resident=resident, sub=sub, KC=KC, n_a=n_a, n_b=n_b, tma=tma)


PLAN_MATRIX = [
    ("res_tma", {}, L([16], 16, 32, 32), TF32X3, _p(1, 1, 16, 4, 0, 1)),
    ("res_tma_tf32", {}, L([16], 16, 16, 16), TF32, _p(1, 1, 16, 4, 0, 1)),
    ("res_tma_nn48", {}, L([16], 48, 32, 32), TF32X3, _p(1, 1, 16, 4, 0, 1)),
    ("res_tma_kc32_tf32", {}, L([32], 80, 16, 16), TF32, _p(1, 1, 32, 4, 0, 1)),
    ("res_tma_off", {"ATOMAI_B200_TMA": "0"}, L([16], 16, 32, 32), TF32X3, _p(1, 1, 16, 4, 0, 0)),
    ("res_tma_kc8", {"ATOMAI_B200_TMA_KC8": "1"}, L([8], 32, 16, 16), TF32X3, _p(1, 1, 8, 4, 0, 1)),
    ("res_kc8", {"ATOMAI_B200_PLAN": "0,8"}, L([16], 16, 32, 32), TF32X3, _p(1, 1, 8, 4, 0, 0)),
    ("res_kc32", {"ATOMAI_B200_PLAN": "0,32"}, L([16, 16], 16, 32, 32), TF32X3, _p(1, 1, 32, 4, 0, 0)),
    ("res_tma_concat", {"ATOMAI_B200_PLAN": "0,16"}, L([16, 16], 16, 32, 32), TF32X3,
     _p(1, 1, 16, 4, 0, 1)),
    ("res_na2_nn80", {}, L([32], 80, 16, 16), TF32X3, _p(1, 1, 16, 2, 0, 0)),
    ("res_one_stage", {"ATOMAI_B200_SMEM_KB": "64"}, L([16], 16, 16, 16), TF32X3,
     _p(1, 1, 16, 2, 0, 0)),
    ("res_split_12_4_kc8", {"ATOMAI_B200_PLAN": "0,8"}, L([12, 4], 32, 16, 16), TF32X3,
     _p(1, 1, 8, 4, 0, 0)),
    ("res_split_12_4", {}, L([12, 4], 32, 16, 16), TF32X3, _p(1, 1, 16, 4, 0, 0)),
    ("res_split_20_12", {}, L([20, 12], 64, 16, 16), TF32X3, _p(1, 1, 16, 4, 0, 0)),
    ("str_sub2", {}, L([64], 64, 32, 32), TF32X3, _p(0, 2, 16, 4, 14, 0)),
    ("str_sub2_kc8", {"ATOMAI_B200_PLAN": "1,8"}, L([64], 64, 32, 32), TF32X3, _p(0, 2, 8, 4, 32, 0)),
    ("str_sub2_kc32", {"ATOMAI_B200_PLAN": "1,32"}, L([64], 64, 32, 32), TF32X3,
     _p(0, 2, 32, 2, 8, 0)),
    ("str_sub2_na4off", {"ATOMAI_B200_NA4": "0"}, L([64], 64, 32, 32), TF32X3, _p(0, 2, 32, 2, 8, 0)),
    ("str_sub2_one_stage", {"ATOMAI_B200_SMEM_KB": "64"}, L([64], 64, 32, 32), TF32X3,
     _p(0, 2, 8, 2, 8, 0)),
    ("str_sub2_nn16", {"ATOMAI_B200_PLAN": "1,16"}, L([16], 16, 16, 24), TF32X3,
     _p(0, 2, 16, 4, 32, 0)),
    ("str_sub2_nn32", {"ATOMAI_B200_PLAN": "1,16"}, L([16], 32, 16, 24), TF32X3,
     _p(0, 2, 16, 4, 32, 0)),
    ("str_sub2_nn48", {"ATOMAI_B200_PLAN": "1,16"}, L([16], 48, 16, 24), TF32X3,
     _p(0, 2, 16, 4, 20, 0)),
    ("str_sub1_kc8", {"ATOMAI_B200_PLAN": "2,8"}, L([64], 64, 32, 32), TF32X3, _p(0, 1, 8, 4, 32, 0)),
    ("str_sub1_kc16", {"ATOMAI_B200_PLAN": "2,16"}, L([64], 64, 32, 32), TF32X3,
     _p(0, 1, 16, 4, 20, 0)),
    ("str_sub1_kc32", {"ATOMAI_B200_PLAN": "2,32"}, L([64], 64, 32, 32), TF32X3,
     _p(0, 1, 32, 4, 6, 0)),
    ("str_split_20_12_kc8", {"ATOMAI_B200_PLAN": "2,8"}, L([20, 12], 64, 16, 16), TF32X3,
     _p(0, 1, 8, 4, 32, 0)),
    ("str_nb4", {"ATOMAI_B200_SMEM_KB": "64"}, L([16], 128, 16, 16), TF32X3, _p(0, 1, 8, 4, 4, 0)),
    ("str_nn96", {}, L([40], 96, 16, 16), TF32X3, _p(0, 1, 8, 4, 32, 0)),
    ("str_nn112", {}, L([64], 112, 16, 16), TF32X3, _p(0, 1, 32, 4, 4, 0)),
    ("str_nn128", {}, L([128], 128, 16, 16), TF32X3, _p(0, 1, 16, 4, 10, 0)),
    ("str_nn128_tf32", {}, L([128], 128, 16, 16), TF32, _p(0, 1, 32, 4, 10, 0)),
    ("str_144", {}, L([48, 16], 144, 16, 16), TF32X3, _p(0, 1, 16, 4, 8, 0)),
    ("str_208", {}, L([256], 208, 16, 16), TF32X3, _p(0, 1, 16, 4, 6, 0)),
    ("str_256", {}, L([64], 256, 16, 16), TF32X3, _p(0, 1, 16, 4, 4, 0)),
]
PLAN_IDS = [e[0] for e in PLAN_MATRIX]

PLAN_RE = re.compile(r"resident=(\d+) sub=(\d+) KC=(\d+) n_a=(\d+) n_b=(\d+) tma=(\d+)")


def parse_plan(text):
    """The fields of the last `conv_tc plan:` line in `text` (ATOMAI_B200_PLAN_LOG output)."""
    found = PLAN_RE.findall(text)
    assert found, f"no plan line in {text!r}"
    return dict(zip(("resident", "sub", "KC", "n_a", "n_b", "tma"), map(int, found[-1])))


def launch_widths(cout):
    """Output channels of each conv_tc launch (one per 128 channels)."""
    return [min(128, cout - n0) for n0 in range(0, cout, 128)]


def plan_line(d) -> str:
    """The plan conv_tc picks for descriptor `d` under the current environment (for messages)."""
    if d.math == FP32:
        return "simt"
    old = os.environ.get("ATOMAI_B200_PLAN_LOG")
    os.environ["ATOMAI_B200_PLAN_LOG"] = "1"
    saved = os.dup(2)
    try:
        with tempfile.TemporaryFile() as f:
            os.dup2(f.fileno(), 2)
            try:
                import ctypes as C
                g, b, s = C.c_int(), C.c_int(), C.c_int()
                _C.lib().atomai_b200_conv_info(C.byref(d), C.byref(g), C.byref(b), C.byref(s))
            finally:
                os.dup2(saved, 2)
            f.seek(0)
            text = f.read().decode(errors="replace")
    finally:
        os.close(saved)
        if old is None:
            del os.environ["ATOMAI_B200_PLAN_LOG"]
        else:
            os.environ["ATOMAI_B200_PLAN_LOG"] = old
    m = PLAN_RE.search(text)
    return m.group(0) if m else text.strip()


def _env_str():
    return " ".join(f"{k}={v}" for k, v in sorted(os.environ.items())
                    if k.startswith("ATOMAI_B200_") and k != "ATOMAI_B200_PLAN_LOG")


# ----------------------------------------------------------------------------- values
def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def ints(g, shape, amp=3, zero=0.3):
    v = torch.randint(-amp, amp + 1, shape, generator=g).double()
    return torch.where(torch.rand(shape, generator=g) < zero, torch.zeros_like(v), v)


def lo_vals(g, shape, dens):
    """i + k 2^-16, i in {-1, 0, 1} (non-zero with probability dens), |k| <= 15."""
    i = torch.randint(0, 2, shape, generator=g).double() * 2 - 1
    i = torch.where(torch.rand(shape, generator=g) < dens, i, torch.zeros_like(i))
    k = torch.randint(-15, 16, shape, generator=g).double()
    return i + k * 2.0 ** -16


def unit_vals(g, shape, dens):
    """{-1, 0, 1}, non-zero with probability dens."""
    return ints(g, shape, amp=1, zero=0.0) * (torch.rand(shape, generator=g) < dens).double()


def grid_of(*ts):
    """Largest power of two 2^-e (e >= 0) that divides every value of the tensors."""
    for e in range(0, 60):
        s = 2.0 ** e
        if all(bool(torch.all(torch.frac(t.double() * s) == 0)) for t in ts if t is not None):
            return 2.0 ** -e
    raise AssertionError("values are not on a binary grid")


def tf32_exact(t):
    return bool(torch.all((t.float().contiguous().view(torch.int32) & 0x1FFF) == 0))


def bf16_exact(t):
    return bool(torch.all((t.float().contiguous().view(torch.int32) & 0xFFFF) == 0))


# ----------------------------------------------------------------------------- operands
class Inputs:
    """Device sources of a layer plus the float64 (N, C, H, W) tensor the convolution sees."""

    def __init__(self, layer: Layer, g, dev, gen_x):
        self.srcs, self.keep, refs = [], [], []
        N, H, W = layer.N, layer.H, layer.W
        for s in layer.srcs:
            h, w = {ops.SRC_PLAIN: (H, W), ops.SRC_POOL: (2 * H, 2 * W)}.get(s.tr, (H // 2, W // 2))
            x = gen_x(g, (N, s.C, h, w))
            buf = torch.full((N, h, w, s.C + s.pad), float("nan"), device=dev)
            buf[..., :s.C] = x.permute(0, 2, 3, 1).float().to(dev)
            assert torch.equal(buf[..., :s.C].double().cpu(), x.permute(0, 2, 3, 1))
            xr = x.to(dev)
            sc = sh = None
            if s.aff:
                sc = torch.tensor([0.5, 1.0, 2.0])[torch.randint(0, 3, (s.C,), generator=g)] * \
                    (torch.randint(0, 2, (s.C,), generator=g).double() * 2 - 1)
                sh = torch.randint(-4, 5, (s.C,), generator=g).double() * 0.5
                xr = xr * sc.to(dev).view(1, -1, 1, 1) + sh.to(dev).view(1, -1, 1, 1)
                sc, sh = sc.float().to(dev), sh.float().to(dev)
            if s.tr == ops.SRC_POOL:
                xr = F.max_pool2d(xr, 2, 2)
            elif s.tr == ops.SRC_UP_BILINEAR:
                xr = F.interpolate(xr, scale_factor=2, mode="bilinear", align_corners=False)
            elif s.tr == ops.SRC_UP_NEAREST:
                xr = F.interpolate(xr, scale_factor=2, mode="nearest")
            self.keep += [buf, sc, sh]
            self.srcs.append(Source(buf[..., :s.C], sc, sh, s.tr))
            refs.append(xr)
        self.x = torch.cat(refs, 1)      # float64, (N, Ctot, H, W)


def nhwc_buf(t64, dev, pad=0):
    """float64 (N, C, H, W) -> float32 NHWC view with pixel stride C + pad (pad channels NaN)."""
    N, C, H, W = t64.shape
    buf = torch.full((N, H, W, C + pad), float("nan"), device=dev)
    buf[..., :C] = t64.permute(0, 2, 3, 1).float().to(dev)
    return buf, buf[..., :C]


def first_mismatch(got, ref, names="nhwc"):
    bad = ~(got.double() == ref)
    n = int(bad.sum())
    if n == 0:
        return None
    idx = tuple(int(i) for i in bad.nonzero()[0])
    return (f"{n}/{bad.numel()} elements differ, first at ({','.join(names)})={idx}: "
            f"got {float(got[idx])!r}, want {float(ref[idx])!r}")


def _ctx(tag, layer, d, math):
    return f"[{tag}] {layer} math={MATH_NAMES[math]} env=({_env_str()}) plan=({plan_line(d)})"


# ----------------------------------------------------------------------------- forward
def run_fwd(layer: Layer, math, dev, *, tag="", data="int", amp=3, slope=1.0, stats=False,
            out="nhwc", bias=True, seed=0, expect_exact=True):
    """Run conv_fwd and compare with the float64 reference.  data: "int" (a), "lo_x" / "lo_w"
    (b).  Returns (got NHWC float32, ref NHWC float64)."""
    g = _gen("fwd", repr(layer), data, seed)
    K = layer.taps * layer.ctot
    dens = min(0.6, (48.0 / K) ** 0.5)
    if data == "int":
        gx, gw = (lambda g_, s: ints(g_, s, amp)), (lambda g_, s: ints(g_, s, amp))
    elif data == "lo_x":
        gx, gw = (lambda g_, s: lo_vals(g_, s, dens)), (lambda g_, s: unit_vals(g_, s, dens))
    else:
        gx, gw = (lambda g_, s: unit_vals(g_, s, dens)), (lambda g_, s: lo_vals(g_, s, dens))
    inp = Inputs(layer, g, dev, gx)
    w = gw(g, (layer.cout, layer.ctot) + layer.ks)
    b = ints(g, (layer.cout,), amp) if bias and data == "int" else torch.zeros(layer.cout).double()
    if not bias:
        b = None
    x64, w64 = inp.x, w.to(dev)
    b64 = b.to(dev) if b is not None else None
    conv = lambda a, ww, bb: F.conv2d(a, ww, bb, padding=layer.pad, dilation=layer.dil)
    ref = F.leaky_relu(conv(x64, w64, b64), slope)
    # precondition: every partial sum is a multiple of the value grid and below 2^24 of it
    unit = grid_of(x64) * grid_of(w64)
    assert b64 is None or grid_of(b64) >= unit
    m = conv(x64.abs(), w64.abs(), b64.abs() if b64 is not None else None)
    assert float(m.max()) / unit < LIMIT, f"[{tag}] {layer}: bad case, max m = {float(m.max())} grid {unit}"
    if math != FP32 and data == "int":
        assert tf32_exact(x64) and tf32_exact(w64), f"[{tag}] operands not TF32-exact"
    if data == "lo_x":
        assert bf16_exact(w64), "weights must be bf16-exact"
    if data == "lo_w":
        assert bf16_exact(x64), "activations must be bf16-exact"
    st = None
    if stats:
        gy = unit * (0.25 if slope == 0.25 else 1.0)
        assert slope in (1.0, 0.25)
        s1 = ref.abs().sum((0, 2, 3)).max() / gy
        s2 = (ref * ref).sum((0, 2, 3)).max() / (gy * gy)
        assert float(s1) < LIMIT and float(s2) < LIMIT, f"[{tag}] {layer}: statistics not exact"
        st = torch.zeros(2 * layer.cout, device=dev, dtype=torch.float64)
    d = ops.conv_desc(inp.srcs, layer.N, layer.H, layer.W, layer.cout, layer.ks, layer.dil, slope,
                      math, out_nchw=(out == "nchw"))
    assert math == FP32 or ops.conv_supported(d, 0), f"[{tag}] {layer} not a tensor-core shape"
    wp = ops.prep_weights(w.float().to(dev), ops.WMODE_FWD, math)
    bd = b.float().to(dev) if b is not None else None
    N, H, W, Co = layer.N, layer.H, layer.W, layer.cout
    if out == "nchw":
        o = torch.full((N, Co, H, W), float("nan"), device=dev)
        ops.conv_fwd(d, wp, bd, o, st)
        got = o.permute(0, 2, 3, 1)
    elif out == "slice":
        buf = torch.full((N, H, W, Co + 24), float("nan"), device=dev)
        ops.conv_fwd(d, wp, bd, buf[..., 8:8 + Co], st)
        got = buf[..., 8:8 + Co]
        nan_bits = torch.full((1,), float("nan"), device=dev).view(torch.int32)
        for part in (buf[..., :8], buf[..., 8 + Co:]):
            assert bool(torch.all(part.contiguous().view(torch.int32) == nan_bits)), \
                f"{_ctx(tag, layer, d, math)}: wrote outside its channel slice"
    else:
        o = torch.full((N, H, W, Co), float("nan"), device=dev)
        ops.conv_fwd(d, wp, bd, o, st)
        got = o
    torch.cuda.synchronize()
    ref_nhwc = ref.permute(0, 2, 3, 1)
    if expect_exact:
        msg = first_mismatch(got, ref_nhwc)
        assert msg is None, f"{_ctx(tag, layer, d, math)}: {msg}"
        if st is not None:
            want = torch.cat([ref.sum((0, 2, 3)), (ref * ref).sum((0, 2, 3))])
            msg = first_mismatch(st, want, names="c")
            assert msg is None, f"{_ctx(tag, layer, d, math)} BN statistics: {msg}"
    return got, ref_nhwc


# ----------------------------------------------------------------------------- data gradient
def run_dgrad(layer: Layer, math, dev, *, tag="", data="int", amp=3, out_pad=0, seed=0,
              expect_exact=True):
    """dx = conv_fwd with WMODE_DGRAD weights on dy, vs float64 autograd of the forward conv;
    the dx of a two-source layer is checked as one ld view per source."""
    assert all(s.tr == ops.SRC_PLAIN and not s.aff for s in layer.srcs)
    g = _gen("dgrad", repr(layer), data, seed)
    K = layer.taps * layer.cout
    dens = min(0.6, (48.0 / K) ** 0.5)
    N, H, W = layer.N, layer.H, layer.W
    if data == "int":
        dy, w = ints(g, (N, layer.cout, H, W), amp), ints(g, (layer.cout, layer.ctot) + layer.ks, amp)
    elif data == "lo_x":
        dy, w = lo_vals(g, (N, layer.cout, H, W), dens), unit_vals(g, (layer.cout, layer.ctot) + layer.ks, dens)
    else:
        dy, w = unit_vals(g, (N, layer.cout, H, W), dens), lo_vals(g, (layer.cout, layer.ctot) + layer.ks, dens)
    dy64, w64 = dy.to(dev), w.to(dev)

    def vjp(dyv, wv):
        xin = torch.zeros(N, layer.ctot, H, W, device=dev, dtype=torch.float64, requires_grad=True)
        F.conv2d(xin, wv, None, padding=layer.pad, dilation=layer.dil).backward(dyv)
        return xin.grad

    ref = vjp(dy64, w64)
    m = vjp(dy64.abs(), w64.abs())
    unit = grid_of(dy64) * grid_of(w64)
    assert float(m.max()) / unit < LIMIT, f"[{tag}] {layer}: bad dgrad case"
    dbuf, dyv = nhwc_buf(dy64, dev)
    d = ops.conv_desc([Source(dyv)], N, H, W, layer.ctot, layer.ks, layer.dil, 1.0, math)
    assert math == FP32 or ops.conv_supported(d, 0), f"[{tag}] {layer} dgrad not a tensor-core shape"
    wp = ops.prep_weights(w.float().to(dev), ops.WMODE_DGRAD, math)
    buf = torch.full((N, H, W, layer.ctot + out_pad), float("nan"), device=dev)
    ops.conv_fwd(d, wp, None, buf[..., :layer.ctot], None)
    torch.cuda.synchronize()
    got = buf[..., :layer.ctot]
    ref_nhwc = ref.permute(0, 2, 3, 1)
    if expect_exact:
        c0 = 0
        for i, s in enumerate(layer.srcs):
            msg = first_mismatch(got[..., c0:c0 + s.C], ref_nhwc[..., c0:c0 + s.C])
            assert msg is None, f"{_ctx(tag, layer, d, math)} dgrad of source {i}: {msg}"
            c0 += s.C
        if out_pad:
            assert bool(torch.isnan(buf[..., layer.ctot:]).all()), f"[{tag}] wrote past ld slice"
    return got, ref_nhwc, m.permute(0, 2, 3, 1)


# ----------------------------------------------------------------------------- weight gradient
def run_wgrad(layer: Layer, math, dev, *, tag="", data="int", amp=3, dy_pad=0, prefill=True, seed=0,
              expect_exact=True):
    """dW (+)= conv_wgrad(x, dy) vs float64 autograd, dW pre-filled with integers."""
    g = _gen("wgrad", repr(layer), data, seed)
    N, H, W = layer.N, layer.H, layer.W
    npx = N * H * W
    dens = min(0.6, (48.0 / npx) ** 0.5)
    if data == "int":
        gx, gdy = (lambda g_, s: ints(g_, s, amp)), (lambda g_, s: ints(g_, s, amp))
    elif data == "lo_x":
        gx, gdy = (lambda g_, s: lo_vals(g_, s, dens)), (lambda g_, s: unit_vals(g_, s, dens))
    else:   # lo_dy
        gx, gdy = (lambda g_, s: unit_vals(g_, s, dens)), (lambda g_, s: lo_vals(g_, s, dens))
    inp = Inputs(layer, g, dev, gx)
    dy64 = gdy(g, (N, layer.cout, H, W)).to(dev)
    pre = ints(g, (layer.cout, layer.ctot) + layer.ks, 7) if prefill else \
        torch.zeros((layer.cout, layer.ctot) + layer.ks).double()
    pre64 = pre.to(dev)

    def wgrad(x, dy):
        w = torch.zeros((layer.cout, layer.ctot) + layer.ks, device=dev, dtype=torch.float64,
                        requires_grad=True)
        F.conv2d(x, w, None, padding=layer.pad, dilation=layer.dil).backward(dy)
        return w.grad

    ref = pre64 + wgrad(inp.x, dy64)
    m = pre64.abs() + wgrad(inp.x.abs(), dy64.abs())
    unit = grid_of(inp.x) * grid_of(dy64)
    assert float(m.max()) / unit < LIMIT, f"[{tag}] {layer}: bad wgrad case, m={float(m.max())}"
    dbuf, dyv = nhwc_buf(dy64, dev, dy_pad)
    d = ops.conv_desc(inp.srcs, N, H, W, layer.cout, layer.ks, layer.dil, 1.0, math)
    assert math == FP32 or ops.conv_supported(d, 1), f"[{tag}] {layer} not a wgrad_tc shape"
    dw = pre.float().to(dev)
    ops.conv_wgrad(d, dyv, dw)
    torch.cuda.synchronize()
    if expect_exact:
        msg = first_mismatch(dw, ref, names=("co", "ci", "ky", "kx"))
        assert msg is None, (f"[{tag}] {layer} wgrad math={MATH_NAMES[math]} env=({_env_str()}) "
                             f"prefill={prefill}: {msg}")
    return dw, ref, m, npx


# ============================================================================= (a) exact parity
MATHS = [FP32, TF32, TF32X3]
MATH_IDS = ["fp32", "tf32", "tf32x3"]

FWD_CASES = [
    # every consumer width (Cout 16 .. 128), second launches (144, 208, 256), every Cin
    ("c8_16", L([8], 16, 16, 16), {}),
    ("c16_32", L([16], 32, 16, 16), {}),
    ("c24_48", L([24], 48, 16, 16), {}),
    ("c40_64", L([40], 64, 16, 16), {}),
    ("c64_80", L([64], 80, 16, 16), {}),
    ("c128_96", L([128], 96, 16, 16), {}),
    ("c256_112", L([256], 112, 8, 16), {}),
    ("c16_128", L([16], 128, 16, 16), {}),
    ("c24_144", L([24], 144, 16, 16), {}),
    ("c40_208", L([40], 208, 16, 16), {}),
    ("c8_256", L([8], 256, 16, 16), {}),
    # sources
    ("affine", L([S(16, aff=True)], 32, 16, 16), {}),
    ("pool", L([S(16, ops.SRC_POOL)], 32, 16, 16), {}),
    ("pool_affine_neg", L([S(32, ops.SRC_POOL, aff=True)], 32, 12, 20), {}),
    ("up_bilinear", L([S(16, ops.SRC_UP_BILINEAR)], 32, 16, 16), {}),
    ("up_bilinear_affine", L([S(16, ops.SRC_UP_BILINEAR, aff=True)], 16, 20, 28), {}),
    ("up_nearest", L([S(16, ops.SRC_UP_NEAREST, aff=True)], 32, 16, 24), {}),
    ("cat_16_16", L([16, 16], 16, 16, 16), {}),
    ("cat_64_64", L([64, 64], 64, 16, 16), {}),
    ("cat_48_16", L([48, 16], 48, 16, 16), {}),
    ("cat_16_48", L([16, 48], 32, 16, 16), {}),
    ("cat_12_4", L([12, 4], 32, 16, 16), {}),
    ("cat_20_12", L([20, 12], 64, 16, 16), {}),
    ("cat_decoder_up", L([S(16, aff=True), S(16, ops.SRC_UP_BILINEAR, aff=True)], 16, 16, 16), {}),
    ("cat_pool_plain", L([S(16, ops.SRC_POOL, aff=True), S(16, aff=True)], 32, 8, 16), {}),
    ("src_ld", L([S(16, pad=8)], 32, 16, 16), {}),
    ("cat_ld", L([S(12, pad=4), S(20, pad=12, aff=True)], 48, 16, 16), {}),
    # outputs
    ("out_slice", L([16], 32, 16, 16), {"out": "slice"}),
    ("out_slice_144", L([16, 16], 144, 8, 16), {"out": "slice"}),
    ("out_nchw", L([16], 48, 12, 20), {"out": "nchw"}),
    ("slope_quarter", L([16], 32, 16, 16), {"slope": 0.25}),
    # kernel sizes and dilation (halo larger than the image at 6 on 5 x 7)
    ("k1x1", L([64], 32, 16, 16, ks=1), {}),
    ("k1x1_kc8", L([24], 16, 13, 21, ks=1), {}),
    ("k1x3_h1", L([16], 32, 1, 40, ks=(1, 3)), {}),
    ("k1x3_h1_dil2", L([32], 48, 1, 37, ks=(1, 3), dil=2), {}),
    ("dil2", L([16], 32, 16, 16, dil=2), {}),
    ("dil4", L([32], 64, 20, 20, dil=4), {}),
    ("dil6", L([16], 32, 24, 24, dil=6), {}),
    ("dil6_halo_gt_image", L([16], 16, 5, 7, dil=6), {}),
    ("dil4_pool", L([S(16, ops.SRC_POOL, aff=True)], 32, 12, 12, dil=4), {}),
    # ragged shapes
    ("ragged_13x21", L([16], 32, 13, 21), {}),
    ("ragged_w5", L([32], 16, 11, 5), {}),
    ("ragged_n1_w8", L([16], 64, 9, 8, N=1), {}),
    ("ragged_sub2", L([64], 64, 13, 19), {}),
    ("one_pixel", L([16], 16, 1, 1, N=3), {}),
]


@pytest.mark.gpu
@pytest.mark.parametrize("math", MATHS, ids=MATH_IDS)
@pytest.mark.parametrize("tag,layer,kw", FWD_CASES, ids=[c[0] for c in FWD_CASES])
def test_forward_exact(cuda, tag, layer, kw, math):
    plain = all(s.tr == ops.SRC_PLAIN and not s.aff for s in layer.srcs)
    amp = 3 if layer.taps * layer.ctot <= 300 else 1
    run_fwd(layer, math, cuda, tag=tag, amp=amp, stats=plain and kw.get("out") != "nchw", **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("math", [TF32, TF32X3], ids=["tf32", "tf32x3"])
@pytest.mark.parametrize("entry", PLAN_MATRIX, ids=PLAN_IDS)
def test_plan_variants_exact(cuda, monkeypatch, entry, math):
    """Every forced plan variant, integer data with statistics, in both tensor-core modes."""
    tag, env, layer, _, _ = entry
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    amp = 3 if layer.taps * layer.ctot <= 300 else 1
    run_fwd(layer, math, cuda, tag=tag, amp=amp, stats=True)
    run_fwd(layer, math, cuda, tag=tag + "/slope0.25", amp=1, slope=0.25, out="slice", seed=1)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
@pytest.mark.parametrize("math", [TF32, TF32X3], ids=["tf32", "tf32x3"])
@pytest.mark.parametrize("extra", [0, 1, -1], ids=["even", "pipe1_short", "one_less"])
def test_tile_counts_around_the_grid(cuda, monkeypatch, math, extra):
    """Tile counts of 2 * SMs + extra and 3 * SMs + extra (resident and streamed plans): the
    second pipeline of some CTAs runs one tile fewer than the first, or the last CTA gets one
    tile less than the others; and a grid one CTA short of the SM count."""
    sms = _sms()
    run_fwd(L([16], 32, 8, 8 * (2 * sms + extra), N=1), math, cuda, tag="2sms", amp=1, stats=True)
    with monkeypatch.context() as mp:
        mp.setenv("ATOMAI_B200_PLAN", "2,16")
        run_fwd(L([16], 32, 8, 8 * (3 * sms + extra), N=1), math, cuda, tag="3sms", amp=1, stats=True)
    run_fwd(L([16], 16, 8, 8 * (sms - 1), N=1), math, cuda, tag="sms-1", amp=1, stats=True)


DGRAD_CASES = [
    ("d32_64", L([64], 32, 16, 16)),
    ("d16_16_cat", L([16, 16], 16, 16, 16)),
    ("d48_16_cat", L([48, 16], 32, 13, 21)),
    ("d_dil2", L([32], 64, 16, 16, dil=2)),
    ("d_dil4_ragged", L([16], 16, 11, 9, dil=4)),
    ("d_k1x1", L([64], 32, 16, 16, ks=1)),
    ("d_k1x3", L([32], 16, 1, 40, ks=(1, 3))),
    ("d_144", L([144], 64, 8, 16)),
    ("d_to_208", L([208], 32, 8, 16)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("math", MATHS, ids=MATH_IDS)
@pytest.mark.parametrize("tag,layer", DGRAD_CASES, ids=[c[0] for c in DGRAD_CASES])
def test_dgrad_exact(cuda, tag, layer, math):
    amp = 3 if layer.taps * layer.cout <= 300 else 1
    run_dgrad(layer, math, cuda, tag=tag, amp=amp, out_pad=8 if len(layer.srcs) > 1 else 0)


DGRAD_PLAN_ENVS = [{}, {"ATOMAI_B200_PLAN": "0,8"}, {"ATOMAI_B200_PLAN": "1,8"},
                   {"ATOMAI_B200_PLAN": "2,16"}, {"ATOMAI_B200_TMA": "0"}, {"ATOMAI_B200_SMEM_KB": "64"}]


@pytest.mark.gpu
@pytest.mark.parametrize("env", DGRAD_PLAN_ENVS, ids=lambda e: ",".join(f"{k[12:]}={v}" for k, v in e.items()) or "default")
def test_dgrad_plan_variants(cuda, monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    layer = L([16, 16], 32, 16, 24)
    for math in (TF32, TF32X3):
        run_dgrad(layer, math, cuda, tag="dgrad_plan", out_pad=4)
    for data in ("lo_x", "lo_w"):
        run_dgrad(layer, TF32X3, cuda, tag=f"dgrad_plan/{data}", data=data)


WGRAD_CASES = [
    # cib 16 / 32 / 64 with partial channel blocks, Cout not a multiple of 64
    ("w4_20", L([4], 20, 16, 16)),
    ("w16_64", L([16], 64, 16, 16)),
    ("w20_4", L([20], 4, 16, 16)),
    ("w32_68", L([32], 68, 16, 16)),
    ("w40_132", L([40], 132, 16, 16)),
    ("w64_64", L([64], 64, 16, 16)),
    ("w72_20", L([72], 20, 16, 16)),
    ("w128_68", L([128], 68, 8, 16)),
    # kernel sizes, dilation
    ("w_k1x1", L([32], 64, 16, 16, ks=1)),
    ("w_k1x3_h1", L([16], 20, 1, 40, ks=(1, 3))),
    ("w_dil2", L([16], 32, 16, 16, dil=2)),
    ("w_dil4_ragged", L([20], 4, 11, 13, dil=4)),
    # concats and transformed sources
    ("w_cat_48_16", L([48, 16], 32, 16, 16)),
    ("w_cat_20_28", L([20, 28], 20, 16, 16)),
    ("w_affine", L([S(32, aff=True)], 32, 16, 16)),
    ("w_pool", L([S(16, ops.SRC_POOL, aff=True)], 32, 12, 20)),
    ("w_up_bilinear", L([S(16), S(16, ops.SRC_UP_BILINEAR, aff=True)], 16, 16, 16)),
    ("w_up_nearest", L([S(16, ops.SRC_UP_NEAREST)], 20, 16, 24)),
    ("w_src_ld", L([S(20, pad=12)], 20, 16, 16)),
    # tile counts: 1, 2, 3 (one range), many (many ranges), ragged
    ("w_1tile", L([16], 32, 8, 8, N=1)),
    ("w_2tiles_ragged", L([16], 32, 5, 13, N=1)),
    ("w_3tiles", L([32], 64, 8, 24, N=1)),
    ("w_many_tiles", L([16], 16, 64, 64, N=2)),
    ("w_many_ragged", L([40], 20, 37, 45, N=3)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("math", MATHS, ids=MATH_IDS)
@pytest.mark.parametrize("tag,layer", WGRAD_CASES, ids=[c[0] for c in WGRAD_CASES])
def test_wgrad_exact(cuda, tag, layer, math):
    run_wgrad(layer, math, cuda, tag=tag, dy_pad=4 if tag.endswith("ld") else 0)


# ----------------------------------------------------------------------------- exact-fp32 kernels
SIMT_FWD = [
    ("c1_tile", L([1], 32, 40, 64)),
    ("c1_16_dil2", L([1], 16, 24, 30, dil=2)),
    # 70 columns: the last 64-wide tile of conv_c1_tile would be mostly empty, so conv_c1<16> runs
    ("c1_16_forced", L([1], 32, 40, 70)),
    ("pix4", L([16], 3, 20, 24, ks=1)),
    ("pix4_3x3", L([S(8, aff=True)], 4, 13, 17)),
    ("pix8", L([4], 8, 20, 24)),
    ("pix_quad", L([8], 16, 20, 24, ks=1)),
    # pooled source: not a quad-lane shape, so conv_pix<16> runs
    ("pix16_no_quad", L([S(8, ops.SRC_POOL)], 16, 20, 24, ks=1)),
    ("pix16", L([4], 16, 13, 17)),
    ("pix32", L([4], 64, 13, 17)),
    ("generic", L([12], 24, 13, 21)),
    ("generic_cat_pool", L([S(8, ops.SRC_POOL, aff=True), S(4)], 20, 10, 12)),
]
SIMT_WGRAD = [
    ("c1_tile", L([1], 16, 40, 64)),
    ("c1_16", L([1], 16, 24, 30, dil=2)),
    ("small_8_1_3x3", L([2], 8, 20, 24)),
    ("small_16_1_1x3", L([2], 16, 1, 50, ks=(1, 3))),
    ("small_16_2_1x1", L([2], 16, 20, 24, ks=1)),
    ("pix_quad", L([16], 4, 20, 24, ks=1)),
    # pixel stride 17: not a quad-lane shape, so wgrad_small<4, 16, 1, 1> runs
    ("small_4_16_1x1", L([S(16, pad=1)], 3, 20, 24, ks=1)),
    ("small_4_4_3x3", L([8], 3, 20, 24)),
    ("small_4_4_1x3", L([8], 3, 1, 50, ks=(1, 3))),
    ("generic", L([12], 24, 13, 21)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("tag,layer", SIMT_FWD, ids=[c[0] for c in SIMT_FWD])
def test_simt_forward_exact(cuda, tag, layer):
    run_fwd(layer, FP32, cuda, tag=tag, stats=True)


@pytest.mark.gpu
@pytest.mark.parametrize("tag,layer", SIMT_WGRAD, ids=[c[0] for c in SIMT_WGRAD])
def test_simt_wgrad_exact(cuda, tag, layer):
    run_wgrad(layer, FP32, cuda, tag=tag)


def _twice(fn):
    a, b = fn(), fn()
    torch.cuda.synchronize()
    return a, b


@pytest.mark.gpu
@pytest.mark.parametrize("tag,layer", SIMT_FWD, ids=[c[0] for c in SIMT_FWD])
def test_simt_forward_reproducible(cuda, tag, layer):
    """Normal data: two launches of each exact-fp32 forward branch give identical outputs and BN
    statistics (the statistics are ordered cross-CTA sums, not float atomics)."""
    g = _gen("simt_rep", tag)
    inp = _normal_inputs(layer, g, cuda)
    w = torch.randn((layer.cout, layer.ctot) + layer.ks, generator=g).to(cuda)
    b = torch.randn(layer.cout, generator=g).to(cuda)
    d = ops.conv_desc(inp.srcs, layer.N, layer.H, layer.W, layer.cout, layer.ks, layer.dil, 0.01, FP32)
    wp = ops.prep_weights(w, ops.WMODE_FWD, FP32)

    def run():
        o = torch.full((layer.N, layer.H, layer.W, layer.cout), float("nan"), device=cuda)
        st = torch.zeros(2 * layer.cout, device=cuda, dtype=torch.float64)
        ops.conv_fwd(d, wp, b, o, st)
        return o, st

    (o1, s1), (o2, s2) = _twice(run)
    assert _same_bits(o1, o2), f"[{tag}] {layer}: outputs differ between two launches"
    assert torch.equal(s1, s2), f"[{tag}] {layer}: BN statistics differ between two launches"


@pytest.mark.gpu
@pytest.mark.parametrize("tag,layer", SIMT_WGRAD, ids=[c[0] for c in SIMT_WGRAD])
def test_simt_wgrad_reproducible(cuda, tag, layer):
    """Normal data: two launches of each exact-fp32 weight-gradient branch give identical dW."""
    g = _gen("simt_rep_w", tag)
    inp = _normal_inputs(layer, g, cuda)
    _, dyv = nhwc_buf(torch.randn((layer.N, layer.cout, layer.H, layer.W), generator=g).double(), cuda)
    d = ops.conv_desc(inp.srcs, layer.N, layer.H, layer.W, layer.cout, layer.ks, layer.dil, 1.0, FP32)

    def run():
        dw = torch.zeros((layer.cout, layer.ctot) + layer.ks, device=cuda)
        ops.conv_wgrad(d, dyv, dw)
        return dw

    dw1, dw2 = _twice(run)
    assert _same_bits(dw1, dw2), f"[{tag}] {layer}: dW differs between two launches"


# ----------------------------------------------------------------------------- headline geometry
@pytest.mark.gpu
def test_headline_geometry_exact(cuda):
    """32 x 512 x 512 (bench.py's batch): the [16, 16] -> 16 decoder layer and the pooled 16 -> 32
    layer, data non-zero only at a few pixels of the first and last image (corners, tile seams),
    forward with statistics and wgrad bitwise exact at the largest offsets."""
    dev = cuda
    N, H = 32, 512
    g = _gen("headline")
    pts = [(0, 0), (0, H - 1), (H - 1, 0), (H - 1, H - 1), (7, 8), (8, 7), (255, 256), (256, 255),
           (H - 9, H - 8), (127, 383)]

    def sparse(C, h):
        """(N, h, h, C), non-zero at the points (scaled to h) and their lower neighbours of the
        first and the last image"""
        x = torch.zeros(N, h, h, C, device=dev)
        for n in (0, N - 1):
            for (i, j) in pts:
                a, b = i * h // H, j * h // H
                for aa in (a, min(a + 1, h - 1)):
                    x[n, aa, b] = ints(g, (C,), 3, 0.2).float().to(dev)
        return x

    def ref_of(xs64, w64, b64, slope, pool):
        xin = torch.cat(xs64, 1)
        if pool:
            xin = F.max_pool2d(xin, 2, 2)
        return F.leaky_relu(F.conv2d(xin, w64, b64, padding=1), slope)

    for name, cins, cout, pool in (("decoder", [16, 16], 16, False), ("pooled", [16], 32, True)):
        xs = [sparse(c, H) for c in cins]
        Ho = H // 2 if pool else H
        w = ints(g, (cout, sum(cins), 3, 3), 3)
        b = ints(g, (cout,), 1, 0.0)
        srcs = [Source(x, None, None, ops.SRC_POOL if pool else ops.SRC_PLAIN) for x in xs]
        x64 = [x[[0, N - 1]].permute(0, 3, 1, 2).double() for x in xs]
        ref_ends = ref_of(x64, w.to(dev), b.to(dev), 0.25, pool)
        const = F.leaky_relu(b.to(dev), 0.25)
        # statistics: the fp32 partials of one CTA hold at most its share of the tiles (P pixels
        # of background) plus every deviation from the background; y is on a 1/4 grid
        tiles = N * (-(-Ho // 8)) ** 2
        P = -(-tiles // min(tiles, _sms())) * 128
        for k, gk in ((1, 4.0), (2, 16.0)):
            dev_k = (ref_ends.abs() ** k - const.abs().view(1, -1, 1, 1) ** k).abs().sum((0, 2, 3))
            assert float((dev_k + P * const.abs() ** k).max()) * gk < LIMIT, f"headline {name}: stats"
        for math in MATHS:
            d = ops.conv_desc(srcs, N, Ho, Ho, cout, (3, 3), 1, 0.25, math)
            wp = ops.prep_weights(w.float().to(dev), ops.WMODE_FWD, math)
            out = torch.full((N, Ho, Ho, cout), float("nan"), device=dev)
            st = torch.zeros(2 * cout, device=dev, dtype=torch.float64)
            ops.conv_fwd(d, wp, b.float().to(dev), out, st)
            torch.cuda.synchronize()
            ctx = f"[headline {name}] math={MATH_NAMES[math]} plan=({plan_line(d)})"
            for k, n in enumerate((0, N - 1)):
                msg = first_mismatch(out[n], ref_ends[k].permute(1, 2, 0), names="hwc")
                assert msg is None, f"{ctx} image {n}: {msg}"
            mid = out[1:N - 1]
            msg = first_mismatch(mid, const.view(1, 1, 1, -1).expand_as(mid))
            assert msg is None, f"{ctx} images 1..{N - 2}: {msg}"
            y1 = ref_ends.sum((0, 2, 3)) + (N - 2) * Ho * Ho * const
            y2 = (ref_ends ** 2).sum((0, 2, 3)) + (N - 2) * Ho * Ho * const ** 2
            msg = first_mismatch(st, torch.cat([y1, y2]), names="c")
            assert msg is None, f"{ctx} statistics: {msg}"
            del out
            # weight gradient over all 32 x Ho x Ho pixels, dy sparse as well
            dy = sparse(cout, Ho)
            dw = torch.zeros(cout, sum(cins), 3, 3, device=dev)
            ops.conv_wgrad(d, dy, dw)
            torch.cuda.synchronize()
            wref = torch.zeros(cout, sum(cins), 3, 3, device=dev, dtype=torch.float64, requires_grad=True)
            xin = torch.cat(x64, 1)
            if pool:
                xin = F.max_pool2d(xin, 2, 2)
            F.conv2d(xin, wref, None, padding=1).backward(dy[[0, N - 1]].permute(0, 3, 1, 2).double())
            msg = first_mismatch(dw, wref.grad, names=("co", "ci", "ky", "kx"))
            assert msg is None, f"{ctx} wgrad: {msg}"
            del dy, dw
        del xs, srcs


# ============================================================================= (b) correction terms
def _differs(got, ref):
    return bool((got.double() != ref).any())


@pytest.mark.gpu
@pytest.mark.parametrize("data", ["lo_x", "lo_w"])
@pytest.mark.parametrize("entry", PLAN_MATRIX, ids=PLAN_IDS)
def test_correction_terms_forward(cuda, monkeypatch, entry, data):
    """tf32x3 exact on operands with low parts under every plan variant; tf32 is not."""
    tag, env, layer, _, _ = entry
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    run_fwd(layer, TF32X3, cuda, tag=f"{tag}/{data}", data=data, stats=False)
    got, ref = run_fwd(layer, TF32, cuda, tag=f"{tag}/{data}", data=data, expect_exact=False)
    assert _differs(got, ref), f"[{tag}/{data}] tf32 matches float64: the low parts are not exercised"


@pytest.mark.gpu
@pytest.mark.parametrize("data", ["lo_x", "lo_w"])
@pytest.mark.parametrize("tag,layer", DGRAD_CASES, ids=[c[0] for c in DGRAD_CASES])
def test_correction_terms_dgrad(cuda, tag, layer, data):
    run_dgrad(layer, TF32X3, cuda, tag=f"{tag}/{data}", data=data)
    got, ref, _ = run_dgrad(layer, TF32, cuda, tag=f"{tag}/{data}", data=data, expect_exact=False)
    assert _differs(got, ref), f"[{tag}/{data}] tf32 dgrad matches float64"


WGRAD_LO_CASES = [c for c in WGRAD_CASES
                  if all(not s.aff and s.tr in (ops.SRC_PLAIN, ops.SRC_POOL) for s in c[1].srcs)]


@pytest.mark.gpu
@pytest.mark.parametrize("data", ["lo_x", "lo_dy"])
@pytest.mark.parametrize("tag,layer", WGRAD_LO_CASES, ids=[c[0] for c in WGRAD_LO_CASES])
def test_correction_terms_wgrad(cuda, tag, layer, data):
    """wgrad_tc issues (hi, hi), (lo, hi), (hi, lo): exact with low parts on one operand."""
    run_wgrad(layer, TF32X3, cuda, tag=f"{tag}/{data}", data=data)
    got, ref, _, _ = run_wgrad(layer, TF32, cuda, tag=f"{tag}/{data}", data=data, expect_exact=False)
    assert _differs(got, ref), f"[{tag}/{data}] tf32 wgrad matches float64"


# ============================================================================= (c) rounding model
def c_mode(math, K):
    if math == FP32:
        return (K + 2) * 2.0 ** -24
    return (2.0 ** -10 if math == TF32 else 2.0 ** -18) + (K + 2) * 2.0 ** -23


def _normal_inputs(layer, g, dev):
    """Like Inputs, with normal data and random BN affines (plain and pooled sources)."""
    inp = SimpleNamespace(srcs=[], keep=[])
    refs = []
    N, H, W = layer.N, layer.H, layer.W
    for s in layer.srcs:
        h, w = (2 * H, 2 * W) if s.tr == ops.SRC_POOL else (H, W)
        x = torch.randn((N, s.C, h, w), generator=g).double()
        buf, view = nhwc_buf(x, dev, s.pad)
        xr = x.to(dev)
        sc = sh = None
        if s.aff:
            sc = (torch.rand(s.C, generator=g) + 0.5).float() * (torch.randint(0, 2, (s.C,), generator=g) * 2 - 1)
            sh = (torch.randn(s.C, generator=g) * 0.3).float()
            xr = xr * sc.double().to(dev).view(1, -1, 1, 1) + sh.double().to(dev).view(1, -1, 1, 1)
            sc, sh = sc.to(dev), sh.to(dev)
        if s.tr == ops.SRC_POOL:
            xr = F.max_pool2d(xr, 2, 2)
        inp.keep += [buf, sc, sh]
        inp.srcs.append(Source(view, sc, sh, s.tr))
        refs.append(xr)
    inp.x = torch.cat(refs, 1)
    return inp


def _bound_check(tag, got, ref, m, c):
    err = (got.double() - ref).abs()
    ratio = err / (c * m).clamp_min(1e-300)
    worst = float(ratio.max())
    assert worst <= 1.0, (f"[{tag}] error exceeds the model bound: worst |y - y64| / (c m) = {worst:.3g} "
                          f"at {tuple(int(i) for i in (ratio == ratio.max()).nonzero()[0])}")
    return float(err.norm())


def _same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


ROUND_FWD = [
    ("r16_32", L([16], 32, 16, 16)),
    ("r64_64_sub2", L([64], 64, 24, 24)),
    ("r_cat_affine", L([S(16, aff=True), S(16, aff=True)], 16, 16, 16)),
    ("r_pool_affine", L([S(32, ops.SRC_POOL, aff=True)], 80, 12, 12)),
    ("r256_208", L([256], 208, 8, 16)),
    ("r_k1x1", L([64], 32, 16, 16, ks=1)),
    ("r_dil4", L([32], 48, 20, 20, dil=4)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("tag,layer", ROUND_FWD, ids=[c[0] for c in ROUND_FWD])
def test_forward_rounding_model(cuda, tag, layer):
    dev = cuda
    g = _gen("round", tag)
    inp = _normal_inputs(layer, g, dev)
    K = layer.taps * layer.ctot
    w = (torch.randn((layer.cout, layer.ctot) + layer.ks, generator=g) * K ** -0.5).float()
    b = (torch.randn(layer.cout, generator=g) * 0.1).float()
    w64, b64 = w.double().to(dev), b.double().to(dev)
    conv = lambda a, ww, bb: F.conv2d(a, ww, bb, padding=layer.pad, dilation=layer.dil)
    ref = F.leaky_relu(conv(inp.x, w64, b64), 0.01).permute(0, 2, 3, 1)
    m = conv(inp.x.abs(), w64.abs(), b64.abs()).permute(0, 2, 3, 1)
    errs = {}
    for math in MATHS:
        d = ops.conv_desc(inp.srcs, layer.N, layer.H, layer.W, layer.cout, layer.ks, layer.dil, 0.01, math)
        wp = ops.prep_weights(w.to(dev), ops.WMODE_FWD, math)
        runs = []
        for _ in range(2):
            o = torch.full((layer.N, layer.H, layer.W, layer.cout), float("nan"), device=dev)
            st = torch.zeros(2 * layer.cout, device=dev, dtype=torch.float64)
            ops.conv_fwd(d, wp, b.to(dev), o, st)
            runs.append((o, st))
        torch.cuda.synchronize()
        ctx = _ctx(tag, layer, d, math)
        errs[math] = _bound_check(ctx, runs[0][0], ref, m, c_mode(math, K))
        assert _same_bits(runs[0][0], runs[1][0]) and _same_bits(runs[0][1], runs[1][1]), \
            f"{ctx}: two launches differ"
    if K >= 72:
        assert errs[TF32X3] <= errs[TF32] / 8, \
            f"[{tag}] tf32x3 error {errs[TF32X3]:.3g} not 8x below tf32 {errs[TF32]:.3g}"


ROUND_WGRAD = [
    ("rw16_32", L([16], 32, 32, 32)),
    ("rw64_64", L([64], 64, 16, 16, N=4)),
    ("rw_cat_pool", L([S(20, aff=True), S(28, ops.SRC_POOL, aff=True)], 20, 16, 16)),
    ("rw_dil2_ragged", L([32], 68, 21, 19, dil=2)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("tag,layer", ROUND_WGRAD, ids=[c[0] for c in ROUND_WGRAD])
def test_wgrad_rounding_model(cuda, tag, layer):
    dev = cuda
    g = _gen("round_w", tag)
    inp = _normal_inputs(layer, g, dev)
    dy64 = torch.randn((layer.N, layer.cout, layer.H, layer.W), generator=g).float().double().to(dev)

    def wgrad(x, dy):
        w = torch.zeros((layer.cout, layer.ctot) + layer.ks, device=dev, dtype=torch.float64,
                        requires_grad=True)
        F.conv2d(x, w, None, padding=layer.pad, dilation=layer.dil).backward(dy)
        return w.grad

    ref, m = wgrad(inp.x, dy64), wgrad(inp.x.abs(), dy64.abs())
    K = layer.N * layer.H * layer.W
    _, dyv = nhwc_buf(dy64, dev)
    errs = {}
    for math in MATHS:
        d = ops.conv_desc(inp.srcs, layer.N, layer.H, layer.W, layer.cout, layer.ks, layer.dil, 1.0, math)
        runs = []
        for _ in range(2):
            dw = torch.zeros((layer.cout, layer.ctot) + layer.ks, device=dev)
            ops.conv_wgrad(d, dyv, dw)
            runs.append(dw)
        torch.cuda.synchronize()
        ctx = f"[{tag}] {layer} wgrad math={MATH_NAMES[math]}"
        errs[math] = _bound_check(ctx, runs[0], ref, m, c_mode(math, K))
        assert _same_bits(runs[0], runs[1]), f"{ctx}: two launches differ"
    assert errs[TF32X3] <= errs[TF32] / 8, \
        f"[{tag}] wgrad tf32x3 error {errs[TF32X3]:.3g} not 8x below tf32 {errs[TF32]:.3g}"


@pytest.mark.gpu
def test_dgrad_rounding_model(cuda):
    dev = cuda
    layer = L([16, 48], 64, 16, 16)
    g = _gen("round_d")
    N, H, W = layer.N, layer.H, layer.W
    dy64 = torch.randn((N, layer.cout, H, W), generator=g).float().double().to(dev)
    w = (torch.randn((layer.cout, layer.ctot, 3, 3), generator=g) * 0.05).float()
    xin = torch.zeros(N, layer.ctot, H, W, device=dev, dtype=torch.float64, requires_grad=True)
    F.conv2d(xin, w.double().to(dev), None, padding=1).backward(dy64)
    ref = xin.grad.permute(0, 2, 3, 1)
    xin2 = torch.zeros_like(xin, requires_grad=True)
    F.conv2d(xin2, w.double().abs().to(dev), None, padding=1).backward(dy64.abs())
    m = xin2.grad.permute(0, 2, 3, 1)
    K = 9 * layer.cout
    _, dyv = nhwc_buf(dy64, dev)
    errs = {}
    for math in MATHS:
        d = ops.conv_desc([Source(dyv)], N, H, W, layer.ctot, (3, 3), 1, 1.0, math)
        wp = ops.prep_weights(w.to(dev), ops.WMODE_DGRAD, math)
        o = torch.full((N, H, W, layer.ctot), float("nan"), device=dev)
        ops.conv_fwd(d, wp, None, o, None)
        o2 = torch.full_like(o, float("nan"))
        ops.conv_fwd(d, wp, None, o2, None)
        torch.cuda.synchronize()
        ctx = _ctx("dgrad_round", layer, d, math)
        errs[math] = _bound_check(ctx, o, ref, m, c_mode(math, K))
        assert _same_bits(o, o2), f"{ctx}: two launches differ"
    assert errs[TF32X3] <= errs[TF32] / 8, (errs[TF32X3], errs[TF32])
