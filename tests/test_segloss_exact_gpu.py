"""Exact and float64 parity of the segmentation objectives beyond cross-entropy (segloss.cu: dice
sums, finalise and backward, the focal finalise, the IoU histogram and finalise) and of the VAE
reconstruction loss (rowloss in frontend.cu), driven through the C ABI (`atomai_b200.ops`).
NHWC operands sit in NaN-filled buffers (Slot of test_elementwise_exact_gpu.py) with padded pixel
strides and a misaligned start; the references are float64 (oracle/seg_objectives_ref.py).

Rounding model (U = 2^-24; expf is CUDA's 2-ulp expf, so 4 U relative, plus |x - max| U for its
rounded argument; log1pf 1 ulp; divisions correctly rounded):
(a) dice_sums.  Softmax probability p_c: relative error (4 + |x_c - m|) U + max_c of the same
    + (C + 1) U; sigmoid: (4 U e/(1+e) + 2 U), 1 - s adds U (1 - s) to the absolute error.  A cell
    is a per-thread serial float sum of n_t terms (n_t rows of the CTA's row chunk per warp), an
    ordered 8-warp float sum (binary: a 5-level warp butterfly and 8 warps) and an ordered double
    sum over row chunks: bound = sum of the term errors + (n_t + 7) U sum|terms| (binary
    n_t + 12) + ny 2^-53 sum|terms|.  Exact tier: equal logits with C a power of two give p = 1/C,
    logits 200 apart give p in {0, 1}, binary logits 0 / +-200 give s in {0.5, 0, 1}; every cell
    must then equal the float64 count formula bit for bit.
(b) dice_finalize.  coef is computed in double and rounded once: bitwise equal to the float64
    restatement with eps rounded to fp32.  loss: one fp32 rounding + (n_t + 15) 2^-53 sum|2I/d| / K.
(c) dice_bwd, from the same fp32 coef: G = t A + B one rounding, p as in (a), the dot product
    sum_c p_c G_c C + 2 roundings, G - dot one rounding, three products and the gscale product.
(d) focal_finalize: double arithmetic, one fp32 rounding; 1 - exp(-CE) loses 2^-52 / (1 - pt)
    relative, which the power gamma (gamma - 1 for the tail) multiplies.
(e) iou_hist counts are integers: equal to the oracle's.  Probabilities stay MARGIN away from the
    threshold except in the exact-tie cases, where p = thresh exactly.  iou_finalize is the
    float32 formula over exact int64 row / column sums rounded once: bitwise equal to that.
(f) rowloss: per-thread serial float sums of n_t = ceil(D / (256 gx)) terms, a warp butterfly,
    8 warps and one double atomic per block: (n_t + 12) U sum|terms| + term errors.
(g) Every ordered reduction and every finalise is bitwise identical across two launches (rowloss's
    `out` only with one block per row: its blocks add with double atomics); refusals raise
    NativeError with the outputs untouched.
Largest |err| / bound observed on the first run (H100 80GB HBM3, 700 W power limit; printed by
test_zz_report_measured under -s): 0.96 focal_finalize, 0.87 dice_finalize loss, 0.74 rowloss
BCE, 0.67 dice_bwd, 0.66 rowloss MSE, 0.37 dice_sums multi-class, 0.11 dice_sums binary.  The
exact tiers, the coef, the IoU counts and iou_finalize are bitwise.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from atomai_b200 import _C, ops
from oracle import seg_objectives_ref as ref
from test_elementwise_exact_gpu import NAN_BITS, U, Slot, _gen, assert_intact, exact_case, \
    first_mismatch, same_bits, sm_count

gpu = pytest.mark.gpu
D53 = 2.0 ** -53
MARGIN = 1e-3
WS_DOUBLES = 1 << 21           # kDiceWsDoubles


# ----------------------------------------------------------------------------- helpers
def bound_check(got, ref64, bound, what):
    """|got - ref64| <= bound elementwise; returns the largest err / bound."""
    got, ref64, bound = got.double(), ref64.double(), bound.double()
    err = (got - ref64).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.numel()} outside the bound, first at "
                             f"{idx}: got {float(got[idx])!r}, want {float(ref64[idx])!r}, "
                             f"bound {float(bound[idx])!r}")
    return float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0


def bitwise(got, want, what):
    msg = first_mismatch(got, want)
    assert msg is None, f"{what}: {msg}"


def nan_intact(t, what):
    bits = t.view(torch.int32) if t.dtype == torch.float32 else t
    ok = bits == NAN_BITS if t.dtype == torch.float32 else torch.isnan(t)
    assert bool(ok.all()), f"{what}: output was written"


def cdiv(a, b):
    return -(-a // b)


def dice_ny(rows, W, C):
    """Row chunks of the multi-class dice_sums launch (atomai_b200_dice_sums)."""
    ncb = cdiv(W, 32)
    per_chunk = 2 * C * 32 * ncb
    sm_cap = cdiv(sm_count() * 4, ncb)
    ny = max(1, min(sm_cap, cdiv(rows, 8), WS_DOUBLES // per_chunk, 65535))
    return ny, sm_cap


def softmax_err(l64):
    """(p, relative error bound of the kernel's fp32 probability) of NHWC float64 logits."""
    m = l64.max(-1, keepdim=True).values
    e = torch.exp(l64 - m)
    p = e / e.sum(-1, keepdim=True)
    rel_e = (4 + (l64 - m).abs()) * U
    rel = rel_e + rel_e.max(-1, keepdim=True).values + (l64.shape[-1] + 1) * U
    return p, p * rel + 1e-44           # 1e-44: expf underflow to zero / subnormal results


def sigmoid_err(x64):
    s = torch.sigmoid(x64)
    e = torch.exp(-x64)
    err_s = s * (4 * U * e / (1 + e) + 2 * U) + 1e-44
    return s, err_s


def labels_mc(g, N, H, W, C):
    y = torch.randint(0, C, (N, H, W), generator=g)
    col = y[..., ::3]
    col[col == 0] = 1 % C               # class 0 absent from every third column (I = 0 there)
    y[..., ::3] = col
    return y


# ----------------------------------------------------------------------------- dice_sums, C > 1
ROWS = ("few", "mid", "cap")


def rows_shape(kind, W, C):
    if kind == "few":
        return 1, 3                     # fewer rows than warps
    if kind == "mid":
        return 2, 19
    ny_cap = cdiv(sm_count() * 4, cdiv(W, 32))
    rows = 16 * ny_cap + 5              # enough rows for ny to reach the SM cap, uneven chunks
    return 2, cdiv(rows, 2)


def run_dice_sums(L, y, K):
    outs = []
    for _ in range(2):
        cells = torch.full((2 * K,), float("nan"), dtype=torch.float64, device=L.t.device)
        ops.dice_sums(L.t, y, cells)
        outs.append(cells)
    torch.cuda.synchronize()
    same_bits(outs[0], outs[1], "dice cells reproducible")
    return outs[0]


@gpu
@pytest.mark.parametrize("lay", [(0, 0), (3, 1)], ids=["ld=C", "padded"])
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("W", [1, 7, 31, 32, 33, 100, 512])
@pytest.mark.parametrize("C", [2, 3, 5, 16])
def test_dice_sums_multiclass(cuda, C, W, rows, lay):
    N, H = rows_shape(rows, W, C)
    R = N * H
    ny, sm_cap = dice_ny(R, W, C)
    if rows == "cap":
        assert ny == sm_cap, (ny, sm_cap)
    g = _gen("dice_mc", C, W, rows, lay)
    y = labels_mc(g, N, H, W, C)
    yd = y.to(cuda)
    t = F.one_hot(y, C).double()                             # (N, H, W, C)
    K = C * W
    tiers = ["onehot"] + (["uniform"] if C & (C - 1) == 0 else [])
    for tier in tiers:
        if tier == "uniform":
            l = torch.randn((N, H, W, 1), generator=g).float().double().expand(N, H, W, C)
            assert bool((l == l[..., :1]).all())
            p = torch.full((N, H, W, C), 1.0 / C, dtype=torch.float64)
            unit = 1.0 / C
        else:
            hot = torch.randint(0, C, (N, H, W), generator=g)
            l = torch.where(F.one_hot(hot, C).bool(), 0.0, -200.0).double() + \
                torch.randint(-3, 4, (N, H, W, 1), generator=g).double()
            p = F.one_hot(hot, C).double()
            unit = 1.0
        L = Slot((N, H, W, C), cuda, lay, l.contiguous().float())
        cells = run_dice_sums(L, yd, K).cpu()
        I = (p * t).sum((0, 1)).T.reshape(-1)
        S = (p + t).sum((0, 1)).T.reshape(-1)
        exact_case(S, unit, f"dice {tier}")
        bitwise(cells[:K], I, f"dice_sums C={C} W={W} rows={R} {tier} I")
        bitwise(cells[K:], S, f"dice_sums C={C} W={W} rows={R} {tier} S")
        assert_intact(f"dice_sums {tier}", L)
    # normal tier: 2 randn, pixels at +-80
    l = (torch.randn((N, H, W, C), generator=g) * 2).float().double()
    l.view(-1, C)[::5, 0] = 80.0
    l.view(-1, C)[2::7, C - 1] = -80.0
    L = Slot((N, H, W, C), cuda, lay, l.float())
    cells = run_dice_sums(L, yd, K).cpu()
    p, errp = softmax_err(l)
    termI, termS = p * t, p + t
    eI, eS = errp * t, errp + U * termS
    n_t = cdiv(cdiv(R, ny), 8)              # rows of the largest chunk per warp
    slack = (n_t + 7) * U + ny * D53
    bI = (eI.sum((0, 1)) + slack * termI.sum((0, 1))).T.reshape(-1)
    bS = (eS.sum((0, 1)) + slack * termS.sum((0, 1))).T.reshape(-1)
    i64, s64 = ref.dice_cells(l.permute(0, 3, 1, 2), y)
    rI = bound_check(cells[:K], i64, bI, f"dice_sums C={C} W={W} rows={R} I")
    rS = bound_check(cells[K:], s64, bS, f"dice_sums C={C} W={W} rows={R} S")
    MEASURED.setdefault("dice_sums", []).append(max(rI, rS))
    assert_intact("dice_sums randn", L)


@gpu
def test_dice_sums_widest_accepted(cuda):
    """C = 16, W = 65536: one row chunk holds exactly kDiceWsDoubles partials, ny = 1."""
    N, H, W, C = 1, 3, 65536, 16
    assert 2 * C * 32 * (W // 32) == WS_DOUBLES and dice_ny(N * H, W, C)[0] == 1
    g = _gen("dice_wide")
    y = labels_mc(g, N, H, W, C)
    l = torch.randn((N, H, W, 1), generator=g).float().double().expand(N, H, W, C).contiguous()
    L = Slot((N, H, W, C), cuda, (0, 0), l.float())
    cells = run_dice_sums(L, y.to(cuda), C * W).cpu()
    t = F.one_hot(y, C).double()
    I = (t / C).sum((0, 1)).T.reshape(-1)
    S = (t + 1.0 / C).sum((0, 1)).T.reshape(-1)
    bitwise(cells, torch.cat([I, S]), "dice_sums C=16 W=65536")


# ----------------------------------------------------------------------------- dice_sums, C == 1
BIN_N = (1, 255, 256, 257, "multi")


def bin_labels(g, n, ltype):
    if ltype == "int64":
        return torch.randint(-1, 3, (n,), generator=g)       # -1 and 2 count as neither class
    vals = torch.tensor([0.0, 1.0, 0.5, 1.7, -0.5, 2.0, -1.0, 0.999])
    return vals[torch.randint(0, len(vals), (n,), generator=g)]


@gpu
@pytest.mark.parametrize("ltype", ["int64", "float32"])
@pytest.mark.parametrize("lay", [(0, 0), (2, 1)], ids=["ld=1", "padded"])
@pytest.mark.parametrize("npix", BIN_N)
def test_dice_sums_binary(cuda, npix, lay, ltype):
    n = npix if npix != "multi" else 3 * 8 * sm_count() * 256 + 123   # grid-stride loop x 4
    N, H, W = 1, 1, n
    g = _gen("dice_bin", npix, lay, ltype)
    yl = bin_labels(g, n, ltype)
    y = yl.reshape(N, 1, H, W).to(cuda)
    yt = yl.long()                                        # the reference's truncation
    t0, t1 = (yt == 1).double(), (yt == 0).double()
    for tier in ("zero", "pm200"):
        x = torch.zeros(n, dtype=torch.float64) if tier == "zero" else \
            torch.where(torch.rand(n, generator=g) < 0.5, 200.0, -200.0).double()
        s = torch.full((n,), 0.5, dtype=torch.float64) if tier == "zero" else (x > 0).double()
        L = Slot((N, H, W, 1), cuda, lay, x.reshape(N, H, W, 1).float())
        cells = run_dice_sums(L, y, 2).cpu()
        want = torch.stack([(s * t0).sum(), ((1 - s) * t1).sum(), (s + t0).sum(), (1 - s + t1).sum()])
        exact_case(want, 0.5, "binary dice")
        bitwise(cells, want, f"dice_sums binary n={n} {tier}")
        assert_intact("dice_sums binary", L)
    x = (torch.randn(n, generator=g) * 2).float().double()
    x[::5] = 80.0
    x[2::7] = -80.0
    L = Slot((N, H, W, 1), cuda, lay, x.reshape(N, H, W, 1).float())
    cells = run_dice_sums(L, y, 2).cpu()
    s, es = sigmoid_err(x)
    q = 1 - s
    eq = es + U * q
    terms = [s * t0, q * t1, s + t0, q + t1]
    errs = [es * t0, eq * t1, es + U * (s + t0), eq + U * (q + t1)]
    grid = min(cdiv(n, 256), 8 * sm_count())
    n_t = cdiv(n, grid * 256)
    slack = (n_t + 12) * U + grid * D53
    bound = torch.stack([e.sum() + slack * tm.sum() for e, tm in zip(errs, terms)])
    i64, s64 = ref.dice_cells(x.reshape(N, 1, H, W), yl.reshape(N, 1, H, W).double())
    r = bound_check(cells, torch.cat([i64, s64]), bound, f"dice_sums binary n={n}")
    MEASURED.setdefault("dice_sums binary", []).append(r)


# ----------------------------------------------------------------------------- dice_finalize
def finalize_mirror(cells, eps):
    """The kernel's double arithmetic, rounded to fp32 once."""
    K = cells.numel() // 2
    I, d = cells[:K], cells[K:] + float(np.float32(eps))
    g = 2.0 / K
    return (-g / d).float(), (g * I / (d * d)).float(), 2.0 * I / d


@gpu
@pytest.mark.parametrize("K", [1, 2, 255, 256, 257, 16 * 65536])
def test_dice_finalize(cuda, K):
    g = _gen("dice_fin", K)
    S = torch.exp(torch.randn(K, generator=g, dtype=torch.float64) * 3)
    S[::4] = 0.0                                          # empty cells: only eps remains
    I = S * torch.rand(K, generator=g, dtype=torch.float64)
    I[::3] = 0.0
    cells = torch.cat([I, S]).to(cuda)
    eps = 1e-7
    runs = []
    for _ in range(2):
        buf = torch.full((2 * K + 2,), float("nan"), device=cuda)
        loss = torch.full((1,), float("nan"), device=cuda)
        ops.dice_finalize(cells, eps, loss, buf[1:-1])
        runs.append((loss, buf))
    loss_only = torch.full((1,), float("nan"), device=cuda)
    ops.dice_finalize(cells, eps, loss_only)
    torch.cuda.synchronize()
    same_bits(runs[0][0], runs[1][0], "dice_finalize loss reproducible")
    same_bits(runs[0][1], runs[1][1], "dice_finalize coef reproducible")
    same_bits(runs[0][0], loss_only, "dice_finalize loss without coef")
    loss, buf = runs[0][0].cpu(), runs[0][1].cpu()
    nan_intact(buf[:1], "coef guard")
    nan_intact(buf[-1:], "coef guard")
    A, B, q = finalize_mirror(cells.cpu(), eps)
    bitwise(buf[1:K + 1], A, f"dice_finalize K={K} A")
    bitwise(buf[K + 1:-1], B, f"dice_finalize K={K} B")
    # the oracle's coefficients and loss in float64 from the same cells
    A64, B64 = ref.dice_coefficients(I, S, float(np.float32(eps)))
    assert bool(((A - A64).abs() <= U * A64.abs()).all() and ((B - B64).abs() <= U * B64.abs()).all())
    l64 = 1 - q.mean()
    n_t = cdiv(K, 256)
    bound = U * abs(float(l64)) + (n_t + 15) * D53 * float(q.abs().sum()) / K + 2 * D53
    r = bound_check(loss, l64.reshape(1), torch.tensor([bound]), f"dice_finalize K={K} loss")
    MEASURED.setdefault("dice_finalize loss", []).append(r)


# ----------------------------------------------------------------------------- dice_bwd
def dice_bwd_ref(l64, y, coef, C, W, gscale):
    """float64 dL/dlogits from the fp32 coef the kernel reads, and its error bound."""
    coef = coef.double()
    K = coef.numel() // 2
    if C == 1:
        x = l64[..., 0]
        yl = y.reshape(x.shape).long()
        s, es = sigmoid_err(x)
        G0 = torch.where(yl == 1, coef[0], 0.0) + coef[2]
        G1 = torch.where(yl == 0, coef[1], 0.0) + coef[3]
        dG = G0 - G1
        eG = U * (G0.abs() + G1.abs() + dG.abs())
        sq = s * (1 - s)
        esq = sq * (es / s + 2 * U) + s * es
        d = sq * dG * gscale
        b = gscale * (esq * dG.abs() + sq * eG + 4 * U * (sq * dG).abs())
        return d[..., None], b[..., None]
    A = coef[:K].reshape(C, W).T                           # (W, C)
    Bc = coef[K:].reshape(C, W).T
    t = F.one_hot(y, C).double()
    G = t * A + Bc
    eG = U * G.abs()
    p, ep = softmax_err(l64)
    dot = (p * G).sum(-1, keepdim=True)
    M = (p * G.abs()).sum(-1, keepdim=True)
    e_dot = (ep * G.abs() + p * eG).sum(-1, keepdim=True) + (C + 2) * U * M
    diff = G - dot
    d = p * diff * gscale
    b = gscale * (p * (eG + e_dot + U * diff.abs()) + ep * diff.abs() + 4 * U * (p * diff).abs())
    return d, b


BWD_CASES = [(2, 5, 7, 1, "int64"), (2, 5, 7, 1, "float32"), (1, 9, 33, 3, "int64"),
             (2, 6, 40, 5, "int64"), (1, 4, 64, 16, "int64"), (3, 41, 300, 1, "float32"),
             (2, 37, 129, 3, "int64")]


@gpu
@pytest.mark.parametrize("gdev", [False, True], ids=["gscale", "gscale_dev"])
@pytest.mark.parametrize("case", BWD_CASES, ids=lambda c: "x".join(map(str, c)))
def test_dice_bwd(cuda, case, gdev):
    N, H, W, C, ltype = case
    g = _gen("dice_bwd", case, gdev)
    l = (torch.randn((N, H, W, C), generator=g) * 2).float().double()
    l.view(-1, C)[::9, 0] = 80.0
    l.view(-1, C)[4::11, C - 1] = -80.0
    if C == 1:
        yl = bin_labels(g, N * H * W, ltype).reshape(N, 1, H, W)
        y64 = yl.double()
    else:
        yl = labels_mc(g, N, H, W, C)
        y64 = yl
    y = yl.to(cuda)
    L = Slot((N, H, W, C), cuda, (3, 1), l.float())
    K = 2 if C == 1 else C * W
    cells = run_dice_sums(L, y, K)
    coef = torch.full((2 * K,), float("nan"), device=cuda)
    loss = torch.full((1,), float("nan"), device=cuda)
    ops.dice_finalize(cells, 1e-7, loss, coef)
    gscale, gd = (0.75, torch.tensor([1.5], device=cuda)) if gdev else (1.125, None)
    outs = []
    for _ in range(2):
        D = Slot((N, H, W, C), cuda, (2, 0))
        ops.dice_bwd(L.t, y, coef, D.t, gscale, gd)
        outs.append(D)
    torch.cuda.synchronize()
    what = f"dice_bwd {case} gscale_dev={gdev}"
    same_bits(outs[0].t, outs[1].t, what + " reproducible")
    assert_intact(what, L, outs[0])
    d64, b = dice_bwd_ref(l, yl[:, 0] if C == 1 else yl, coef.cpu(), C, W, 1.125)
    r = bound_check(outs[0].t.cpu(), d64, b + 1e-44, what)
    MEASURED.setdefault("dice_bwd", []).append(r)
    # end to end against float64 autograd of the oracle's dice_loss
    x64 = l.permute(0, 3, 1, 2).clone().requires_grad_(True)
    l_ref = ref.dice_loss(x64, y64)
    (l_ref * 1.125).backward()
    assert abs(float(loss) - l_ref.item()) <= 1e-5 * abs(l_ref.item()), (float(loss), l_ref.item())
    gref = x64.grad.permute(0, 2, 3, 1)
    rel = float((outs[0].t.cpu().double() - gref).abs().max() / gref.abs().max())
    assert rel <= 1e-5, (what, rel)


@gpu
@pytest.mark.parametrize("C", [1, 3])
def test_dice_empty_batch(cuda, C):
    """N = 0: the cells are zeroed on the stream and the loss is the reference's 1.0."""
    from atomai_b200.losses_metrics import dice_loss
    H, W = 4, 6
    K = 2 if C == 1 else C * W
    big = torch.zeros((1, H, W, C), device=cuda)
    lab = torch.zeros((1, H, W), dtype=torch.int64, device=cuda)
    for logits, labels in ((big[:0], lab[:0]), (torch.empty((0, H, W, C), device=cuda),
                                                torch.empty((0, H, W), dtype=torch.int64,
                                                            device=cuda))):
        cells = torch.full((2 * K,), float("nan"), dtype=torch.float64, device=cuda)
        ops.dice_sums(logits, labels, cells)
        loss = torch.full((1,), float("nan"), device=cuda)
        ops.dice_finalize(cells, 1e-7, loss)
        torch.cuda.synchronize()
        assert bool((cells == 0).all()) and float(loss) == 1.0
    x = torch.zeros((0, C, H, W), device=cuda, requires_grad=True)
    y = torch.zeros((0, 1, H, W) if C == 1 else (0, H, W), device=cuda,
                    dtype=torch.float32 if C == 1 else torch.int64)
    out = dice_loss()(x, y)
    out.backward()
    assert out.item() == 1.0 == float(ref.dice_loss(x.detach().cpu().double(), y.cpu()))
    assert x.grad.shape == x.shape


# ----------------------------------------------------------------------------- focal_finalize
CES = [0.0, 1e-8, 1e-4, 0.01, 0.3, 1.0, 3.0, 10.0, 50.0]


@gpu
@pytest.mark.parametrize("alpha", [0.25, 0.5, 1.0])
@pytest.mark.parametrize("gamma", [0.0, 0.5, 1.0, 2.0, 3.7])
def test_focal_finalize(cuda, gamma, alpha):
    worst = 0.0
    for i, ce in enumerate(CES):
        count = (1, 1000, 12345)[i % 3]
        bce = torch.tensor([ce * count], dtype=torch.float64, device=cuda)
        outs = []
        for _ in range(2):
            loss = torch.full((1,), float("nan"), device=cuda)
            fac = torch.full((1,), float("nan"), device=cuda)
            ops.focal_finalize(bce, count, alpha, gamma, loss, fac)
            outs.append((loss, fac))
        torch.cuda.synchronize()
        same_bits(outs[0][0], outs[1][0], "focal loss reproducible")
        same_bits(outs[0][1], outs[1][1], "focal factor reproducible")
        lk, fk = float(outs[0][0]), float(outs[0][1])
        ce64 = torch.tensor(float(bce) / count, dtype=torch.float64)
        a, gm = float(np.float32(alpha)), float(np.float32(gamma))
        pt = torch.exp(-ce64)
        q = 1 - pt
        l64 = float(a * q ** gm * ce64)
        f64 = float(ref.focal_factor(ce64, a, gm))
        # autograd of the oracle's focal_loss with respect to CE, through one logit with t = 0
        if ce > 0:
            x = torch.tensor([math.log(math.expm1(ce64.item()))], dtype=torch.float64,
                             requires_grad=True)
            t0 = torch.zeros(1, dtype=torch.float64)
            lo = ref.focal_loss(x, t0, a, gm)
            lo.backward()
            # the oracle's CE of this logit (torch's BCE loses ~1e-7 relative at CE = 1e-8)
            ce_t = F.binary_cross_entropy_with_logits(x.detach(), t0)
            f_ag = float(x.grad) / float(torch.sigmoid(x.detach()))
            f_t = float(ref.focal_factor(ce_t, a, gm))
            l_t = float(a * (1 - torch.exp(-ce_t)) ** gm * ce_t)
            assert abs(f_ag - f_t) <= 1e-10 * abs(f_t), (ce, f_ag, f_t)
            assert abs(lo.item() - l_t) <= 1e-10 * abs(l_t), (ce, lo.item(), l_t)
        what = f"focal gamma={gamma} alpha={alpha} ce={ce}"
        if ce == 0:
            assert lk == 0.0, what
            if 0 < gamma < 1:           # inf * 0 in the tail, as in autograd
                assert math.isnan(fk) and math.isnan(f64), (what, fk, f64)
            else:
                assert fk == float(np.float32(f64)), (what, fk, f64)
            continue
        qf = float(q)
        A = a * qf ** gm
        tail = f64 - A
        bl = U * abs(l64) + 2 ** -52 * (8 + gm / qf) * abs(l64)
        bf = U * abs(f64) + 2 ** -52 * (8 * abs(f64) + (gm * A + abs(gm - 1) * abs(tail)) / qf)
        worst = max(worst, abs(lk - l64) / bl, abs(fk - f64) / bf)
        assert abs(lk - l64) <= bl, (what, lk, l64, bl)
        assert abs(fk - f64) <= bf, (what, fk, f64, bf)
    MEASURED.setdefault("focal_finalize", []).append(worst)


# ----------------------------------------------------------------------------- IoU
def iou_labels(g, n, nc, ltype):
    y = torch.randint(0, nc, (n,), generator=g)
    out = torch.randint(0, 4, (n,), generator=g)
    bad = torch.tensor([-1, nc, 1000])[torch.randint(0, 3, (n,), generator=g)]
    if ltype == "int64":
        return torch.where(out == 0, bad, y)
    frac = torch.tensor([0.0, 0.5, 0.7])[torch.randint(0, 3, (n,), generator=g)]
    yf = y.double() + frac
    yf = torch.where(out == 0, bad.double(), yf)
    yf[::13] = -0.5                                   # truncates to class 0
    return yf.float()


def iou_values(g, shape, C, act, thresh):
    """fp32 logits (or raw values) with every class probability MARGIN away from thresh."""
    N, H, W = shape
    scale = 2.0 if C <= 5 else 4.0

    def draw(k):
        return (torch.randn((k, C), generator=g) * scale) if act else torch.rand((k, C), generator=g)

    x = draw(N * H * W).float().double()
    while True:
        p = (torch.sigmoid(x) if C == 1 else torch.softmax(x, -1)) if act else x
        bad = ((p - thresh).abs() < MARGIN).any(-1)
        if not bool(bad.any()):
            return x.reshape(N, H, W, C)
        x[bad] = draw(int(bad.sum())).float().double()


def oracle_counts(y, x, thresh, act):
    return ref.iou_counts(y, x.permute(0, 3, 1, 2), thresh, act).reshape(-1)


@gpu
@pytest.mark.parametrize("ltype", ["int64", "float32"])
@pytest.mark.parametrize("thresh", [0.3, 0.5, 0.9])
@pytest.mark.parametrize("act", [True, False], ids=["act", "raw"])
@pytest.mark.parametrize("C", [1, 2, 3, 5, 33, 64])
def test_iou_hist(cuda, C, act, thresh, ltype):
    N, H, W = 2, 13, 29                                # 377 pixels per image
    nc = max(C, 2)
    g = _gen("iou", C, act, thresh, ltype)
    x = iou_values(g, (N, H, W), C, act, thresh)
    yl = iou_labels(g, N * H * W, nc, ltype).reshape(N, H, W)
    y = yl.to(cuda)
    L = Slot((N, H, W, C), cuda, (1, 1), x.float())
    want = oracle_counts(yl, x, thresh, act)
    full = torch.zeros(nc * nc, dtype=torch.int64, device=cuda)
    ops.iou_hist(L.t, y, thresh, full, activation=act)
    halves = torch.zeros(nc * nc, dtype=torch.int64, device=cuda)
    ops.iou_hist(L.t[:1], y[:1].contiguous(), thresh, halves, activation=act)
    ops.iou_hist(L.t[1:], y[1:].contiguous(), thresh, halves, activation=act)
    torch.cuda.synchronize()
    what = f"iou_hist C={C} act={act} thresh={thresh} {ltype}"
    assert torch.equal(full.cpu(), want), what
    assert torch.equal(halves.cpu(), want), what + " (two launches)"
    assert_intact(what, L)
    if C > 2 and thresh == 0.3 and not act:
        # several classes above the threshold: the summed index and its clip to 0 are reached
        s = ((x > thresh).long() * torch.arange(C)).sum(-1)
        assert bool((s > C - 1).any())
        assert C > 5 or bool(((s > 0) & (s <= C - 1)).any())


@gpu
@pytest.mark.parametrize("C", [1, 3, 64])
def test_iou_hist_grid_stride(cuda, C):
    N, H, W = 3, 301, 307
    assert N * H * W > 8 * sm_count() * 256
    g = _gen("iou_big", C)
    x = iou_values(g, (N, H, W), C, True, 0.5)
    yl = iou_labels(g, N * H * W, max(C, 2), "int64").reshape(N, H, W)
    L = Slot((N, H, W, C), cuda, (0, 0), x.float())
    counts = torch.zeros(max(C, 2) ** 2, dtype=torch.int64, device=cuda)
    ops.iou_hist(L.t, yl.to(cuda), 0.5, counts)
    torch.cuda.synchronize()
    assert torch.equal(counts.cpu(), oracle_counts(yl, x, 0.5, True))


@gpu
@pytest.mark.parametrize("C", [1, 2, 3, 4, 5, 64])
def test_iou_hist_exact_ties(cuda, C):
    """p == thresh counts as below (the comparison is strict)."""
    N, H, W = 1, 7, 45
    nc = max(C, 2)
    g = _gen("iou_ties", C)
    yl = torch.randint(0, nc, (N, H, W), generator=g)
    y = yl.to(cuda)
    cases = []
    if C & (C - 1) == 0:            # equal logits: p = 1/C (C = 1: sigmoid(0) = 1/2) exactly
        x = torch.randn((N, H, W, 1), generator=g).float().double().expand(N, H, W, C)
        if C == 1:
            x = torch.zeros((N, H, W, 1), dtype=torch.float64)
        p = 0.5 if C == 1 else 1.0 / C
        cases += [(x, p, True), (x, float(np.nextafter(np.float32(p), np.float32(0))), True)]
    raw = torch.tensor([0.25, 0.5, 0.75], dtype=torch.float64)[
        torch.randint(0, 3, (N, H, W, C), generator=g)]
    cases += [(raw, 0.5, False), (raw, 0.25, False)]
    for x, thresh, act in cases:
        L = Slot((N, H, W, C), cuda, (0, 0), x.contiguous().float())
        counts = torch.zeros(nc * nc, dtype=torch.int64, device=cuda)
        ops.iou_hist(L.t, y, thresh, counts, activation=act)
        torch.cuda.synchronize()
        want = oracle_counts(yl, x, thresh, act)
        assert torch.equal(counts.cpu(), want), (C, thresh, act)
        if act and thresh == (0.5 if C == 1 else 1.0 / C):
            assert int(want.reshape(nc, nc)[:, 1:].sum()) == 0    # no class above p = thresh


def iou_mirror(counts, nc):
    """The kernel's float32 arithmetic over exact int64 row / column sums."""
    h = counts.reshape(nc, nc).numpy()
    s = np.float32(0)
    for i in range(nc):
        a, b, d = np.float32(int(h[i].sum())), np.float32(int(h[:, i].sum())), np.float32(h[i, i])
        s = np.float32(s + d / np.float32(np.float32(np.float32(a + b) - d) + np.float32(1e-10)))
    return float(np.float32(s / np.float32(nc)))


@gpu
@pytest.mark.parametrize("big", [False, True], ids=["counts<2^24", "counts>2^24"])
@pytest.mark.parametrize("nc", [2, 3, 64])
def test_iou_finalize(cuda, nc, big):
    """Below 2^24 per row the float32 sums of the reference are exact, so kernel and reference
    agree up to the order of the final mean.  Above it the kernel keeps the exact int64 sums and
    rounds them once, while the reference's float32 hist.sum() rounds every partial sum: the
    kernel equals the float32 formula over the exact sums bit for bit, and the reference is within
    its own rounding, (3 nc + 4) U, of it."""
    g = _gen("iou_fin", nc, big)
    hi = 2 ** 40 if big else 2 ** 24 // (nc * nc)
    counts = torch.randint(0, hi, (nc, nc), generator=g)
    counts[nc - 1, :] = 0
    counts[:, nc - 1] = 0                                 # an empty class: IoU 0
    if big:
        counts[0, 0] = 2 ** 24
        counts[0, 1:nc - 1] = 1                           # float32 partial sums drop these
    counts = counts.reshape(-1)
    outs = []
    for _ in range(2):
        out = torch.full((1,), float("nan"), device=cuda)
        ops.iou_finalize(counts.to(cuda), nc, out)
        outs.append(out)
    torch.cuda.synchronize()
    same_bits(outs[0], outs[1], "iou_finalize reproducible")
    got = float(outs[0])
    assert got == iou_mirror(counts, nc), (got, iou_mirror(counts, nc))
    r = ref.iou_from_counts(counts.reshape(nc, nc))
    assert abs(got - r) <= (1e-7 if not big else (3 * nc + 4) * U), (got, r)


# ----------------------------------------------------------------------------- rowloss
ROW_CASES = [(1, 1), (3, 1), (65535, 1), (1, 255), (65535, 255), (3, 2048), (3, 2049),
             (1, 64 * 2048), (3, 64 * 2048), (3, 64 * 2048 + 1), (1, 10 ** 6), (3, 10 ** 6)]


@gpu
@pytest.mark.parametrize("case", ROW_CASES, ids=lambda c: f"B{c[0]}xD{c[1]}")
@pytest.mark.parametrize("kind", [0, 1], ids=["mse", "bce"])
def test_rowloss(cuda, kind, case):
    B, D = case
    gx = min(max(cdiv(D, 2048), 1), 64)
    n_t = cdiv(D, gx * 256)
    g = _gen("rowloss", kind, case)
    t = torch.rand((B, D), generator=g).double()          # non-binary targets
    if kind == 0:
        x = (torch.randn((B, D), generator=g) * 2).float().double()
    else:
        x = (torch.randn((B, D), generator=g) * 4).float().double()
        x.view(-1)[::5] = 80.0
        x.view(-1)[2::7] = -80.0
    t = t.float().double()
    xd, td = x.float().to(cuda), t.float().to(cuda)
    out0 = torch.linspace(-3, 5, B, dtype=torch.float64)
    gvec = (0.5 + 1.5 * torch.rand(B, generator=g)).float()
    runs = []
    for gv in (None, gvec.to(cuda), None):
        out = out0.clone().to(cuda)
        dx = torch.full((B, D), float("nan"), device=cuda)
        ops.rowloss(td, xd, kind, out, dx, gv)
        runs.append((out, dx))
    torch.cuda.synchronize()
    what = f"rowloss kind={kind} B={B} D={D}"
    same_bits(runs[0][1], runs[2][1], what + " dxhat reproducible")
    if gx == 1:
        same_bits(runs[0][0], runs[2][0], what + " out reproducible")
    xc, tc = x.to(cuda), t.to(cuda)                      # float64 references on the device
    if kind == 0:
        dd = xc - tc
        per = 0.5 * dd * dd
        e_term = 2 * U * per
        dref = dd
        e_d = 2 * U * dd.abs()
    else:
        per = F.binary_cross_entropy_with_logits(xc, tc, reduction="none")
        e = torch.exp(-xc.abs())
        lg = torch.log1p(e)
        xt = (xc * tc).abs()
        e_term = 2 * U * (xt + (xc.clamp_min(0) - xc * tc).abs() + per + lg) + 4 * U * e
        s = torch.sigmoid(xc)
        e2 = torch.exp(-xc)
        rel_s = torch.where(torch.isinf(e2), 0.0, 4 * U * e2 / (1 + e2)) + 2 * U
        dref = s - tc
        e_d = s * rel_s + 2 * U * dref.abs() + 1e-44
    tot = per.sum(1).cpu()
    mag = per.abs().sum(1).cpu()
    bound = e_term.sum(1).cpu() + (n_t + 12) * U * mag + (gx + 2) * D53 * (out0.abs() + mag)
    worst = 0.0
    for (out, dx), gv in zip(runs[:2], (None, gvec)):
        worst = max(worst, bound_check(out.cpu(), out0 + tot, bound, what + " out"))
        gg = torch.ones(B, dtype=torch.float64) if gv is None else gv.double()
        gg = gg.to(cuda)[:, None]
        worst = max(worst, bound_check(dx, dref * gg, e_d * gg + U * (dref * gg).abs(),
                                       what + f" dxhat gvec={gv is not None}"))
    MEASURED.setdefault(f"rowloss kind {kind}", []).append(worst)


# ----------------------------------------------------------------------------- refusals
@gpu
def test_refusals(cuda):
    """Arguments outside the kernels' limits raise NativeError before any launch: the NaN-filled
    outputs are untouched."""
    dev = cuda
    err = _C.NativeError

    def nan(*s, dtype=torch.float32):
        return torch.full(s, float("nan"), dtype=dtype, device=dev)

    lab = torch.zeros((1, 2, 4), dtype=torch.int64, device=dev)
    for shape, labels, K, pat in (((1, 2, 4, 17), lab, 17 * 4, "17 classes"),
                                  ((1, 2, 4, 3), lab.float(), 12, "int64"),
                                  ((1, 1, 65537, 16), torch.zeros((1, 1, 65537), dtype=torch.int64,
                                                                  device=dev), 16 * 65537,
                                   "workspace")):
        cells = nan(2 * K, dtype=torch.float64)
        with pytest.raises(err, match=pat):
            ops.dice_sums(torch.zeros(shape, device=dev), labels, cells)
        torch.cuda.synchronize()
        nan_intact(cells, "dice_sums cells")
    d = nan(1, 2, 4, 3)
    with pytest.raises(err, match="int64"):
        ops.dice_bwd(torch.zeros(1, 2, 4, 3, device=dev), lab.float(), torch.zeros(24, device=dev), d)
    counts = torch.full((65 * 65,), -7, dtype=torch.int64, device=dev)
    with pytest.raises(err, match="65 classes"):
        ops.iou_hist(torch.zeros(1, 2, 4, 65, device=dev), lab, 0.5, counts)
    out = nan(1)
    with pytest.raises(err, match="bad arguments"):
        ops.iou_finalize(torch.zeros(1, dtype=torch.int64, device=dev), 1, out)
    fl, ff = nan(1), nan(1)
    bce = torch.ones(1, dtype=torch.float64, device=dev)
    for count, gamma in ((1.0, -0.5), (0.0, 2.0), (-1.0, 2.0)):
        with pytest.raises(err, match="focal_finalize"):
            ops.focal_finalize(bce, count, 0.5, gamma, fl, ff)
    rl = nan(65536, dtype=torch.float64)
    with pytest.raises(err, match="batch too large"):
        ops.rowloss(torch.zeros(65536, 1, device=dev), torch.zeros(65536, 1, device=dev), 0, rl)
    torch.cuda.synchronize()
    nan_intact(d, "dice_bwd")
    assert bool((counts == -7).all())
    for t in (out, fl, ff):
        nan_intact(t, "finalise")
    nan_intact(rl, "rowloss")


MEASURED = {}


@gpu
def test_zz_report_measured(cuda):
    """Prints the largest |err| / bound per kernel of the cases above (run with -s)."""
    for k, v in sorted(MEASURED.items()):
        print(f"MEASURED {k}: {max(v):.3f} over {len(v)} cases")
