"""Raw-kernel bring-up check on the GPU (dev tool, not a test): every C-ABI kernel against plain
torch fp32 ops on the GPU.  Each group runs in its own subprocess so that a trapped kernel cannot
poison the others.  Usage: python tools/gpu_check1.py [group ...]; prints one JSON line per group
(and writes them all to $GPU_CHECK1_JSON when that is set)."""
import json
import os
import subprocess
import sys
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GROUPS = ["selftest_tma", "simt", "tc_basic", "tc_fused", "tc_dgrad", "dgrad_diag", "wgrad_simt", "wgrad_tc",
          "elementwise", "vae", "bigshape"]


def rel(a, b):
    import torch
    return float((a - b).abs().max() / (b.abs().max() + 1e-20))


def run_group(name):
    import torch
    import torch.nn.functional as F
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from atomai_b200 import ops
    from atomai_b200.ops import Source
    dev = "cuda"
    g = torch.Generator(device="cpu").manual_seed(0)
    res = {}

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g) * scale).to(dev)

    def nhwc(t):  # NCHW -> NHWC contiguous
        return t.permute(0, 2, 3, 1).contiguous()

    def nchw(t):
        return t.permute(0, 3, 1, 2)

    def conv_case(tag, math, N, H, W, cins, Cout, ks=3, dil=1, affine=False, pool=False,
                  lrelu=0.01, stats=True, nchw_out=False):
        srcs, refs = [], []
        for ci in cins:
            hh, ww = (2 * H, 2 * W) if pool else (H, W)
            x = rnd(N, ci, hh, ww)
            sc = sh = None
            xr = x
            if affine:
                sc = (torch.rand(ci, generator=g) + 0.5).to(dev) * (torch.randint(0, 2, (ci,), generator=g).to(dev) * 2 - 1)
                sh = rnd(ci, scale=0.3)
                xr = x * sc.view(1, -1, 1, 1) + sh.view(1, -1, 1, 1)
            if pool:
                xr = F.max_pool2d(xr, 2, 2)
            srcs.append(Source(nhwc(x), sc, sh, pool))
            refs.append(xr)
        xin = torch.cat(refs, 1)
        cin = xin.shape[1]
        w = rnd(Cout, cin, ks, ks, scale=(1.0 / (cin * ks * ks)) ** 0.5)
        b = rnd(Cout, scale=0.1)
        ref = F.leaky_relu(F.conv2d(xin, w, b, padding=dil * (ks // 2), dilation=dil), lrelu)
        d = ops.conv_desc(srcs, N, H, W, Cout, (ks, ks), dil, lrelu, math, nchw_out)
        wp = ops.prep_weights(w, ops.WMODE_FWD, math)
        if nchw_out:
            out = torch.empty(N, Cout, H, W, device=dev)
        else:
            out = torch.empty(N, H, W, Cout, device=dev)
        st = torch.zeros(2 * Cout, device=dev, dtype=torch.float64) if stats else None
        ops.conv_fwd(d, wp, b, out, st)
        torch.cuda.synchronize()
        got = out if nchw_out else nchw(out)
        r = {"rel": rel(got, ref)}
        if stats:
            s1 = ref.double().sum((0, 2, 3))
            s2 = (ref.double() ** 2).sum((0, 2, 3))
            r["stats_rel"] = max(rel(st[:Cout], s1), rel(st[Cout:], s2))
        res[tag] = r
        return r

    def wgrad_case(tag, math, N, H, W, cins, Cout, ks=3, dil=1, affine=False, pool=False):
        srcs, refs = [], []
        for ci in cins:
            hh, ww = (2 * H, 2 * W) if pool else (H, W)
            x = rnd(N, ci, hh, ww)
            sc = sh = None
            xr = x
            if affine:
                sc = (torch.rand(ci, generator=g) + 0.5).to(dev)
                sh = rnd(ci, scale=0.3)
                xr = x * sc.view(1, -1, 1, 1) + sh.view(1, -1, 1, 1)
            if pool:
                xr = F.max_pool2d(xr, 2, 2)
            srcs.append(Source(nhwc(x), sc, sh, pool))
            refs.append(xr)
        xin = torch.cat(refs, 1)
        cin = xin.shape[1]
        dy = rnd(N, Cout, H, W)
        w = torch.zeros(Cout, cin, ks, ks, device=dev, requires_grad=True)
        F.conv2d(xin, w, None, padding=dil * (ks // 2), dilation=dil).backward(dy)
        d = ops.conv_desc(srcs, N, H, W, Cout, (ks, ks), dil, 1.0, math)
        dw = torch.zeros(Cout, cin, ks, ks, device=dev)
        ops.conv_wgrad(d, nhwc(dy), dw)
        torch.cuda.synchronize()
        res[tag] = {"rel": rel(dw, w.grad)}

    if name == "selftest_tma":
        # TMA box load of an NHWC halo tile: zero fill outside the image, swizzle = f(absolute address)
        x = rnd(2, 24, 20, 32)
        TWp, THp = 10, 6
        for mode, chunk, mask in [(0, 16, 0), (3, 16, 7)]:
            for off in (0, 128, 384):
                for (w0, h0) in [(3, 4), (-1, -1), (15, 20)]:
                    out = torch.full((THp * TWp * 32,), float("nan"), device=dev)
                    ops.selftest_tma(x, 0, w0, h0, 1, TWp, THp, mode, off, out)
                    torch.cuda.synchronize()
                    exp = torch.zeros(THp, TWp, 32, device=dev)
                    for hh in range(THp):
                        for ww in range(TWp):
                            gh, gw = h0 + hh, w0 + ww
                            if 0 <= gh < 24 and 0 <= gw < 20:
                                exp[hh, ww] = x[1, gh, gw]
                    img = torch.zeros(THp * TWp * 32, device=dev)
                    byte = torch.arange(THp * TWp * 32, device=dev) * 4
                    absb = byte + off
                    sw = absb ^ (((absb >> 7) & mask) * chunk) if mask else absb
                    img[((sw - off) // 4).long()] = exp.reshape(-1)
                    res[f"tma_m{mode}_off{off}_{w0}_{h0}"] = {"rel": float((out - img).abs().max())}
    elif name == "simt":
        M = ops.MATH_FP32
        conv_case("c1_1to16", M, 2, 40, 48, [1], 16)
        conv_case("c1_odd_w_affine", M, 3, 37, 29, [1], 16, affine=True)
        conv_case("c1_dil2", M, 2, 24, 30, [1], 16, dil=2)
        conv_case("c1_big", M, 4, 256, 256, [1], 16)
        conv_case("px_16to3", M, 2, 40, 48, [16], 3, ks=1, lrelu=1.0, stats=False)
        conv_case("c1_1to64_affine", M, 2, 40, 48, [1], 64, affine=True)      # ImSpec / VAE first layers
        conv_case("c1_1to128", M, 2, 33, 29, [1], 128)
        conv_case("pw_128to1", M, 2, 40, 48, [128], 1, ks=1, lrelu=1.0, stats=False)   # rDecoder output layer
        conv_case("pw_1to128", M, 2, 40, 48, [1], 128, ks=1, lrelu=1.0, stats=False)   # ... and its dgrad
        conv_case("pw_1to64_stats", M, 2, 24, 30, [1], 64, ks=1)
        conv_case("mid_24to20_dil2", M, 2, 33, 29, [24], 20, dil=2)
        conv_case("cat_affine_pool", M, 2, 16, 24, [8, 12], 16, affine=True, pool=True)
        conv_case("nchw_out", M, 2, 16, 24, [8], 16, nchw_out=True, stats=False)
        conv_case("1d_like", M, 3, 1, 128, [64], 64, dil=3)
    elif name == "tc_basic":
        M = ops.MATH_TF32
        conv_case("32to32_16x8", M, 1, 16, 8, [32], 32)
        conv_case("32to16_64x64", M, 2, 64, 64, [32], 16)
        conv_case("16to32", M, 2, 32, 32, [16], 32)
        conv_case("8to16", M, 2, 32, 32, [8], 16)
        conv_case("64to64", M, 2, 32, 32, [64], 64)
        conv_case("128to128", M, 2, 32, 24, [128], 128)
        conv_case("128to256", M, 1, 16, 16, [128], 256)
        conv_case("1x1_128to64", M, 2, 32, 32, [128], 64, ks=1, lrelu=1.0)
        conv_case("ragged_37x29", M, 3, 37, 29, [32], 32)
        conv_case("big_32to16", M, 8, 256, 256, [32], 16, affine=True)
        conv_case("big_16to32", M, 8, 256, 256, [16], 32, affine=True)
        conv_case("big_64to64", M, 8, 128, 128, [64], 64, affine=True)
        conv_case("big_128to128", M, 8, 64, 64, [128], 128, affine=True)
        conv_case("big_cat", M, 8, 128, 128, [64, 64], 64, affine=True)
    elif name == "tc_fused":
        M = ops.MATH_TF32
        conv_case("affine", M, 2, 32, 32, [32], 32, affine=True)
        conv_case("pool_affine", M, 2, 32, 32, [16], 32, affine=True, pool=True)
        conv_case("cat_16_16", M, 2, 32, 32, [16, 16], 16, affine=True)
        conv_case("cat_64_64", M, 2, 32, 32, [64, 64], 64)
        conv_case("dil2", M, 2, 32, 32, [64], 128, dil=2)
        conv_case("dil4", M, 2, 32, 32, [64], 128, dil=4)
        conv_case("dil6", M, 1, 32, 32, [128], 128, dil=6)
        conv_case("nchw_out", M, 2, 32, 32, [32], 32, nchw_out=True, stats=False)
        # one operand stage per pipeline (n_a = 2, streamed weights, several k-chunks): a plan the
        # shared-memory budget forces on wide layers; the consumer must hand each stage back
        # before it waits for the next chunk in the same stage
        os.environ["ATOMAI_B200_SMEM_KB"], os.environ["ATOMAI_B200_NA4"] = "64", "0"
        try:
            for m_, tag in ((M, "one_stage_tf32"), (ops.MATH_TF32X3, "one_stage_tf32x3")):
                conv_case(tag, m_, 2, 32, 32, [64], 64, affine=True)
                conv_case(tag + "_pool", m_, 2, 32, 32, [64], 64, pool=True)
        finally:
            del os.environ["ATOMAI_B200_SMEM_KB"], os.environ["ATOMAI_B200_NA4"]
    elif name == "tc_dgrad":
        for math, tag in [(ops.MATH_FP32, "simt"), (ops.MATH_TF32, "tc")]:
            for (ci, co, dil) in [(32, 64, 1), (16, 32, 1), (64, 128, 2)]:
                N, H, W = 2, 32, 32
                x = rnd(N, ci, H, W).requires_grad_(True)
                w = rnd(co, ci, 3, 3, scale=0.1)
                y = F.conv2d(x, w, None, padding=dil, dilation=dil)
                dy = rnd(N, co, H, W)
                y.backward(dy)
                dyn = nhwc(dy)   # keep alive: the descriptor only stores its pointer
                d = ops.conv_desc([Source(dyn)], N, H, W, ci, (3, 3), dil, 1.0, math)
                wp = ops.prep_weights(w, ops.WMODE_DGRAD, math)
                out = torch.empty(N, H, W, ci, device=dev)
                ops.conv_fwd(d, wp, None, out, None)
                torch.cuda.synchronize()
                res[f"{tag}_{ci}_{co}_d{dil}"] = {"rel": rel(nchw(out), x.grad)}
    elif name == "dgrad_diag":
        # first-launch / shape sensitivity of the tensor-core path: each case twice, TC vs SIMT
        for rep in range(2):
            for (ci, co, dil) in [(32, 64, 1), (64, 32, 1), (32, 64, 1), (16, 32, 1)]:
                N, H, W = 2, 32, 32
                w = rnd(co, ci, 3, 3, scale=0.1)
                dy = nhwc(rnd(N, co, H, W))
                outs = {}
                for math, tag in [(ops.MATH_TF32, "tc"), (ops.MATH_FP32, "simt")]:
                    d = ops.conv_desc([Source(dy)], N, H, W, ci, (3, 3), dil, 1.0, math)
                    wp = ops.prep_weights(w, ops.WMODE_DGRAD, math)
                    out = torch.full((N, H, W, ci), float("nan"), device=dev)
                    ops.conv_fwd(d, wp, None, out, None)
                    torch.cuda.synchronize()
                    outs[tag] = out
                diff = (outs["tc"] - outs["simt"]).abs()
                bad = diff > 1e-2 * outs["simt"].abs().max()
                info = {"rel": rel(outs["tc"], outs["simt"]), "nbad": int(bad.sum()),
                        "nan": int(torch.isnan(outs["tc"]).sum())}
                if bad.any():
                    idx = bad.nonzero()
                    info["bad_n"] = sorted(set(idx[:, 0].tolist()))
                    info["bad_h"] = [int(idx[:, 1].min()), int(idx[:, 1].max())]
                    info["bad_w"] = [int(idx[:, 2].min()), int(idx[:, 2].max())]
                    info["bad_c"] = [int(idx[:, 3].min()), int(idx[:, 3].max())]
                res[f"rep{rep}_{ci}_{co}"] = info
        # same through the forward weight mode (K = 64 -> N = 32)
        conv_case("fwd_64to32", ops.MATH_TF32, 2, 32, 32, [64], 32)
        conv_case("fwd_64to32_again", ops.MATH_TF32, 2, 32, 32, [64], 32)
    elif name == "wgrad_simt":
        M = ops.MATH_FP32
        wgrad_case("1to16", M, 2, 40, 48, [1], 16)
        wgrad_case("16to3_1x1", M, 2, 40, 48, [16], 3, ks=1)
        wgrad_case("cat_pool_affine", M, 2, 16, 24, [8, 12], 16, affine=True, pool=True)
        wgrad_case("70to130_dil2", M, 1, 17, 19, [70], 130, dil=2)
        wgrad_case("1to16_affine", M, 3, 37, 29, [1], 16, affine=True)
        wgrad_case("1to16_dil2", M, 2, 24, 30, [1], 16, dil=2)
        wgrad_case("1to16_big", M, 4, 256, 256, [1], 16)
        wgrad_case("16to3_1x1_affine", M, 3, 37, 29, [16], 3, ks=1, affine=True)
        wgrad_case("2to16_1x1", M, 2, 20, 24, [2], 16, ks=1)
        wgrad_case("8to3_3x3", M, 2, 20, 24, [8], 3)
    elif name == "wgrad_tc":
        M = ops.MATH_TF32
        wgrad_case("32to32_16x8", M, 1, 16, 8, [32], 32)
        wgrad_case("32to16", M, 2, 64, 64, [32], 16)
        wgrad_case("16to32", M, 2, 32, 32, [16], 32)
        wgrad_case("64to64", M, 2, 32, 32, [64], 64)
        wgrad_case("128to128", M, 2, 32, 24, [128], 128)
        wgrad_case("128to256", M, 1, 16, 16, [128], 256)
        wgrad_case("1x1_128to64", M, 2, 32, 32, [128], 64, ks=1)
        wgrad_case("cat_affine_pool", M, 2, 32, 32, [16, 16], 32, affine=True, pool=True)
        wgrad_case("ragged", M, 3, 37, 29, [32], 48)
        wgrad_case("dil2", M, 2, 32, 32, [64], 128, dil=2)
        wgrad_case("1x1_40to24", M, 2, 32, 32, [40], 24, ks=1)
        wgrad_case("cat_48_16_affine", M, 2, 40, 24, [48, 16], 20, affine=True)
    elif name == "elementwise":
        N, H, W, Cc = 3, 20, 24, 32
        a = rnd(N, Cc, H, W)
        # BN train forward + backward vs torch
        bn = torch.nn.BatchNorm2d(Cc).to(dev)
        bn.weight.data = rnd(Cc).abs() + 0.5
        bn.bias.data = rnd(Cc, scale=0.2)
        a_r = a.clone().requires_grad_(True)
        act = F.leaky_relu(a_r, 0.01)
        y = bn(act)
        dy = rnd(N, Cc, H, W)
        y.backward(dy)
        a_n = nhwc(act.detach())
        stats = torch.stack([a_n.double().sum((0, 1, 2)), (a_n.double() ** 2).sum((0, 1, 2))]).reshape(-1).contiguous()
        scale = torch.empty(Cc, device=dev); shift = torch.empty(Cc, device=dev)
        mean = torch.empty(Cc, device=dev); invstd = torch.empty(Cc, device=dev)
        rm = torch.zeros(Cc, device=dev); rv = torch.ones(Cc, device=dev)
        ops.bn_finalize(stats, N * H * W, bn.weight.data, bn.bias.data, rm, rv, 0.1, 1e-5, True, scale, shift, mean, invstd)
        yy = torch.empty(N, H, W, Cc, device=dev)
        ops.affine(a_n, scale, shift, yy)
        res["bn_fwd"] = {"rel": rel(nchw(yy), y.detach())}
        res["bn_running"] = {"rel": max(rel(rm, bn.running_mean), rel(rv, bn.running_var))}
        sums = torch.zeros(2 * Cc, device=dev, dtype=torch.float64)
        dyn = nhwc(dy)
        ops.bn_bwd_reduce(dyn, a_n, mean, invstd, sums)
        dpre = torch.empty(N, H, W, Cc, device=dev)
        dbias = torch.zeros(Cc, device=dev, dtype=torch.float64)
        ops.bn_act_bwd(dyn, a_n, mean, invstd, scale, sums, N * H * W, None, ops.ACT_LRELU, 0.01, dpre, dbias)
        res["bn_bwd_dx"] = {"rel": rel(nchw(dpre), a_r.grad)}
        res["bn_bwd_dgamma"] = {"rel": rel(sums[Cc:].float(), bn.weight.grad)}
        res["bn_bwd_dbeta"] = {"rel": rel(sums[:Cc].float(), bn.bias.grad)}
        res["dbias"] = {"rel": rel(dbias.float(), a_r.grad.sum((0, 2, 3)))}
        # pool fwd / bwd
        sc = (torch.rand(Cc, generator=g) + 0.5).to(dev) * -1.0
        sh = rnd(Cc)
        xr = (a * sc.view(1, -1, 1, 1) + sh.view(1, -1, 1, 1)).requires_grad_(True)
        pr = F.max_pool2d(xr, 2, 2)
        dp = rnd(N, Cc, H // 2, W // 2)
        pr.backward(dp)
        po = torch.empty(N, H // 2, W // 2, Cc, device=dev)
        ops.pool_fwd(nhwc(a), sc, sh, po)
        res["pool_fwd"] = {"rel": rel(nchw(po), pr.detach())}
        df = torch.full((N, H, W, Cc), 7.0, device=dev)
        ops.pool_bwd(nhwc(dp), nhwc(a), sc, sh, df, False)
        res["pool_bwd"] = {"rel": rel(nchw(df), xr.grad)}
        # upsample fwd/bwd
        for bil in (True, False):
            xs = rnd(N, Cc, 9, 7).requires_grad_(True)
            up = F.interpolate(xs, scale_factor=2, mode="bilinear" if bil else "nearest")
            du = rnd(N, Cc, 18, 14)
            up.backward(du)
            uo = torch.empty(N, 18, 14, Cc, device=dev)
            ops.upsample_fwd(nhwc(xs.detach()), uo, bil)
            dxo = torch.empty(N, 9, 7, Cc, device=dev)
            ops.upsample_bwd(nhwc(du), dxo, bil)
            res[f"up_fwd_{bil}"] = {"rel": rel(nchw(uo), up.detach())}
            res[f"up_bwd_{bil}"] = {"rel": rel(nchw(dxo), xs.grad)}
        # CE
        lg = rnd(N, 3, H, W).requires_grad_(True)
        lab = torch.randint(0, 3, (N, H, W), generator=g).to(dev)
        loss = F.cross_entropy(lg, lab)
        loss.backward()
        ls = torch.zeros(1, device=dev, dtype=torch.float64)
        dl = torch.empty(N, H, W, 3, device=dev)
        ops.ce_fwd_bwd(nhwc(lg.detach()), lab, ls, dl, 1.0 / (N * H * W))
        res["ce_loss"] = {"rel": abs(float(ls) / (N * H * W) - float(loss)) / float(loss)}
        res["ce_grad"] = {"rel": rel(nchw(dl), lg.grad)}
        # adam
        ps = [rnd(1000), rnd(37), rnd(16, 3, 3, 3)]
        gs = [rnd(*p.shape) for p in ps]
        ref_p = [p.clone().requires_grad_(True) for p in ps]
        opt = torch.optim.Adam(ref_p, lr=1e-3)
        ms = [torch.zeros_like(p) for p in ps]; vs = [torch.zeros_like(p) for p in ps]
        tab = torch.tensor([[p.data_ptr(), gg.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel()] for p, gg, m, v in zip(ps, gs, ms, vs)], dtype=torch.int64, device=dev)
        for step in (1, 2, 3):
            for p, gg in zip(ref_p, gs):
                p.grad = gg.clone()
            opt.step()
            ops.adam_multi(tab, len(ps), max(p.numel() for p in ps), 1e-3, 0.9, 0.999, 1e-8, 0.0, step)
        res["adam"] = {"rel": max(rel(p, r.detach()) for p, r in zip(ps, ref_p))}
    elif name == "vae":
        x = rnd(10, 4096); w = rnd(5, 4096, scale=0.02); b = rnd(5)
        y = torch.empty(10, 5, device=dev)
        ops.linear_fwd(x, w, b, y)
        res["linear_fwd"] = {"rel": rel(y, x @ w.t() + b)}
        dy = rnd(10, 5)
        dx = torch.empty_like(x); dw = torch.empty_like(w); db = torch.empty(5, device=dev)
        ops.linear_bwd(x, w, dy, dx, dw, db)
        res["linear_bwd"] = {"rel": max(rel(dx, dy @ w), rel(dw, dy.t() @ x), rel(db, dy.sum(0)))}
        x1 = rnd(300, 128); x2 = rnd(200, 128)
        ils = (torch.rand(128, generator=g) * 0.1 + 0.05).to(dev)
        Kmat = torch.empty(300, 200, device=dev)
        ops.gram(x1, x2, ils, 1.7, 0, Kmat)
        d2 = torch.cdist((x1 * ils).double(), (x2 * ils).double()) ** 2
        res["gram_rbf"] = {"rel": rel(Kmat, (1.7 * torch.exp(-0.5 * d2)).float())}
        ops.gram(x1, x2, ils, 1.0, 1, Kmat)
        r = d2.sqrt()
        mat = (1 + 5 ** 0.5 * r + 5.0 / 3 * d2) * torch.exp(-(5 ** 0.5) * r)
        res["gram_matern"] = {"rel": rel(Kmat, mat.float())}
    elif name == "bigshape":
        import time
        M = ops.MATH_TF32
        r = conv_case("c6_like_512", M, 4, 512, 512, [16, 16], 16, affine=True)
        r = conv_case("bn_like", M, 8, 64, 64, [128], 128)
        wgrad_case("wg_c5_like", M, 2, 256, 256, [32, 32], 32)
        # timing of one bottleneck conv, events on the current stream
        N, H, W, ci, co = 32, 64, 64, 128, 128
        x = nhwc(rnd(N, ci, H, W)); w = rnd(co, ci, 3, 3, scale=0.03); b = rnd(co)
        out = torch.empty(N, H, W, co, device=dev)
        for math, tag in [(ops.MATH_TF32, "tc"), (ops.MATH_FP32, "simt")]:
            d = ops.conv_desc([Source(x)], N, H, W, co, (3, 3), 1, 0.01, math)
            wp = ops.prep_weights(w, ops.WMODE_FWD, math)
            st = torch.zeros(2 * co, device=dev, dtype=torch.float64)
            for _ in range(3):
                ops.conv_fwd(d, wp, b, out, st)
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                ops.conv_fwd(d, wp, b, out, st)
            e1.record(); torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 10
            res[f"time_bn3_{tag}"] = {"ms": ms, "tflops": 2 * N * H * W * ci * co * 9 / ms / 1e9}
        xc = rnd(N, ci, H, W);
        torch.backends.cudnn.allow_tf32 = True
        for _ in range(3):
            F.conv2d(xc, w, b, padding=1)
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            F.conv2d(xc, w, b, padding=1)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        res["time_bn3_cudnn_tf32"] = {"ms": ms, "tflops": 2 * N * H * W * ci * co * 9 / ms / 1e9}
    return res


def main():
    if len(sys.argv) >= 3 and sys.argv[1] == "--child":
        name = sys.argv[2]
        try:
            out = {"ok": True, "res": run_group(name)}
        except Exception as e:  # noqa
            out = {"ok": False, "error": f"{type(e).__name__}: {e}", "tb": traceback.format_exc()[-1500:]}
        print("@@RESULT@@" + json.dumps(out))
        return
    groups = sys.argv[1:] or GROUPS
    allres = {}
    for gname in groups:
        try:
            pr = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", gname],
                                capture_output=True, text=True, timeout=300)
            line = [l for l in pr.stdout.splitlines() if l.startswith("@@RESULT@@")]
            if line:
                allres[gname] = json.loads(line[-1][len("@@RESULT@@"):])
            else:
                allres[gname] = {"ok": False, "error": "no result", "stdout": pr.stdout[-1500:], "stderr": pr.stderr[-1500:], "rc": pr.returncode}
            if pr.stdout and not line:
                pass
            extra = [l for l in pr.stdout.splitlines() if "atomai_b200:" in l]
            if extra:
                allres[gname]["device_msgs"] = extra[:5]
        except subprocess.TimeoutExpired:
            allres[gname] = {"ok": False, "error": "timeout"}
        print(gname, json.dumps(allres[gname])[:3000], flush=True)
        if os.environ.get("GPU_CHECK1_JSON"):
            with open(os.environ["GPU_CHECK1_JSON"], "w") as f:
                json.dump(allres, f, indent=1)


if __name__ == "__main__":
    main()
