"""Tile plans of the thin layers of the bench Unet (batch 32 x 512^2 input), without a GPU: the
plan search is host code and the descriptors carry fake, aligned device pointers.  3x3 layers of
at most 32 output channels with resident weights and two operand stages per pipeline take two
tiles per consumer pass (csrc/conv_tc.cu, ConvTcParams::pair); every other layer keeps one.  Also
checks that each consumer instantiation keeps its accumulators within 64 registers per thread."""
import ctypes as C
import os
import re

import pytest

from atomai_b200 import _C, ops

PLAN_RE = re.compile(r"conv_tc plan: .*\| resident=(\d+) sub=(\d+) KC=(\d+) n_a=(\d+) n_b=(\d+) "
                     r"tma=(\d+) n_r=(\d+) a_stage=(\d+) smem=(\d+)")
TILE_RE = re.compile(r"conv_tc tile: 8x(\d+) px, (\d+) tile\(s\) per consumer pass")
BUDGET = 224 * 1024
SRC = os.path.join(os.path.dirname(_C.__file__), "csrc", "conv_tc.cu")

# (layer, H, source channels, Cout, kernel size, pooled source) of the bench Unet's tensor-core
# layers; the data gradient of a 3x3 layer swaps Cin and Cout (tools/bench_layers.py)
LAYERS = [("c2.0", 256, [16], 32, 3, True), ("c2.1", 256, [32], 32, 3, False),
          ("c3.0", 128, [32], 64, 3, True), ("c3.1", 128, [64], 64, 3, False),
          ("bn.0", 64, [64], 128, 3, True), ("bn.1", 64, [128], 128, 3, False),
          ("u1", 64, [128], 64, 1, False), ("c4.0", 128, [64, 64], 64, 3, False),
          ("c4.1", 128, [64], 64, 3, False), ("u2", 128, [64], 32, 1, False),
          ("c5.0", 256, [32, 32], 32, 3, False), ("c5.1", 256, [32], 32, 3, False),
          ("u3", 256, [32], 16, 1, False), ("c6.0", 512, [16, 16], 16, 3, False)]

# tf32x3 plans: (resident, sub, KC, n_a, tma, n_r) and tiles per consumer pass
WANT = {
    "c2.0 fwd": ((1, 1, 16, 4, 0, 0), 2),
    "c2.1 fwd": ((1, 1, 16, 4, 1, 8), 2), "c2.1 dgrad": ((1, 1, 16, 4, 1, 8), 2),
    "c3.0 fwd": None, "c3.1 fwd": ((0, 2, 16, 4, 0, 0), 1), "c3.1 dgrad": ((0, 2, 16, 4, 0, 0), 1),
    "bn.0 fwd": None, "bn.1 fwd": ((0, 1, 16, 4, 0, 0), 1), "bn.1 dgrad": ((0, 1, 16, 4, 0, 0), 1),
    "u1 fwd": None, "c4.0 fwd": None, "c4.0 dgrad": None, "c4.1 fwd": None, "c4.1 dgrad": None,
    "u2 fwd": None,
    "c5.0 fwd": ((1, 1, 16, 4, 0, 0), 2), "c5.0 dgrad": ((1, 1, 16, 4, 0, 0), 1),
    "c5.1 fwd": ((1, 1, 16, 4, 1, 8), 2), "c5.1 dgrad": ((1, 1, 16, 4, 1, 8), 2),
    "u3 fwd": None,
    "c6.0 fwd": ((1, 1, 16, 4, 1, 8), 2), "c6.0 dgrad": ((1, 1, 16, 4, 1, 8), 2),
}


# the layers that take two tiles per consumer pass.  tf32 plans of the 32-channel layers use
# 32-channel k-chunks, 7 loader elements per thread, for which there is no paired loader.
PAIRED = {ops.MATH_TF32X3: {"c2.0 fwd", "c2.1 fwd", "c2.1 dgrad", "c5.0 fwd", "c5.1 fwd", "c5.1 dgrad",
                            "c6.0 fwd", "c6.0 dgrad"},
          ops.MATH_TF32: {"c2.0 fwd", "c6.0 fwd", "c6.0 dgrad"}}


def desc(cins, hw, cout, ks, pool, math):
    d = _C.Conv()
    d.N, d.H, d.W, d.Cout = 32, hw, hw, cout
    d.ks_h, d.ks_w, d.dil = ks, ks, 1
    d.nsrc = len(cins)
    for i, ci in enumerate(cins):
        e = d.src[i]
        e.ptr = 0x10000000 * (i + 1)
        e.scale, e.shift = 0x1000, 0x2000
        e.C, e.ld, e.pool = ci, ci, (1 if (pool and i == 0) else 0)
    d.lrelu, d.math, d.out_nchw, d.act = 0.01, math, 0, ops.ACT_LRELU
    return d


def plan(d, capfd):
    capfd.readouterr()
    g, b, s = C.c_int(), C.c_int(), C.c_int()
    rc = _C.lib().atomai_b200_conv_info(C.byref(d), C.byref(g), C.byref(b), C.byref(s))
    err = capfd.readouterr().err
    assert rc == 0, _C.lib().atomai_b200_last_error()
    m, t = PLAN_RE.search(err), TILE_RE.search(err)
    assert m and t, err
    f = tuple(int(v) for v in m.groups())
    return dict(resident=f[0], sub=f[1], KC=f[2], n_a=f[3], n_b=f[4], tma=f[5], n_r=f[6],
                smem=f[8], info_smem=s.value, tile_w=int(t.group(1)), pair=int(t.group(2)))


def bench_descs(math):
    for name, hw, cins, cout, ks, pool in LAYERS:
        yield f"{name} fwd", ks, cout, desc(cins, hw, cout, ks, pool, math)
        if ks == 3 and not pool:
            yield f"{name} dgrad", ks, sum(cins), desc([cout], hw, sum(cins), ks, False, math)


@pytest.mark.parametrize("math", [ops.MATH_TF32, ops.MATH_TF32X3], ids=["tf32", "tf32x3"])
def test_bench_layer_plans(math, monkeypatch, capfd):
    monkeypatch.setenv("ATOMAI_B200_PLAN_LOG", "1")
    for tag, _, _, d in bench_descs(math):
        p = plan(d, capfd)
        assert p["smem"] == p["info_smem"] <= BUDGET, (tag, p)
        assert p["tile_w"] == 8 * p["sub"], (tag, p)
        assert p["pair"] == (2 if tag in PAIRED[math] else 1), (tag, p)
        if math == ops.MATH_TF32X3 and WANT[tag] is not None:
            want, pair = WANT[tag]
            got = (p["resident"], p["sub"], p["KC"], p["n_a"], p["tma"], p["n_r"])
            assert (got, p["pair"]) == (want, pair), (tag, p)


def test_pairing_knob(monkeypatch, capfd):
    """ATOMAI_B200_PAIR=0 gives every layer one tile per pass and leaves the rest of the plan."""
    monkeypatch.setenv("ATOMAI_B200_PLAN_LOG", "1")
    paired = {tag: plan(d, capfd) for tag, _, _, d in bench_descs(ops.MATH_TF32X3)}
    monkeypatch.setenv("ATOMAI_B200_PAIR", "0")
    for tag, _, _, d in bench_descs(ops.MATH_TF32X3):
        p = plan(d, capfd)
        assert p["pair"] == 1, tag
        assert dict(p, pair=0) == dict(paired[tag], pair=0), tag
    assert sum(p["pair"] == 2 for p in paired.values()) == 8


def test_small_layers_stay_unpaired(monkeypatch, capfd):
    """Pairing needs more than two tiles per CTA (132 SMs without a device): a 3x3 thin layer of
    at most 2 * SMs 8x8 tiles keeps one tile per pass, one more tile pairs."""
    monkeypatch.setenv("ATOMAI_B200_PLAN_LOG", "1")
    sms = 132
    try:
        import torch
        if torch.cuda.is_available():
            sms = torch.cuda.get_device_properties(0).multi_processor_count
    except ImportError:
        pass
    for tiles, want in ((sms - 1, 1), (2 * sms, 1), (2 * sms + 1, 2)):
        d = desc([16], 8, 16, 3, False, ops.MATH_TF32X3)
        d.N, d.H, d.W = 1, 8, 8 * tiles
        assert plan(d, capfd)["pair"] == want, tiles


def test_consumer_accumulators_fit_64_registers():
    """Every consumer instantiation (N, sub-tiles, tiles per pass): N / 2 fp32 accumulators per
    m64 block and thread, sub-tiles x tiles per pass blocks, at most 64 registers."""
    with open(SRC) as f:
        src = f.read()
    cases = [tuple(map(int, c)) for c in re.findall(r"AB_CONS_CASE\((\d+), (\d+), (\d+)\)", src)]
    assert len(cases) >= 14
    assert {(n, s) for n, s, t in cases if t == 1} == \
        {(n, 1) for n in range(16, 129, 16)} | {(n, 2) for n in range(16, 65, 16)}
    assert {(n, s) for n, s, t in cases if t == 2} == {(16, 1), (32, 1)}
    for n, s, t in cases:
        assert s * t * n // 2 <= 64, (n, s, t)
