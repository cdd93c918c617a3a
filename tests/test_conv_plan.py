"""Host-side tile-plan search of conv_tc (csrc/conv_tc.cu::conv_tc_plan) over a grid of layer
shapes: every tensor-core-eligible shape must get a plan that fits the opted-in shared memory,
in every math mode and under the plan knobs.  Runs without a GPU (the plan is host code; the
descriptor carries fake, aligned device pointers that are never dereferenced)."""
import ctypes as C
import itertools

import pytest

from atomai_b200 import _C, ops

OPT_IN = 226 * 1024     # cudaFuncAttributeMaxDynamicSharedMemorySize set by ab_conv_tc_fwd


def make_desc(cins, hw, cout, ks, dil, pool, math, affine=True):
    d = _C.Conv()
    d.N, d.H, d.W, d.Cout = 2, hw, hw, cout
    d.ks_h, d.ks_w, d.dil = ks, ks, dil
    d.nsrc = len(cins)
    for i, ci in enumerate(cins):
        e = d.src[i]
        e.ptr = 0x10000000 * (i + 1)
        e.scale = 0x1000 if affine else None
        e.shift = 0x2000 if affine else None
        e.C, e.ld, e.pool = ci, ci, (1 if (pool and i == 0) else 0)
    d.lrelu, d.math, d.out_nchw, d.act = 0.01, math, 0, ops.ACT_LRELU
    return d


def info(d):
    g, b, s = C.c_int(), C.c_int(), C.c_int()
    rc = _C.lib().atomai_b200_conv_info(C.byref(d), C.byref(g), C.byref(b), C.byref(s))
    return rc, g.value, b.value, s.value


SHAPES = [([c], co) for c in (8, 16, 24, 32, 64, 128, 256) for co in (16, 32, 64, 128, 256)] + \
         [([16, 16], 16), ([32, 32], 32), ([64, 64], 64), ([128, 128], 128), ([16, 48], 32)]


@pytest.mark.parametrize("math", [ops.MATH_TF32, ops.MATH_TF32X3])
def test_every_shape_gets_a_plan(math):
    n = 0
    for (cins, cout), ks, dil, pool in itertools.product(SHAPES, (1, 3), (1, 2, 4), (False, True)):
        if ks == 1 and dil > 1:
            continue
        for hw in (8, 64, 512):
            d = make_desc(cins, hw, cout, ks, dil, pool, math)
            rc, grid, block, smem = info(d)
            assert rc == 0, (cins, cout, ks, dil, pool, hw, _C.lib().atomai_b200_last_error())
            assert block == 512 and 1 <= grid <= 4096
            assert 0 < smem <= OPT_IN, (cins, cout, ks, dil, pool, hw, smem)
            n += 1
    assert n >= 900


KNOB_ENVS = [{"ATOMAI_B200_NA4": "0", "ATOMAI_B200_SMEM_KB": "212", "ATOMAI_B200_MIN_NR": "2"},
             {"ATOMAI_B200_RES_NA4": "1"}, {"ATOMAI_B200_RES_NA4": "0"},
             {"ATOMAI_B200_TMA": "0"}, {"ATOMAI_B200_TMA_KC8": "1"}]
# (source channels, Cout, kernel size, pooled source) of the default Unet's tensor-core layers
UNET = [([16], 32, 3, True), ([32], 32, 3, False), ([32], 64, 3, True), ([64], 64, 3, False),
        ([64], 128, 3, True), ([128], 128, 3, False), ([128], 64, 1, False), ([64, 64], 64, 3, False),
        ([64], 32, 1, False), ([32, 32], 32, 3, False), ([32], 16, 1, False), ([16, 16], 16, 3, False)]


@pytest.mark.parametrize("env", KNOB_ENVS)
def test_plan_knobs_keep_every_unet_layer_plannable(env, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    for cins, cout, ks, pool in UNET:
        for hw in (32, 512):
            rc, _, _, smem = info(make_desc(cins, hw, cout, ks, 1, pool, ops.MATH_TF32X3))
            assert rc == 0 and smem <= OPT_IN, (env, cins, cout, smem)


def layer_desc(layer, math):
    """Descriptor of a tests/test_conv_exact_gpu.py Layer on fake, aligned device pointers."""
    d = _C.Conv()
    d.N, d.H, d.W, d.Cout = layer.N, layer.H, layer.W, layer.cout
    d.ks_h, d.ks_w, d.dil = layer.ks[0], layer.ks[1], layer.dil
    d.nsrc = len(layer.srcs)
    for i, s in enumerate(layer.srcs):
        e = d.src[i]
        e.ptr = 0x10000000 * (i + 1)
        e.scale = e.shift = None
        e.C, e.ld, e.pool = s.C, s.C + s.pad, s.tr
    d.lrelu, d.math, d.out_nchw, d.act = 1.0, math, 0, ops.ACT_LRELU
    return d


def test_exact_suite_plan_matrix_covers_every_variant(monkeypatch, capfd):
    """Each forced entry of the exact GPU suite's plan matrix still gets the plan it names, and
    together they cover every conv_tc plan variant and consumer instantiation.  If the plan
    heuristics change, this fails here instead of silently moving GPU coverage.  The plan never
    gives a streamed layer fewer than two weight stages per pipeline (n_b >= 4), so the smallest
    weight ring it can produce, n_b = 4, stands in for the one-stage ring."""
    from test_conv_exact_gpu import PLAN_MATRIX, launch_widths, parse_plan
    monkeypatch.setenv("ATOMAI_B200_PLAN_LOG", "1")
    seen = []
    for tag, env, layer, math, want in PLAN_MATRIX:
        with monkeypatch.context() as mp:
            for k, v in env.items():
                mp.setenv(k, v)
            capfd.readouterr()
            rc, _, _, smem = info(layer_desc(layer, math))
            text = capfd.readouterr().err
        assert rc == 0, (tag, _C.lib().atomai_b200_last_error())
        assert 0 < smem <= OPT_IN, (tag, smem)
        got = parse_plan(text)
        assert got == want, f"{tag}: plan {got}, the matrix expects {want}"
        seen.append((got, layer))
    plans = [p for p, _ in seen]
    assert any(p["resident"] for p in plans)
    assert any(not p["resident"] and p["sub"] == 1 for p in plans)
    assert any(not p["resident"] and p["sub"] == 2 for p in plans)
    assert {p["KC"] for p in plans} == {8, 16, 32}
    assert {p["n_a"] for p in plans} == {2, 4}
    assert any(p["n_a"] == 2 and p["resident"] for p in plans)
    assert any(p["n_a"] == 2 and not p["resident"] for p in plans)
    assert any(p["n_b"] == 4 for p in plans)
    assert {p["tma"] for p in plans} == {0, 1}
    assert any(p["tma"] and p["KC"] == 8 for p in plans)
    consumers = {(nn, p["sub"]) for p, layer in seen for nn in launch_widths(layer.cout)}
    every = {(nn, 1) for nn in range(16, 129, 16)} | {(nn, 2) for nn in range(16, 65, 16)}
    assert consumers == every, f"missing consumer instantiations: {sorted(every - consumers)}"
    assert any(len(launch_widths(layer.cout)) > 1 for _, layer in seen)
    assert any(len(layer.srcs) == 2 and layer.srcs[0].C % p["KC"] for p, layer in seen), \
        "no concat whose split falls inside a k-chunk"
