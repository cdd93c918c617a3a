"""
Generates tests/golden/conv_tc_plans.json, which pins the tile plan conv_tc picks.  One row per
case: the `conv_tc plan:` line that ATOMAI_B200_PLAN_LOG prints and the atomai_b200_conv_info
result (rc, grid, block, smem), for

  grid/...     the tests/test_conv_plan.py shape grid, tf32 and tf32x3, hw in {8, 64, 512}
  knobs/...    every knob set of test_conv_plan.py on the default Unet's layers, hw in {32, 512}
  matrix/...   every entry of tests/test_conv_exact_gpu.py::PLAN_MATRIX under its environment
  dgrad/...    every DGRAD_PLAN_ENVS entry on the data-gradient convolution of the layer
               test_dgrad_plan_variants uses, tf32 and tf32x3

The file keeps, per group of rows (one grid shape, one knob set, one matrix entry, one dgrad
environment), the row count and SHA-256 prefixes of the rows without and with `grid`.
tests/test_conv_plan_table.py requires the library to reproduce every group exactly and prints
the current rows of a group that differs.  The plan search is host code, so this runs without a
GPU (descriptors carry fake, aligned device pointers that are never dereferenced); `grid` is
min(tiles, SMs) with the 132 SMs of an H100 SXM, which is also the library's fallback when no
device is present.

    python tests/golden/make_conv_tc_plans.py
"""
import ctypes as C
import hashlib
import itertools
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
sys.path.insert(0, TESTS)
sys.path.insert(0, os.path.dirname(TESTS))

from atomai_b200 import _C, ops  # noqa: E402

OUT = os.path.join(HERE, "conv_tc_plans.json")
MATHS = {ops.MATH_TF32: "tf32", ops.MATH_TF32X3: "tf32x3"}


def env_key(env):
    return ",".join(f"{k[len('ATOMAI_B200_'):]}={v}" for k, v in sorted(env.items())) or "default"


def cases():
    """(group, id, environment, descriptor) of every recorded plan."""
    import test_conv_plan as tp
    from test_conv_exact_gpu import DGRAD_PLAN_ENVS, PLAN_MATRIX, L
    out = []
    for math, name in MATHS.items():
        for cins, cout in tp.SHAPES:
            group = f"grid/{name}/{'+'.join(map(str, cins))}->{cout}"
            for ks, dil, pool, hw in itertools.product((1, 3), (1, 2, 4), (False, True), (8, 64, 512)):
                if ks == 1 and dil > 1:
                    continue
                out.append((group, f"{group} k{ks} d{dil} pool{int(pool)} {hw}", {},
                            tp.make_desc(cins, hw, cout, ks, dil, pool, math)))
    for env in tp.KNOB_ENVS:
        group = f"knobs/{env_key(env)}"
        for (cins, cout, ks, pool), hw in itertools.product(tp.UNET, (32, 512)):
            out.append((group, f"{group}/{'+'.join(map(str, cins))}->{cout} k{ks} pool{int(pool)} {hw}", env,
                        tp.make_desc(cins, hw, cout, ks, 1, pool, ops.MATH_TF32X3)))
    for tag, env, layer, math, _ in PLAN_MATRIX:
        out.append((f"matrix/{tag}", f"matrix/{tag}", env, tp.layer_desc(layer, math)))
    dgrad = L([32], 32, 16, 24)     # dy of test_dgrad_plan_variants' [16, 16] -> 32 layer
    for env in DGRAD_PLAN_ENVS:
        for math, name in MATHS.items():
            group = f"dgrad/{env_key(env)}"
            out.append((group, f"{group}/{name}", env, tp.layer_desc(dgrad, math)))
    return out


def plan(env, d):
    """(plan line, rc, grid, block, smem) of descriptor `d` under the plan knobs `env` (and no
    other ATOMAI_B200_* variable)."""
    saved_env = {k: v for k, v in os.environ.items() if k.startswith("ATOMAI_B200_")}
    for k in saved_env:
        del os.environ[k]
    os.environ.update(env)
    os.environ["ATOMAI_B200_PLAN_LOG"] = "1"
    g, b, s = C.c_int(), C.c_int(), C.c_int()
    saved_fd = os.dup(2)
    try:
        with tempfile.TemporaryFile() as f:
            os.dup2(f.fileno(), 2)
            try:
                rc = _C.lib().atomai_b200_conv_info(C.byref(d), C.byref(g), C.byref(b), C.byref(s))
            finally:
                os.dup2(saved_fd, 2)
            f.seek(0)
            text = f.read().decode(errors="replace")
    finally:
        os.close(saved_fd)
        for k in [k for k in os.environ if k.startswith("ATOMAI_B200_")]:
            del os.environ[k]
        os.environ.update(saved_env)
    lines = [ln for ln in text.splitlines() if ln.startswith("conv_tc plan:")]
    return (lines[-1] if lines else "", rc, g.value, b.value, s.value)


def rows():
    """{group: [(row without grid, grid), ...]} of every case, in case order."""
    out = {}
    for group, tag, env, d in cases():
        line, rc, grid, block, smem = plan(env, d)
        out.setdefault(group, []).append((f"{tag} | {line} | rc={rc} block={block} smem={smem}", grid))
    return out


def _sha(texts):
    return hashlib.sha256("\n".join(texts).encode()).hexdigest()[:16]


def digest(group_rows):
    """[row count, hash of the rows without grid, hash of the rows with grid]"""
    return [len(group_rows), _sha(r for r, _ in group_rows), _sha(f"{r} grid={g}" for r, g in group_rows)]


if __name__ == "__main__":
    t = {group: digest(r) for group, r in rows().items()}
    with open(OUT, "w") as f:      # one group per line
        f.write("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v)}" for k, v in sorted(t.items())) + "\n}\n")
    print(f"{OUT}: {len(t)} groups, {sum(v[0] for v in t.values())} plans")
