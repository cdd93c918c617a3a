"""
Generates tests/golden/imgen_ref.npz by running the UNMODIFIED reference's atomai.utils.imgen
(MakeAtom, create_atom_mask_pair, create_lattice_mask, create_multiclass_lattice_mask[_]) and
atomai.utils.img (extract_patches_, extract_patches, extract_patches_and_spectra, with sklearn's
extract_patches_2d) through oracle/ref_shim.py on the seeded cases of imgen_cases.py:

  atom/<i>/<g|mask|x|y>      MakeAtom(sc, r_mask, intensity, theta, offset=i % 3).gen_atom_mask()
  pair/<i>/<atom|mask>       create_atom_mask_pair(sc, r_mask, intensity)
  <case>/out/<k>             the k-th output (a list result is flattened into its items)
  <case>/kind                "array", "list" or "tuple"
  <case>/arg/<k>             the coordinate arrays after the call (the in-place class shift)
  <case>/error               the exception's first builtin base class, when the call raises

Run in the build container only:

    python tests/golden/make_golden_imgen.py
"""
import builtins
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import imgen_cases as ic  # noqa: E402


def error_name(e: BaseException) -> str:
    return next(t.__name__ for t in type(e).__mro__ if getattr(builtins, t.__name__, None) is t)


def coord_args(fn, args):
    """the coordinate arrays a case passes (their state after the call is recorded)"""
    if fn.startswith("create_multiclass_lattice_mask"):
        c = args[1]
        return [c[k] for k in sorted(c)] if isinstance(c, dict) else [c]
    return []


def record(out, name, fns):
    fn = ic.all_cases()[name][0]
    try:
        res, args = ic.call(fns, name)
    except Exception as e:  # noqa: BLE001 — the exception type is the golden
        out[f"{name}/error"] = np.array(error_name(e))
        return
    if isinstance(res, tuple):
        kind, items = "tuple", list(res)
    elif isinstance(res, list):
        kind, items = "list", res
    else:
        kind, items = "array", [res]
    out[f"{name}/kind"] = np.array(kind)
    for k, a in enumerate(items):
        out[f"{name}/out/{k}"] = np.asarray(a)
    for k, a in enumerate(coord_args(fn, args)):
        out[f"{name}/arg/{k}"] = np.asarray(a)


def main():
    from oracle import ref_shim
    ref = ref_shim.import_reference()
    from atomai.utils import img, imgen
    fns = {n: getattr(imgen, n) for n in ("create_lattice_mask", "create_multiclass_lattice_mask",
                                          "create_multiclass_lattice_mask_")}
    fns.update({n: getattr(img, n) for n in ("extract_patches_", "extract_patches",
                                             "extract_patches_and_spectra")})
    out = {}
    for i, (sc, rm, it, th) in enumerate(ic.ATOM_GRID):
        g, m = imgen.MakeAtom(sc, rm, it, th, i % 3).gen_atom_mask()
        a = imgen.MakeAtom(sc, rm, it, th, i % 3)
        out[f"atom/{i}/g"], out[f"atom/{i}/mask"] = g, m
        out[f"atom/{i}/x"], out[f"atom/{i}/y"] = a.x, a.y
        out[f"pair/{i}/atom"], out[f"pair/{i}/mask"] = imgen.create_atom_mask_pair(sc, rm, it)
    for name in ic.all_cases():
        record(out, name, fns)
    path = os.path.join(HERE, "imgen_ref.npz")
    np.savez_compressed(path, **out)
    print(f"{path}: {len(out)} arrays, {os.path.getsize(path)} bytes ({ref.__name__})")


if __name__ == "__main__":
    main()
