"""utils.imgen and the patch functions without a GPU: MakeAtom and create_atom_mask_pair equal the
reference bit for bit; the host restatement (oracle/imgen_ref.py) reproduces the reference's masks
in tests/golden/imgen_ref.npz; every error the reference raises is raised, with its type, before
any device work; spectra (host only) equal the goldens; the public signatures are the reference's."""
import inspect
import os

import numpy as np
import pytest

import imgen_cases as ic
from atomai_b200 import ops, utils
from atomai_b200.utils import graphx, img, imgen
from oracle import imgen_ref

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "imgen_ref.npz"))
FNS = {n: getattr(utils, n) for n in ("create_lattice_mask", "create_multiclass_lattice_mask",
                                      "create_multiclass_lattice_mask_", "extract_patches_",
                                      "extract_patches", "extract_patches_and_spectra")}


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("i", range(len(ic.ATOM_GRID)))
def test_make_atom_bit_identical(i):
    sc, rm, it, th = ic.ATOM_GRID[i]
    a = imgen.MakeAtom(sc, rm, it, th, i % 3)
    assert same_bits(a.x, GOLD[f"atom/{i}/x"]) and same_bits(a.y, GOLD[f"atom/{i}/y"])
    g, m = a.gen_atom_mask()
    assert same_bits(g, GOLD[f"atom/{i}/g"]) and same_bits(m, GOLD[f"atom/{i}/mask"])
    g, m = imgen.create_atom_mask_pair(sc, rm, it)
    assert same_bits(g, GOLD[f"pair/{i}/atom"]) and same_bits(m, GOLD[f"pair/{i}/mask"])
    for attr in ("xo", "yo", "sigma_x", "sigma_y", "intensity", "theta", "offset", "r_mask"):
        assert hasattr(a, attr)


def _oracle(name):
    fn, args, kwargs, mask, _ = ic.all_cases()[name]
    a = args()
    make = mask or imgen.create_atom_mask_pair
    if fn == "create_lattice_mask":
        return [imgen_ref.lattice_mask(a[0], a[1], make, **kwargs)]
    if fn == "create_multiclass_lattice_mask_":
        return [imgen_ref.multiclass_mask(a[0].shape, a[1], make, **kwargs)]
    imgs = a[0] if a[0].ndim == 3 else a[0][None]
    d = a[1] if isinstance(a[1], dict) else {0: a[1]}
    return [imgen_ref.multiclass_mask(im.shape, d[i], make, **kwargs) for i, im in enumerate(imgs)]


MASK_CASES = [n for n, c in ic.all_cases().items()
              if c[0].startswith("create_") and f"{n}/error" not in GOLD.files]


@pytest.mark.parametrize("name", MASK_CASES)
def test_oracle_equals_goldens(name):
    got = _oracle(name)
    if str(GOLD[f"{name}/kind"]) == "list":
        ref = [GOLD[f"{name}/out/{k}"] for k in range(len(got))]
    else:
        ref = GOLD[f"{name}/out/0"]
        ref = list(ref) if ref.ndim == 4 else [ref]
    assert len(got) == len(ref)
    for a, b in zip(got, ref):
        assert same_bits(a, b), name


def _no_device(monkeypatch):
    def fail(*a, **k):
        raise AssertionError("device work before the argument checks")
    for name in ("imgen_masks", "gather_patches"):
        monkeypatch.setattr(ops, name, fail)
    monkeypatch.setattr(img, "_device_bits", fail)
    monkeypatch.setattr(imgen, "_device_bits", fail)
    monkeypatch.setattr(graphx, "_check_free", fail)


ERROR_CASES = [n for n in ic.all_cases() if f"{n}/error" in GOLD.files]


@pytest.mark.parametrize("name", ERROR_CASES)
def test_errors_before_device_work(monkeypatch, name):
    _no_device(monkeypatch)
    ic.assert_case(GOLD, FNS, name)


def test_unsupported_dtypes_raise_type_error(monkeypatch):
    _no_device(monkeypatch)
    xy = np.array([[8.0, 8.0]])
    with pytest.raises(TypeError):
        utils.create_lattice_mask(np.zeros((16, 16), np.complex128), xy)
    with pytest.raises(TypeError):
        utils.create_lattice_mask(np.zeros((16, 16), object), xy)
    with pytest.raises(TypeError):
        utils.extract_patches_(np.zeros((16, 16), np.longdouble), np.zeros((16, 16)), 4, 2)


@pytest.mark.parametrize("name", [n for n, c in ic.all_cases().items()
                                  if c[0] == "extract_patches_and_spectra"])
def test_spectra_equal_goldens(name):
    ic.assert_case(GOLD, FNS, name)


def test_exports_and_signatures_equal_the_reference():
    ref = {
        "MakeAtom": "(sc=5, r_mask=3, intensity=1, theta=0, offset=0)",
        "create_atom_mask_pair": "(sc=5, r_mask=5, intensity=1)",
        "create_lattice_mask": "(lattice, xy_atoms, *args, **kwargs)",
        "create_multiclass_lattice_mask": "(imgdata, coord_class_dict, *args, **kwargs)",
        "create_multiclass_lattice_mask_": "(lattice, xyz_atoms, *args, **kwargs)",
        "extract_patches_": "(lattice_im, lattice_mask, patch_size, num_patches, **kwargs)",
        "extract_patches": "(images, masks, patch_size, num_patches, **kwargs)",
        "extract_patches_and_spectra": "(hdata, *args, coordinates=None, window_size=None, "
                                       "avg_pool=2, **kwargs)",
    }
    for name, sig in ref.items():
        f = getattr(utils, name)
        assert f is getattr(imgen if hasattr(imgen, name) else img, name)
        s = inspect.signature(f)
        plain = s.replace(parameters=[p.replace(annotation=p.empty) for p in s.parameters.values()],
                          return_annotation=s.empty)
        assert str(plain) == sig, name
    for meth, sig in (("atom2dgaussian", "()"), ("circularmask", "(image, radius)"),
                      ("gen_atom_mask", "()")):
        s = inspect.signature(getattr(imgen.MakeAtom(), meth))
        assert str(s.replace(parameters=[p.replace(annotation=p.empty)
                                         for p in s.parameters.values()],
                             return_annotation=s.empty)) == sig
