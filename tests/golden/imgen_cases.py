"""
Seeded inputs of the utils.imgen / patch-extraction tests (tests/test_imgen*.py,
tests/golden/make_golden_imgen.py).  Every case is (name, function, args, kwargs, setup): `args`
is rebuilt on each call of the case function, so a test can hand the same inputs to the reference
and to the package; `setup` (or None) runs just before the call (the global numpy seed for
random_state=None).  Images stay at 128² or below so the goldens stay small.
"""
import numpy as np

# ------------------------------------------------------------------ lattices


def square(n: int, spacing: float, seed: int, jitter: float = 0.3, origin: float = 4.0):
    rng = np.random.default_rng(seed)
    ij = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 2)
    return origin + ij * spacing + rng.normal(0, jitter, ij.shape)


def honeycomb(nx: int, ny: int, a: float, seed: int, jitter: float = 0.25, origin: float = 6.0):
    rng = np.random.default_rng(seed)
    pts = []
    for i in range(nx):
        for j in range(ny):
            x0, y0 = origin + i * 1.5 * a, origin + j * np.sqrt(3) * a + (i % 2) * np.sqrt(3) / 2 * a
            pts += [(x0, y0), (x0 + a, y0)]
    pts = np.array(pts)
    return pts + rng.normal(0, jitter, pts.shape)


def with_classes(xy: np.ndarray, classes, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    return np.concatenate([xy, rng.choice(classes, (len(xy), 1)).astype(np.float64)], 1)


def image(h: int, w: int, seed: int, dtype=np.float64, channels: int = 0):
    rng = np.random.default_rng(seed)
    shape = (h, w) if not channels else (h, w, channels)
    return (rng.random(shape) * 200).astype(dtype)


# ------------------------------------------------------------------ mask functions


def asym_mask(scale, rmask, z=1):
    """odd 5 x 5 template with every element distinct, so a transposition or a shift shows"""
    t = np.arange(25, dtype=np.float64).reshape(5, 5) / 7.0 + 0.25 * z
    t[0, 0] = -1.5              # negative: clamped in multiclass masks, wraps in uint8
    return None, t


def row_mask(scale, rmask, z=1):
    """1-D template of 5: broadcasts over any number of rows"""
    return None, np.array([0.5, 1.0, 2.0, 3.0, 4.0]) * z


def even_mask(scale, rmask, z=1):
    return None, np.ones((4, 4))


def class_mask(scale, rmask, z):
    """class-dependent 5 x 5 template of non-binary values, so the background sums are inexact"""
    t = np.full((5, 5), 0.1 * z + 0.013)
    t[1:4, 1:4] = 0.37 / z
    return None, t


def small_class_mask(scale, rmask, z):
    """class_mask scaled down, so sums over many classes stay below 1 and the background shows
    the order of the sum"""
    t = np.full((5, 5), 0.003 * np.sqrt(z) + 1e-4)
    t[1:4, 1:4] = 0.0017 / z
    return None, t


def bad_mask(scale, rmask, z=1):
    raise ZeroDivisionError("mask function failed")


def tiny_mask(scale, rmask, z=1):
    return None, np.ones((1, 1)) * 3


# ------------------------------------------------------------------ cases


def _pile(seed):
    rng = np.random.default_rng(seed)
    xy = 30 + rng.uniform(-1.4, 1.4, (64, 2))
    z = (np.arange(64) % 2).astype(np.float64)
    return np.concatenate([xy, z[:, None]], 1)


def _many_classes(seed):
    """300 atoms of 200 classes piled into a 10 x 10 patch, so a pixel holds many classes and the
    background sums more than 128 channels (numpy's recursive pairwise split)"""
    rng = np.random.default_rng(seed)
    xy = rng.uniform(7, 16, (300, 2))
    z = np.concatenate([np.arange(1, 201), rng.integers(1, 201, 100)]).astype(np.float64)
    return np.concatenate([xy, rng.permutation(z)[:, None]], 1)


def _ties():
    return np.array([[10.5, 11.5], [20.5, 20.5], [12.5, 30.0], [31.5, 8.5], [40.0, 40.5]])


def _edges(h):
    # far edge, negative wrapped (x = -3 with 5 rows: rows h-6 ... h-2), and clamped slices
    return np.array([[h - 1.0, 10.0], [h - 2.2, 20.0], [-3.0, 30.0], [5.0, -3.0], [1.0, 40.0],
                     [-1.0, 50.0]])


def lattice_cases():
    sq = square(7, 8.0, 1)
    hc = honeycomb(5, 5, 5.0, 2)
    return [
        ("lat_square_f64", "create_lattice_mask", lambda: (image(64, 64, 1), sq.copy()), {}),
        ("lat_honeycomb_f32", "create_lattice_mask",
         lambda: (image(80, 80, 2, np.float32), hc.copy()), {}),
        ("lat_ties_u8", "create_lattice_mask", lambda: (image(48, 48, 3, np.uint8), _ties()), {}),
        ("lat_wrap_default", "create_lattice_mask",
         lambda: (image(40, 64, 4), np.array([[-3.0, 10.0], [20.0, -3.0], [-3.2, -2.8]])), {}),
        ("lat_edges_row", "create_lattice_mask",
         lambda: (image(40, 64, 4, np.float32), _edges(40)), {}, row_mask),
        ("lat_overlap_2px", "create_lattice_mask",
         lambda: (image(32, 32, 5), np.array([[10.0, 10.0], [12.0, 12.0]])), {}),
        ("lat_asym_u8", "create_lattice_mask", lambda: (image(40, 40, 6, np.uint8), sq[:12] / 2 + 4),
         {}, asym_mask),
        ("lat_asym_f32", "create_lattice_mask", lambda: (image(40, 40, 6, np.float32), sq[:12] / 2 + 4),
         {}, asym_mask),
        ("lat_scale_rmask", "create_lattice_mask", lambda: (image(64, 64, 7), sq.copy()),
         {"scale": 9, "rmask": 7}),
        ("lat_tiny", "create_lattice_mask", lambda: (image(16, 16, 8), sq[:4] / 3), {}, tiny_mask),
        ("lat_empty", "create_lattice_mask", lambda: (image(16, 16, 8), np.zeros((0, 2))), {}),
        ("lat_list_rows", "create_lattice_mask", lambda: (image(32, 32, 9), [(8, 8), (20.5, 9.5)]),
         {}),
        # the reference's errors
        ("err_lat_edge", "create_lattice_mask", lambda: (image(32, 32, 1), np.array([[5., 5.],
                                                                                    [31., 10.]])),
         {}),
        ("err_lat_even", "create_lattice_mask", lambda: (image(32, 32, 1), sq[:3] / 2), {},
         even_mask),
        ("err_lat_nan", "create_lattice_mask",
         lambda: (image(32, 32, 1), np.array([[5., 5.], [np.nan, 3.], [np.inf, 3.]])), {}),
        ("err_lat_inf", "create_lattice_mask",
         lambda: (image(32, 32, 1), np.array([[5., 5.], [8., -np.inf], [np.nan, 3.]])), {}),
        ("err_lat_cols", "create_lattice_mask", lambda: (image(32, 32, 1), np.ones((3, 3)) * 9), {}),
        ("err_lat_func", "create_lattice_mask", lambda: (image(32, 32, 1), sq[:3]), {}, bad_mask),
        ("err_lat_edge_before_nan", "create_lattice_mask",
         lambda: (image(32, 32, 1), np.array([[0., 5.], [np.nan, 3.]])), {}),
    ]


def multiclass_cases():
    sq = square(7, 8.0, 11)
    hc = honeycomb(5, 5, 5.0, 12)
    dense = square(14, 2.0, 13, jitter=0.4, origin=5.0)
    two = {0: with_classes(sq, [0, 1], 14), 1: with_classes(sq + 0.7, [0, 1], 15)}
    return [
        ("mc_square_class0", "create_multiclass_lattice_mask_",
         lambda: (image(64, 64, 1), with_classes(sq, [0, 1], 1)), {}),
        ("mc_honeycomb_123", "create_multiclass_lattice_mask_",
         lambda: (image(80, 80, 2, np.float32), with_classes(hc, [1, 2, 3], 2)), {}),
        ("mc_nine_dense", "create_multiclass_lattice_mask_",
         lambda: (image(40, 40, 3), with_classes(dense, np.arange(1, 10), 3)), {}, class_mask),
        ("mc_twelve_dense", "create_multiclass_lattice_mask_",
         lambda: (image(40, 40, 3), with_classes(dense, np.arange(0, 12), 4)), {}, class_mask),
        ("mc_pile64", "create_multiclass_lattice_mask_", lambda: (image(64, 64, 4), _pile(4)), {}),
        ("mc_asym_negative", "create_multiclass_lattice_mask_",
         lambda: (image(40, 40, 5), with_classes(sq[:12] / 2 + 4, [2, 5], 5)), {}, asym_mask),
        ("mc_edges_row", "create_multiclass_lattice_mask_",
         lambda: (image(40, 64, 6), np.concatenate([_edges(40), np.ones((6, 1))], 1)), {},
         row_mask),
        ("mc_ties", "create_multiclass_lattice_mask_",
         lambda: (image(48, 48, 7), np.concatenate([_ties(), np.zeros((5, 1))], 1)),
         {"scale": 5, "rmask": 5}),
        ("mcs_dict2", "create_multiclass_lattice_mask",
         lambda: (np.stack([image(64, 64, 8), image(64, 64, 9)]),
                  {k: v.copy() for k, v in two.items()}), {}),
        ("mcs_2d_array", "create_multiclass_lattice_mask",
         lambda: (image(64, 64, 10), with_classes(sq, [1, 3], 10)), {}),
        ("mcs_list_result", "create_multiclass_lattice_mask",
         lambda: (np.stack([image(64, 64, 11)] * 3),
                  {0: with_classes(sq, [0, 1], 16), 1: with_classes(sq, [1, 2, 3], 17),
                   2: with_classes(sq, [4], 18)}), {}),
        ("mcs_by_key", "create_multiclass_lattice_mask",
         lambda: (np.stack([image(64, 64, 12)] * 2),
                  {1: with_classes(sq, [1, 2], 19), 0: with_classes(sq[:5], [1], 20)}), {}),
        ("mc_200_classes", "create_multiclass_lattice_mask_",
         lambda: (image(24, 24, 21), _many_classes(21)), {}, small_class_mask),
        ("err_mc_nan_class", "create_multiclass_lattice_mask_",
         lambda: (image(32, 32, 1), np.array([[5., 5., 1.], [12., 10., np.nan], [31., 10., 1.]])),
         {}, asym_mask),
        ("err_mc_nan_class_default", "create_multiclass_lattice_mask_",
         lambda: (image(32, 32, 1), np.array([[5., 5., 1.], [12., 10., np.nan]])), {}),
        ("err_mc_edge_before_nan_class", "create_multiclass_lattice_mask_",
         lambda: (image(32, 32, 1), np.array([[5., 5., 1.], [31., 10., 1.], [12., 10., np.nan]])),
         {}, asym_mask),
        ("err_mc_inf_before_nan_class", "create_multiclass_lattice_mask_",
         lambda: (image(32, 32, 1), np.array([[5., np.inf, 1.], [12., 10., np.nan]])), {},
         asym_mask),
        ("err_mc_cols", "create_multiclass_lattice_mask_",
         lambda: (image(32, 32, 1), np.ones((3, 4)) * 9), {}),
        ("err_mc_edge", "create_multiclass_lattice_mask_",
         lambda: (image(32, 32, 1), np.array([[5., 5., 0.], [31., 10., 1.]])), {}),
        ("err_mcs_key", "create_multiclass_lattice_mask",
         lambda: (np.stack([image(32, 32, 1)] * 2), {0: with_classes(sq[:2] + 10, [1], 1)}), {}),
    ]


def _seed7():
    np.random.seed(7)


def patch_cases():
    im = lambda: image(28, 30, 21)
    m_bool = lambda: image(28, 30, 22) > 100
    m_u8 = lambda: image(28, 30, 23, np.uint8, channels=1)
    m_f64 = lambda: image(28, 30, 24, channels=3)
    return [
        ("p_int_none", "extract_patches_", lambda: (im(), m_bool(), 16, None), {}),
        ("p_int_below", "extract_patches_", lambda: (im(), m_u8(), 16, 50), {"random_state": 3}),
        ("p_int_above", "extract_patches_", lambda: (im(), m_f64(), 16, 10**6), {}),
        ("p_frac", "extract_patches_", lambda: (im(), m_bool(), 16, 0.3), {"random_state": 11}),
        ("p_frac_rounding", "extract_patches_",
         lambda: (image(25, 25, 27), image(25, 25, 28, channels=3), 16, 0.29),
         {"random_state": 4}),
        ("p_rect", "extract_patches_", lambda: (im(), m_f64(), (12, 20), 30), {"random_state": 5}),
        ("p_rect_list", "extract_patches_", lambda: (im(), m_u8(), [20, 12], 30), {}),
        ("p_randomstate", "extract_patches_",
         lambda: (im(), m_f64(), 16, 40, ), {"random_state": "RandomState(5)"}),
        ("p_none_seed", "extract_patches_", lambda: (im(), m_bool(), 16, 40),
         {"random_state": None}, None, _seed7),
        ("p_u8_image", "extract_patches_",
         lambda: (image(40, 40, 25, np.uint8), image(40, 40, 26, np.float32), 8, 20), {}),
        ("pb_stack", "extract_patches",
         lambda: (np.stack([image(40, 40, s) for s in (31, 32, 33)]),
                  np.stack([image(40, 40, s, channels=3) for s in (34, 35, 36)]), 16, 25),
         {"random_state": 2}),
        ("pb_stack_none", "extract_patches",
         lambda: (np.stack([image(40, 40, s) for s in (31, 32)]),
                  np.stack([image(40, 40, s) > 90 for s in (34, 35)]), 16, 25),
         {"random_state": None}, None, _seed7),
        ("pb_2d", "extract_patches", lambda: (im(), m_bool(), 16, 10), {}),
        ("pb_list_frames", "extract_patches",
         lambda: ([image(28, 30, s) for s in (37, 38)], [image(28, 30, s) > 50 for s in (39, 40)],
                  12, 15), {"random_state": 6}),
        ("err_p_list_image", "extract_patches_",
         lambda: (image(28, 30, 21).tolist(), m_bool(), 16, 10), {}),
        ("err_p_big", "extract_patches_", lambda: (im(), m_bool(), (16, 31), 10), {}),
        ("err_p_nan", "extract_patches_",
         lambda: (np.where(im() > 190, np.nan, im()), m_bool(), 16, 10), {}),
        ("err_p_mask_inf", "extract_patches_",
         lambda: (im(), np.where(m_f64() > 190, np.inf, 0.0), 16, 10), {}),
        ("err_p_complex", "extract_patches_", lambda: (im() + 1j, m_bool(), 16, 10), {}),
        ("err_p_zero", "extract_patches_", lambda: (im(), m_bool(), 16, 0), {}),
        ("err_p_float", "extract_patches_", lambda: (im(), m_bool(), 16, 1.5), {}),
    ]


def spectra_cases():
    rng = np.random.default_rng(41)
    h3 = rng.random((32, 32, 16))
    h4 = rng.random((24, 24, 8, 8)).astype(np.float32)
    c3 = np.concatenate([rng.uniform(0, 31, (30, 2)),
                         [[0.2, 5.0], [31.4, 30.6], [-0.7, 10.0], [-4.6, -4.5], [15.5, 16.5]]])
    c4 = np.concatenate([rng.uniform(0, 23, (20, 2)), [[23.0, 23.0], [-2.3, 7.0], [3.5, -3.5]]])
    return [
        ("s3_int_band", "extract_patches_and_spectra", lambda: (h3.copy(),),
         {"coordinates": c3, "window_size": 8, "band": 3}),
        ("s3_list_band", "extract_patches_and_spectra", lambda: (h3.copy(),),
         {"coordinates": c3, "window_size": 7, "band": [2, 6], "avg_pool": 4}),
        ("s3_image", "extract_patches_and_spectra", lambda: (h3.copy(), image(32, 32, 42)),
         {"coordinates": c3, "window_size": 8}),
        ("s4_int_band", "extract_patches_and_spectra", lambda: (h4.copy(),),
         {"coordinates": c4, "window_size": 6, "band": 2}),
        ("s4_list2", "extract_patches_and_spectra", lambda: (h4.copy(),),
         {"coordinates": c4, "window_size": 6, "band": [1, 4]}),
        ("s4_list4", "extract_patches_and_spectra", lambda: (h4.copy(),),
         {"coordinates": c4, "window_size": 5, "band": [1, 4, 2, 6], "avg_pool": 4}),
        ("err_s_2d", "extract_patches_and_spectra", lambda: (h3[..., 0].copy(),),
         {"coordinates": c3, "window_size": 8}),
        ("err_s_image3d", "extract_patches_and_spectra", lambda: (h3.copy(), h3.copy()),
         {"coordinates": c3, "window_size": 8}),
    ]


def all_cases():
    """name -> (function name, args factory, kwargs, mask function or None, setup or None)"""
    out = {}
    for case in lattice_cases() + multiclass_cases() + patch_cases() + spectra_cases():
        name, fn, args, kwargs = case[:4]
        mask = case[4] if len(case) > 4 else None
        setup = case[5] if len(case) > 5 else None
        out[name] = (fn, args, kwargs, mask, setup)
    return out


def call(module_fns, name):
    """runs case `name` with the functions of `module_fns` (a dict or module); returns
    (result, args) so a test can see the in-place class shift"""
    fn, args, kwargs, mask, setup = all_cases()[name]
    a = list(args())
    kw = dict(kwargs)
    if kw.get("random_state") == "RandomState(5)":
        kw["random_state"] = np.random.RandomState(5)
    if mask is not None:
        a.append(mask)
    if setup is not None:
        setup()
    f = module_fns[fn] if isinstance(module_fns, dict) else getattr(module_fns, fn)
    return f(*a, **kw), a


# (sc, r_mask, intensity, theta) grid of MakeAtom / create_atom_mask_pair
ATOM_GRID = [(sc, rm, it, th) for sc in (4, 5, 7, 12) for rm in (3, 5, 8)
             for it in (1, 0.5) for th in (0, 0.4)]


def assert_case(gold, fns, name, host=lambda a: a):
    """runs case `name` with `fns` and checks it against the goldens bit for bit: values, dtype,
    shape, array / list / tuple, the caller's coordinates after the call, or the exception's type.
    `host` turns a result item into numpy (for CUDA results)."""
    import builtins
    import pytest
    if f"{name}/error" in gold.files:
        with pytest.raises(getattr(builtins, str(gold[f"{name}/error"]))):
            call(fns, name)
        return
    res, args = call(fns, name)
    kind = str(gold[f"{name}/kind"])
    assert (kind == "list") == isinstance(res, list) and (kind == "tuple") == isinstance(res, tuple)
    items = list(res) if kind != "array" else [res]
    assert len(items) == len([k for k in gold.files if k.startswith(f"{name}/out/")])
    for k, a in enumerate(items):
        a, ref = np.asarray(host(a)), gold[f"{name}/out/{k}"]
        assert a.shape == ref.shape and a.dtype == ref.dtype, (name, k, a.shape, a.dtype)
        assert a.tobytes() == ref.tobytes(), (name, k)
    fn = all_cases()[name][0]
    if fn.startswith("create_multiclass_lattice_mask"):
        c = args[1]
        for k, a in enumerate([c[i] for i in sorted(c)] if isinstance(c, dict) else [c]):
            np.testing.assert_array_equal(a, gold[f"{name}/arg/{k}"])
