"""
Seeded inputs of the filter_cells / filter_cells_ tests (tests/test_blobs*.py,
tests/golden/make_golden_blobs.py).  Every case is name -> (function name, args factory, kwargs);
the factory rebuilds the inputs on each call, so the reference and the package get the same
arrays.  Frames stay small enough for compact goldens, but several cross many 32 x 32 tile
boundaries, the unit of the GPU labelling.
"""
import numpy as np

ACCEPTED = (np.uint8, np.int16, np.uint16, np.float32, np.float64)
REJECTED = (np.int8, np.int32, np.int64, np.float16, bool)


def field(h: int, w: int, seed: int, fill: float, dtype=np.float32) -> np.ndarray:
    """uniform noise in [0, 1) whose pixels above 1 - fill (the threshold the cases use) are
    foreground with probability `fill`"""
    return np.random.default_rng(seed).random((h, w)).astype(dtype)


def stack(n: int, h: int, w: int, seed: int, fill: float, dtype=np.float32) -> np.ndarray:
    return np.stack([field(h, w, seed + i, fill, dtype) for i in range(n)]) if n else \
        np.zeros((0, h, w), dtype)


def typed(h: int, w: int, seed: int, dtype):
    """a frame of `dtype` with threshold 0.5 splitting its values roughly 55 / 45, and the
    threshold that does that for its range"""
    rng = np.random.default_rng(seed)
    if dtype == np.uint8:
        return rng.integers(0, 256, (h, w)).astype(dtype), 114.5
    if dtype == np.int16:
        return rng.integers(-3000, 3000, (h, w)).astype(dtype), -300.0
    if dtype == np.uint16:
        return rng.integers(0, 65536, (h, w)).astype(dtype), 29000.25
    return rng.random((h, w)).astype(dtype), 0.45


def sized_blobs() -> np.ndarray:
    """float32 64 x 64 with separated blobs of 1, 3, 4, 5, 9, 12 and 16 pixels, twice each"""
    img = np.zeros((64, 64), np.float32)
    shapes = [(1, 1), (1, 3), (2, 2), (5, 1), (3, 3), (3, 4), (4, 4)]
    for k, (bh, bw) in enumerate(shapes):
        for j in range(2):
            r, c = 2 + 8 * k, 2 + 30 * j + 5 * k % 20
            img[r:r + bh, c:c + bw] = 1.0
    return img


def checkerboard(h: int, w: int) -> np.ndarray:
    return ((np.add.outer(np.arange(h), np.arange(w)) % 2) == 0).astype(np.float32)


def staircases(h: int, w: int) -> np.ndarray:
    """diagonal lines of pixels touching only at corners (one component per pixel under
    4-connectivity), and two-pixel-thick staircases (one component each)"""
    img = np.zeros((h, w), np.float32)
    for i in range(min(h, w)):
        img[i, i] = 1.0
        if i + 40 < w:
            img[i, i + 40] = 1.0
            if i + 41 < w:
                img[i, i + 41] = 1.0
    return img


def snake(h: int, w: int, transpose: bool = False) -> np.ndarray:
    """one 1-pixel-wide path: down a column, two columns right along the edge, up the next, ...;
    every vertical run crosses all horizontal tile boundaries"""
    img = np.zeros((h, w), np.float32)
    for k, c in enumerate(range(0, w, 2)):
        img[:, c] = 1.0
        if c + 2 < w:
            r = h - 1 if k % 2 == 0 else 0
            img[r, c:c + 3] = 1.0
    return img.T.copy() if transpose else img


def comb(h: int, w: int, joined: bool = True) -> np.ndarray:
    """vertical teeth one pixel apart, joined only along the last row (or not at all)"""
    img = np.zeros((h, w), np.float32)
    img[:, ::2] = 1.0
    if joined:
        img[-1, :] = 1.0
    return img


def special(dtype) -> np.ndarray:
    """NaN, +inf and -inf pixels inside foreground blobs, and pixels exactly at float32(0.1)"""
    img = np.zeros((40, 50), dtype)
    img[2:12, 2:12] = 0.7
    img[5, 5] = np.nan            # splits nothing: a NaN pixel is background
    img[5:8, 20:40] = np.inf
    img[20:30, 3:9] = -np.inf
    img[25:35, 20:30] = np.float32(0.1)
    img[30, 20:30] = 0.3
    return img


def all_cases():
    c = {}
    # every accepted dtype, through both functions
    for i, dt in enumerate(ACCEPTED):
        img, th = typed(70, 90, 10 + i, dt)
        name = np.dtype(dt).name
        c[f"dtype_{name}_"] = ("filter_cells_", lambda img=img: (img.copy(),),
                               dict(im_thresh=th, blob_thresh=6))
        st = np.stack([typed(45, 66, 20 + i + 7 * k, dt)[0] for k in range(3)])
        c[f"dtype_{name}_stack"] = ("filter_cells", lambda st=st: (st.copy(),),
                                    dict(im_thresh=th, blob_thresh=4, filter_='above'))
    for dt in REJECTED:
        name = np.dtype(dt).name
        c[f"reject_{name}_"] = ("filter_cells_", lambda dt=dt: (np.ones((8, 8), dt),), {})
        c[f"reject_{name}_stack"] = ("filter_cells", lambda dt=dt: (np.ones((2, 8, 8), dt),), {})
    # size tests: 'below', 'above', an unknown string; areas equal to the threshold
    for bt in (1, 3, 4, 4.5, 9, 12, 16, 17, 0, -1, -2.5, np.nan, 3.9999999, 1e300):
        for f in ("below", "above", "other"):
            c[f"sizes_{bt}_{f}"] = ("filter_cells_", lambda: (sized_blobs(),),
                                    dict(im_thresh=0.5, blob_thresh=bt, filter_=f))
    c["sizes_np_int_above"] = ("filter_cells_", lambda: (sized_blobs(),),
                               dict(blob_thresh=np.int64(9), filter_='above'))
    c["sizes_np_float32"] = ("filter_cells_", lambda: (sized_blobs(),),
                             dict(blob_thresh=np.float32(4.5)))
    # threshold comparisons
    for dt in (np.float32, np.float64):
        name = np.dtype(dt).name
        for th in (0.1, 0.3, 0.7, -1e30, 0.0):
            c[f"special_{name}_{th}"] = ("filter_cells_", lambda dt=dt: (special(dt),),
                                         dict(im_thresh=th, blob_thresh=2))
    u8 = np.random.default_rng(3).integers(0, 6, (50, 60)).astype(np.uint8)
    for th in (2.0, 2.5, 1.9999, -0.5, 255.0, 254.5, 300.0, -300.0):
        c[f"uint8_{th}"] = ("filter_cells_", lambda: (u8.copy(),), dict(im_thresh=th, blob_thresh=3))
    i16 = np.random.default_rng(4).integers(-4, 4, (50, 60)).astype(np.int16)
    for th in (-1.5, -1.0, 0.5, 32767.0, -40000.0):
        c[f"int16_{th}"] = ("filter_cells_", lambda: (i16.copy(),), dict(im_thresh=th, blob_thresh=3))
    # connectivity
    c["checkerboard"] = ("filter_cells_", lambda: (checkerboard(70, 67),), dict(blob_thresh=1))
    c["checkerboard_2"] = ("filter_cells_", lambda: (checkerboard(70, 67),), dict(blob_thresh=2))
    c["staircases"] = ("filter_cells_", lambda: (staircases(90, 130),), dict(blob_thresh=2))
    c["staircases_above"] = ("filter_cells_", lambda: (staircases(90, 130),),
                             dict(blob_thresh=1, filter_='above'))
    c["snake"] = ("filter_cells_", lambda: (snake(130, 161),), dict(blob_thresh=10000))
    c["snake_keep"] = ("filter_cells_", lambda: (snake(130, 161),), dict(blob_thresh=10))
    c["snake_t"] = ("filter_cells_", lambda: (snake(97, 200, True),), dict(blob_thresh=9801))
    c["snake_t_keep"] = ("filter_cells_", lambda: (snake(97, 200, True),), dict(blob_thresh=9800))
    c["comb_joined"] = ("filter_cells_", lambda: (comb(100, 131),), dict(blob_thresh=200))
    c["comb_open"] = ("filter_cells_", lambda: (comb(100, 131, False),), dict(blob_thresh=101))
    c["comb_t"] = ("filter_cells_", lambda: (comb(100, 131).T.copy(),), dict(blob_thresh=200))
    for fill in (0.3, 0.59, 0.8):
        c[f"field_{fill}"] = ("filter_cells_", lambda fill=fill: (field(150, 170, 7, fill),),
                              dict(im_thresh=1 - fill, blob_thresh=20))
    # whole, empty and thin frames; sizes that are not tile multiples
    c["all_fg"] = ("filter_cells_", lambda: (np.ones((100, 90), np.float32),), dict(blob_thresh=9000))
    c["all_fg_drop"] = ("filter_cells_", lambda: (np.ones((100, 90), np.float32),),
                        dict(blob_thresh=9001))
    c["all_bg"] = ("filter_cells_", lambda: (np.zeros((100, 90), np.float32),), {})
    for h, w in ((1, 300), (300, 1), (1, 1), (37, 1000), (1025, 33)):
        c[f"thin_{h}x{w}"] = ("filter_cells_", lambda h=h, w=w: (field(h, w, h + w, 0.6),),
                              dict(im_thresh=0.4, blob_thresh=3))
    c["one_fg_pixel"] = ("filter_cells_", lambda: (np.ones((1, 1)),), dict(blob_thresh=1))
    c["one_fg_pixel_drop"] = ("filter_cells_", lambda: (np.ones((1, 1)),), dict(blob_thresh=2))
    c["empty_frame_"] = ("filter_cells_", lambda: (np.zeros((0, 5), np.float32),), {})
    # stacks
    c["stack_1"] = ("filter_cells", lambda: (stack(1, 80, 75, 30, 0.55),), dict(im_thresh=0.45))
    c["stack_7"] = ("filter_cells", lambda: (stack(7, 66, 99, 40, 0.59),),
                    dict(im_thresh=0.41, blob_thresh=12))
    c["stack_7_above"] = ("filter_cells", lambda: (stack(7, 66, 99, 40, 0.59),),
                          dict(im_thresh=0.41, blob_thresh=30, filter_='above'))
    c["stack_f64_defaults"] = ("filter_cells", lambda: (stack(3, 40, 41, 50, 0.6, np.float64),), {})
    c["stack_empty"] = ("filter_cells", lambda: (stack(0, 10, 10, 0, 0.5),), {})
    c["stack_empty_frames"] = ("filter_cells", lambda: (np.zeros((2, 0, 4), np.float32),), {})
    return c


def call(fns, name):
    """runs case `name` with the functions of `fns` (a dict or a module)"""
    fn, args, kwargs = all_cases()[name]
    f = fns[fn] if isinstance(fns, dict) else getattr(fns, fn)
    return f(*args(), **kwargs)


# The reference's cv2.error (an Exception subclass) for a dtype cv2.threshold rejects is a
# TypeError here; every other exception has the reference's type.
def expected_error(gold_name: str) -> type:
    import builtins
    return TypeError if gold_name == "Exception" else getattr(builtins, gold_name)
