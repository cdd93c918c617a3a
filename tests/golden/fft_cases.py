"""
Seeded inputs of the FFTmask / FFTsub / threshImg tests (tests/test_fft*.py,
tests/golden/make_golden_fft.py).  Every case is name -> (function name, args factory, kwargs).
The factory takes `gold`, a getter of earlier results by key ("<case>/F3", "<case>/out"), so an
FFTsub case can take the spectrum an FFTmask case produced and a threshImg case the difference
an FFTsub case produced: the generator passes the reference's own results, the tests the
committed ones.  FFTmask results are stored as <case>/F2 and <case>/F3box, the others as
<case>/out.  F3box is the slice F3[m-l:m+l, m-l:m+l] the reference rewrites; outside it F3 is
F2's copy bit for bit, so load_golden rebuilds the whole F3 from the two.  Sides stay at or below
128, and the size cases use float32 images (complex64 spectra), to keep the goldens small; the
GPU tests check the float64 path at every one of these sizes against the float64 oracle.
"""
import numpy as np

DTYPES = (np.uint8, np.int16, np.int32, np.int64, np.bool_, np.float16, np.float32, np.float64,
          np.complex64, np.complex128)
SIZES = ((1, 1), (2, 2), (5, 7), (16, 16), (17, 17), (63, 63), (64, 64), (65, 65), (97, 97),
         (100, 100), (128, 128), (64, 80), (80, 64), (128, 40))
RATIOS = (-5, 0, 1, 1.5, 2, 2.5, 10, 100)


def image(h: int, w: int, seed: int, dtype=np.float64) -> np.ndarray:
    """a smooth lattice-like pattern plus noise, cast to `dtype` over a range that suits it"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    base = np.cos(2 * np.pi * x / 7.3) * np.cos(2 * np.pi * y / 6.1) + 0.3 * rng.standard_normal((h, w))
    dt = np.dtype(dtype)
    if dt == np.bool_:
        return base > 0.2
    if dt.kind in "ui":
        lo = 0 if dt.kind == "u" else -1000
        return np.round(lo + (base + 2) * (200 if dt == np.uint8 else 500)).astype(dt)
    if dt.kind == "c":
        return (base + 1j * rng.standard_normal((h, w))).astype(dt)
    return base.astype(dt)


def special(kind: str) -> np.ndarray:
    img = image(32, 32, 5)
    img[11, 20] = np.nan if kind == "nan" else np.inf
    return img


def all_cases():
    c = {}
    # sizes: powers of two, primes, Bluestein lengths, non-square; the default maskratio
    for h, w in SIZES:
        img = lambda h=h, w=w: image(h, w, h * 1000 + w, np.float32)
        c[f"mask_{h}x{w}"] = ("FFTmask", lambda g, img=img: (img(),), {})
        # 128 x 40 is narrower than the disk's box for every positive ratio: only l < 0 runs
        key = f"mask_{h}x{w}"
        if w < h // 2:
            key = f"mask_{h}x{w}_r-5"
            c[key] = ("FFTmask", lambda g, img=img: (img(),), dict(maskratio=-5))
        if h * w < 10000:   # FFTsub of the largest two: on the GPU against the oracle only
            c[f"sub_{h}x{w}"] = ("FFTsub", lambda g, img=img, key=key: (img(), g(f"{key}/F3")), {})
    # maskratios: negative, zero, too small for the slices, fractional, large; on 32 x 32
    for r in RATIOS:
        c[f"mask_ratio_{r}"] = ("FFTmask", lambda g: (image(32, 32, 3, np.float32),),
                                dict(maskratio=r))
    c["mask_ratio_default"] = ("FFTmask", lambda g: (image(40, 40, 4, np.float32),), {})
    # dtypes, 24 x 32 with a disk of radius 6
    for dt in DTYPES:
        name = np.dtype(dt).name
        img = lambda dt=dt: image(24, 32, 7, dt)
        c[f"mask_{name}"] = ("FFTmask", lambda g, img=img: (img(),), dict(maskratio=4))
        c[f"sub_{name}"] = ("FFTsub", lambda g, img=img, name=name: (img(), g(f"mask_{name}/F3")), {})
        if dt in (np.uint8, np.float32, np.float64):
            # the unmasked spectrum: the difference is rounding noise
            c[f"sub_noise_{name}"] = ("FFTsub", lambda g, img=img, name=name:
                                      (img(), g(f"mask_{name}/F2")), {})
    # a spectrum of the other precision
    c["sub_float32_c128"] = ("FFTsub", lambda g: (image(24, 32, 7, np.float32),
                                                  g("mask_float64/F3")), {})
    c["sub_float64_c64"] = ("FFTsub", lambda g: (image(24, 32, 7), g("mask_float32/F3")), {})
    # non-finite pixels
    for kind in ("nan", "inf"):
        c[f"mask_{kind}"] = ("FFTmask", lambda g, kind=kind: (special(kind),), dict(maskratio=4))
        c[f"sub_{kind}"] = ("FFTsub", lambda g, kind=kind: (special(kind), g("mask_ratio_2.5/F3")),
                            {})
    # constant images: a power-of-two transform of a constant is exact, so the masked spectrum is
    # exactly zero, the difference exactly constant, and the normalisation 0 / 0
    c["mask_const"] = ("FFTmask", lambda g: (np.full((32, 32), 3.0),), dict(maskratio=4))
    c["sub_const"] = ("FFTsub", lambda g: (np.full((32, 32), 3.0), g("mask_const/F3")), {})
    c["mask_const_u8"] = ("FFTmask", lambda g: (np.full((16, 16), 7, np.uint8),), dict(maskratio=4))
    c["sub_const_u8"] = ("FFTsub", lambda g: (np.full((16, 16), 7, np.uint8), g("mask_const_u8/F3")),
                         {})
    # errors
    c["mask_1d"] = ("FFTmask", lambda g: (np.ones(16),), {})
    c["mask_empty"] = ("FFTmask", lambda g: (np.ones((0, 4)),), {})
    c["mask_empty_w"] = ("FFTmask", lambda g: (np.ones((4, 0)),), {})
    c["sub_shapes"] = ("FFTsub", lambda g: (np.ones((20, 32)), g("mask_float64/F3")), {})
    # threshImg on FFTsub results, default and custom thresholds
    for src in ("sub_64x64", "sub_97x97", "sub_float32", "sub_uint8"):
        for lo, hi in ((None, None), (0.1, 0.9), (0.4, 0.6), (0.55, 0.45)):
            kw = {} if lo is None else dict(threshL=lo, threshH=hi)
            c[f"thresh_{src}_{lo}_{hi}"] = ("threshImg", lambda g, src=src: (g(f"{src}/out"),), kw)
    return c


def call(fns, name, gold):
    """runs case `name` with the functions of `fns` (a dict or a module); gold(key) gives earlier
    results"""
    fn, args, kwargs = all_cases()[name]
    f = fns[fn] if isinstance(fns, dict) else getattr(fns, fn)
    return f(*args(gold), **kwargs)


def result_keys(name):
    return ("F2", "F3") if all_cases()[name][0] == "FFTmask" else ("out",)


def mask_slice(name):
    """the slice F3[m-l:m+l, m-l:m+l] FFTmask case `name` rewrites (atomai/utils/img.py:467-471)"""
    _, args, kwargs = all_cases()[name]
    n = args(None)[0].shape[0]
    l, m = int(n / kwargs.get("maskratio", 10)), int(n / 2)
    return np.s_[m - l:m + l, m - l:m + l]


def encode_mask(name, F2: np.ndarray, F3: np.ndarray) -> dict:
    """the stored form of FFTmask's (F2, F3): F2 and the rewritten slice of F3.  Raises if F3
    differs from F2 anywhere else, so load_golden's F3 is the reference's bit for bit."""
    s = mask_slice(name)
    rest = F3.copy()
    rest[s] = F2[s]
    if rest.dtype != F2.dtype or rest.tobytes() != F2.tobytes():
        raise AssertionError(f"{name}: F3 differs from F2 outside the mask slice")
    return {"F2": F2, "F3box": F3[s]}


class load_golden:
    """the goldens of `path` by key, with <case>/F3 rebuilt from <case>/F2 and <case>/F3box"""

    def __init__(self, path):
        self._npz = np.load(path)
        keys = list(self._npz.files)
        self.files = keys + [k[:-len("box")] for k in keys if k.endswith("/F3box")]

    def __getitem__(self, key):
        if key.endswith("/F3") and key not in self._npz.files:
            name = key[:-len("/F3")]
            F3 = self._npz[f"{name}/F2"].copy()
            F3[mask_slice(name)] = self._npz[f"{name}/F3box"]
            return F3
        return self._npz[key]


# ------------------------------------------------------------------ error bounds of the tests
# A radix-2 FFT of L points has a normwise error ||dF|| <= log2(L) eta ||F|| with eta about 3 eps
# (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., thm. 24.2: eta = mu +
# gamma_4 (sqrt 2 + mu), mu the twiddle error).  A Bluestein length runs three such transforms of
# L = next_pow2(2n - 1) points, and a 2-D transform adds the errors of its two axes, so
# 9 log2(L_r L_c) eps bounds the GPU's transform; the host's (numpy's pocketfft or fftpack, both
# mixed-radix) adds at most about 3 log2(n m) eps more.  Hence C64 = 12 against float64 results.
# Single-precision goldens come from fftpack's float32 path, whose error dominates: C32 = 3, plus
# one float32 rounding of the GPU's float64 result.
C64, C32 = 12.0, 3.0
EPS32, EPS64 = float(np.finfo(np.float32).eps), float(np.finfo(np.float64).eps)


def tlen(n: int) -> int:
    """the power-of-two transform length of a side: n itself, or Bluestein's next_pow2(2n - 1)"""
    return n if n & (n - 1) == 0 else 1 << (2 * n - 2).bit_length()


def log2_len(shape) -> float:
    return max(np.log2(tlen(shape[0]) * tlen(shape[1])), 1.0)


def spectrum_tol(F: np.ndarray, single: bool) -> float:
    """normwise bound on ||F_gpu - F_ref||_2 for the reference spectrum F"""
    norm = float(np.linalg.norm(F.astype(np.complex128)))
    if single:
        return (C32 * log2_len(F.shape) + 1) * EPS32 * norm
    return C64 * log2_len(F.shape) * EPS64 * norm


def sub_tol(imgsrc: np.ndarray, imgfft: np.ndarray, raw: np.ndarray, single: bool):
    """elementwise bound on FFTsub's normalised result, or None when the difference is rounding
    noise; `single` when the reference reconstructed in float32 (a complex64 spectrum).  The
    reconstruction's normwise error is the spectrum's divided by sqrt(h w) (Parseval); with the
    rounding of the subtraction it bounds each d by E, and
    (d - min) / (max - min) then moves by at most 4 E / (R - 2 E), R the range of d."""
    eps, c = (EPS32, C32) if single else (EPS64, C64)
    h, w = imgfft.shape
    spec = imgfft.astype(np.complex128)
    recon = float(np.linalg.norm(spec)) / np.sqrt(h * w)
    E = c * log2_len((h, w)) * eps * recon + eps * (float(np.abs(imgsrc.astype(np.complex128)).max())
                                                   + recon)
    R = float(raw.max() - raw.min())
    if not R > 4 * E:
        return None
    return 4 * E / (R - 2 * E) + 4 * eps


def masked(F2: np.ndarray, F3: np.ndarray) -> np.ndarray:
    """where the disk zeroed a non-zero spectrum"""
    return (F3 == 0) & (F2 != 0)
