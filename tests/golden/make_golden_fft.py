"""
Generates tests/golden/fft_ref.npz by running the UNMODIFIED reference's
atomai.utils.img.FFTmask, FFTsub and threshImg (scipy.fftpack) through oracle/ref_shim.py on the
seeded cases of fft_cases.py:

  <case>/F2, <case>/F3box   FFTmask's F2, and the slice of F3 its mask rewrites (the rest of
                            F3 is F2's copy; fft_cases.encode_mask checks that bit for bit)
  <case>/out             FFTsub's or threshImg's result
  <case>/error           the exception's first builtin base class, when the call raises

FFTsub and threshImg cases take their inputs from earlier cases' results, so the cases run in
order.  Run in the build container only:

    python tests/golden/make_golden_fft.py
"""
import builtins
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import fft_cases as fc  # noqa: E402


def error_name(e: BaseException) -> str:
    return next(t.__name__ for t in type(e).__mro__ if getattr(builtins, t.__name__, None) is t)


def main():
    from oracle import ref_shim
    ref = ref_shim.import_reference()
    from atomai.utils import img
    fns = {"FFTmask": img.FFTmask, "FFTsub": img.FFTsub, "threshImg": img.threshImg}
    out, full = {}, {}   # the stored arrays; the whole F3s, which later cases take as input
    getter = lambda k: full[k] if k in full else out[k]
    for name in fc.all_cases():
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", RuntimeWarning)   # 0 / 0 and inf - inf
                res = fc.call(fns, name, getter)
        except Exception as e:  # noqa: BLE001 — the exception type is the golden
            out[f"{name}/error"] = np.array(error_name(e))
            continue
        if fc.all_cases()[name][0] == "FFTmask":
            F2, F3 = (np.asarray(r) for r in res)
            full[f"{name}/F3"] = F3
            for key, r in fc.encode_mask(name, F2, F3).items():
                out[f"{name}/{key}"] = r
        else:
            out[f"{name}/out"] = np.asarray(res)
    path = os.path.join(HERE, "fft_ref.npz")
    np.savez_compressed(path, **out)
    print(f"{path}: {len(out)} arrays, {os.path.getsize(path)} bytes ({ref.__name__})")


if __name__ == "__main__":
    main()
