"""
Host restatement of FFTmask, FFTsub and threshImg (atomai/utils/img.py:455-499) with numpy.fft in
float64, for sizes beyond the goldens.  Every transform runs in complex128 whatever the input's
dtype; the result is then rounded to the dtype the reference returns, as the GPU path does.
fftsub(..., raw=True) also returns the unnormalised difference, whose range the tests divide
error bounds by.
"""
import numpy as np

_SINGLE = tuple(np.dtype(t) for t in (np.float16, np.float32, np.complex64))


def fftmask(imgsrc: np.ndarray, maskratio=10):
    out_dt = np.complex64 if imgsrc.dtype in _SINGLE else np.complex128
    F2 = np.fft.fftshift(np.fft.fft2(imgsrc.astype(np.complex128)))
    F3 = F2.copy()
    l = int(imgsrc.shape[0] / maskratio)
    m = int(imgsrc.shape[0] / 2)
    y, x = np.ogrid[1: 2 * l + 1, 1:2 * l + 1]
    mask = (x - l) * (x - l) + (y - l) * (y - l) <= l * l
    F3[m - l:m + l, m - l:m + l] = F3[m - l:m + l, m - l:m + l] * (1 - mask)
    return F2.astype(out_dt), F3.astype(out_dt)


def fftsub(imgsrc: np.ndarray, imgfft: np.ndarray, raw: bool = False):
    out_dt = np.result_type(imgsrc.dtype, imgfft.real.dtype)
    out_dt = np.empty(0, out_dt).real.dtype
    recon = np.real(np.fft.ifft2(np.fft.ifftshift(imgfft.astype(np.complex128))))
    src = imgsrc.astype(np.complex128 if imgsrc.dtype.kind == "c" else np.float64)
    d = np.abs(src - recon)
    with np.errstate(invalid="ignore", divide="ignore"):
        n = (d - np.amin(d)) / (np.amax(d) - np.amin(d))
    return (n.astype(out_dt), d) if raw else n.astype(out_dt)


def threshimg(diff: np.ndarray, threshL: float = 0.25, threshH: float = 0.75) -> np.ndarray:
    return (diff < threshL) + (diff > threshH)
