"""Pre-filters and mask algebra with the reference's signatures (SURVEY 8f-4), numpy in / numpy out:

  median_blur_filter(matrix, value)   invesalius/data/filters.py:9-12   ndimage.median_filter, size 3, 4 or 5
  mean_blur_filter(matrix, value)     filters.py:15-18                  ndimage.uniform_filter(...).astype(dtype)
  boolean_op(op, m1, m2, out)         Slice.do_boolean_op, slice_.py:1906-1916 (mask bodies)
  convolve_non_zero(volume, kernel, cval)   invesalius_rs.convolve_non_zero (calc_mask_area, slice_.py:2299-2322)

  gaussian_blur_filter / despeckle_filter / sharpening_filter / border_detection_filter   filters.py:5-66,
      built from scipy.ndimage.correlate1d evaluated exactly as SciPy evaluates it (b2v_correlate1d)

Bit-exact against SciPy / NumPy.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from . import device as dev
from .device import _p, _stream

BOOLEAN_UNION, BOOLEAN_DIFF, BOOLEAN_AND, BOOLEAN_XOR = 1, 2, 3, 4     # invesalius/constants.py:818-821


def _i16_volume(matrix):
    a = np.asarray(matrix)
    if a.dtype != np.int16 or a.ndim != 3:
        raise TypeError("filter: int16 3-D matrix expected")
    return a


def median_blur_filter(matrix: np.ndarray, value: float) -> np.ndarray:
    a = _i16_volume(matrix)
    size = max(3, min(int(2 * value + 1), 5))
    t = dev.to_device(a)
    out = torch.empty_like(t)
    with torch.cuda.device(t.device):
        _lib.call("b2v_median_filter_i16", _p(t), *a.shape, size, _p(out), _stream())
    res = np.empty(a.shape, np.int16)
    dev.to_host(out, res)
    return res


def mean_blur_filter(matrix: np.ndarray, value: float) -> np.ndarray:
    a = _i16_volume(matrix)
    size = int(2 * value + 1)
    if size < 1:
        raise RuntimeError("incorrect filter size")      # SciPy's message
    t = dev.to_device(a)
    out, tmp = torch.empty_like(t), torch.empty_like(t)
    with torch.cuda.device(t.device):
        _lib.call("b2v_uniform_filter_i16", _p(t), *a.shape, size, _p(out), _p(tmp), _stream())
    res = np.empty(a.shape, np.int16)
    dev.to_host(out, res)
    return res


def _corr(t: torch.Tensor, axis: int, weights: np.ndarray, symmetry: int, out_dtype) -> torch.Tensor:
    """One scipy.ndimage.correlate1d pass (b2v_correlate1d) on a device volume."""
    w = torch.from_numpy(np.ascontiguousarray(weights, dtype=np.float64)).to(t.device)
    out = torch.empty(t.shape, dtype=out_dtype, device=t.device)
    code = {torch.int16: _lib.I16, torch.float64: _lib.F64, torch.float32: _lib.F32}
    with torch.cuda.device(t.device):
        _lib.call("b2v_correlate1d", _p(t), code[t.dtype], *t.shape, axis, _p(w), len(weights) // 2, symmetry, _p(out),
                  code[out_dtype], _stream())
    return out


def _gaussian(t: torch.Tensor, sigma: float, out_dtype) -> torch.Tensor:
    """ndimage.gaussian_filter(x, sigma): one pass per axis, every pass stored in the output dtype."""
    from scipy.ndimage._filters import _gaussian_kernel1d
    sd = float(sigma)
    lw = int(4.0 * sd + 0.5)                      # truncate = 4.0
    w = _gaussian_kernel1d(sd, 0, lw)[::-1]        # gaussian_filter1d passes the reversed kernel to correlate1d
    for axis in range(3):
        t = _corr(t, axis, w, +1, out_dtype)
    return t


def gaussian_blur_filter(matrix: np.ndarray, sigma: float) -> np.ndarray:
    a = _i16_volume(matrix)
    res = np.empty(a.shape, np.int16)
    dev.to_host(_gaussian(dev.to_device(a), sigma, torch.int16), res)
    return res


def despeckle_filter(matrix: np.ndarray, value: float) -> np.ndarray:
    return gaussian_blur_filter(matrix, value)


def sharpening_filter(matrix: np.ndarray, value: float) -> np.ndarray:
    a = _i16_volume(matrix)
    t = dev.to_device(a)
    mm = dev.minmax(t).cpu()
    blurred = _gaussian(_corr_identity_f64(t), 1.0, torch.float64)
    out = torch.empty_like(t)
    with torch.cuda.device(t.device):
        _lib.call("b2v_sharpen_i16", _p(t), _p(blurred), t.numel(), float(value), float(mm[0]), float(mm[1]), _p(out), _stream())
    res = np.empty(a.shape, np.int16)
    dev.to_host(out, res)
    return res


def _corr_identity_f64(t: torch.Tensor) -> torch.Tensor:
    """matrix.astype(float) on the device, through the same kernel (weights [1])."""
    return _corr(t, 0, np.array([1.0]), +1, torch.float64)


def border_detection_filter(matrix: np.ndarray, value: float = 1.0, normalize: bool = True) -> np.ndarray:
    a = _i16_volume(matrix)
    t = dev.to_device(a)
    g = _gaussian(_corr_identity_f64(t), value, torch.float64)
    mags = []
    for axis in range(3):                         # ndimage.sobel(f, axis): derivative along axis, smoothing along the others
        s = _corr(g, axis, np.array([-1.0, 0.0, 1.0]), -1, torch.float64)
        for other in range(3):
            if other != axis:
                s = _corr(s, other, np.array([1.0, 2.0, 1.0]), +1, torch.float64)
        mags.append(s)
    with torch.cuda.device(t.device):
        _lib.call("b2v_sobel_magnitude", _p(mags[0]), _p(mags[1]), _p(mags[2]), t.numel(), _stream())
    mag = mags[0]
    out = torch.empty_like(t)
    rescale, mag_min, mag_range, span, min_val = 0, 0.0, 1.0, 0.0, 0.0
    if normalize:
        mm = dev.minmax(t).cpu()
        min_val, max_val = float(mm[0]), float(mm[1])
        mag_min = float(mag.min().item())
        mag_range = float(mag.max().item()) - mag_min
        if mag_range > 0:
            rescale, span = 1, max_val - min_val
    with torch.cuda.device(t.device):
        _lib.call("b2v_rescale_cast_i16", _p(mag), t.numel(), rescale, mag_min, mag_range, span, min_val, _p(out), _stream())
    res = np.empty(a.shape, np.int16)
    dev.to_host(out, res)
    return res


def boolean_op(op: int, m1: np.ndarray, m2: np.ndarray, out: np.ndarray) -> None:
    """m[:] = <op>(m1 > 2, m2 > 2) * 255 on mask bodies (uint8, same shape; memmap views welcome)."""
    code = {BOOLEAN_UNION: 0, BOOLEAN_DIFF: 1, BOOLEAN_AND: 2, BOOLEAN_XOR: 3}[op]
    for m in (m1, m2, out):
        if not isinstance(m, np.ndarray) or m.dtype != np.uint8 or m.shape != m1.shape:
            raise TypeError("boolean_op: uint8 masks of one shape expected")
    a, b = dev.to_device(m1 if m1.ndim == 3 else m1[None]), dev.to_device(m2 if m2.ndim == 3 else m2[None])
    o = torch.empty_like(a)
    with torch.cuda.device(a.device):
        _lib.call("b2v_boolean_op", _p(a), _p(b), a.numel(), code, _p(o), _stream())
    dev.to_host(o, out if out.ndim == 3 else out[None])


def convolve_non_zero(volume: np.ndarray, kernel: np.ndarray, cval) -> np.ndarray:
    v = np.ascontiguousarray(volume, dtype=np.float64)
    k = np.ascontiguousarray(kernel, dtype=np.float64)
    if v.ndim != 3 or k.ndim != 3:
        raise TypeError("convolve_non_zero: 3-D float64 volume and kernel expected")
    cval = int(cval)
    if not -32768 <= cval <= 32767:
        raise OverflowError("out of range integral type conversion attempted")    # cval: i16 in the reference
    tv, tk = dev.to_device(v), torch.from_numpy(k).to("cuda")
    out = torch.empty_like(tv)
    with torch.cuda.device(tv.device):
        _lib.call("b2v_convolve_non_zero", _p(tv), *v.shape, _p(tk), *k.shape, float(cval), _p(out), _stream())
    res = np.empty(v.shape, np.float64)
    dev.to_host(out, res)
    return res
