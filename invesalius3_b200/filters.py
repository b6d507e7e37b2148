"""Pre-filters and mask algebra with the reference's signatures (SURVEY 8f-4), numpy in / numpy out:

  median_blur_filter(matrix, value)   invesalius/data/filters.py:9-12   ndimage.median_filter, size 3, 4 or 5
  mean_blur_filter(matrix, value)     filters.py:15-18                  ndimage.uniform_filter(...).astype(dtype)
  boolean_op(op, m1, m2, out)         Slice.do_boolean_op, slice_.py:1906-1916 (mask bodies)
  convolve_non_zero(volume, kernel, cval)   invesalius_rs.convolve_non_zero (calc_mask_area, slice_.py:2299-2322)

  gaussian_blur_filter / despeckle_filter / sharpening_filter / border_detection_filter   filters.py:5-66,
      built from scipy.ndimage.correlate1d evaluated exactly as SciPy evaluates it (b2v_correlate1d)

The six filters take a 3-D int16 volume or a 2-D int16 image (one slice, as the "2D" branch of
Slice.__apply_image_filter passes them). apply_image_filter is that whole branch and the "3D" one
(slice_.py:2363-2422): every slice along the chosen axis is filtered in the same launches, with no pass
along the slice axis and each slice's own statistics where filters.py takes min / max. image_histogram is
the histogram of Slice.matrix (slice_.py:190-192, 2490-2493).

Bit-exact against SciPy / NumPy.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from . import device as dev
from .device import _dense, _p, _stream

BOOLEAN_UNION, BOOLEAN_DIFF, BOOLEAN_AND, BOOLEAN_XOR = 1, 2, 3, 4     # invesalius/constants.py:818-821
ORIENTATION_AXIS = {"Axial": 0, "Coronal": 1, "Sagittal": 2}          # slice_.py:2364
_CODE = {torch.int16: _lib.I16, torch.float64: _lib.F64, torch.float32: _lib.F32}


def _i16_image(matrix):
    a = np.asarray(matrix)
    if a.dtype != np.int16 or a.ndim not in (2, 3):
        raise TypeError("filter: int16 2-D or 3-D matrix expected")
    return a


def _on_device(a: np.ndarray, fn) -> np.ndarray:
    """fn(t, axis) on the uploaded image: a volume whole (axis None), a 2-D image as the one slice of a
    (1, ny, nx) volume (axis 0)."""
    t = dev.to_device(a if a.ndim == 3 else a[None])
    out = fn(t, None if a.ndim == 3 else 0)
    res = np.empty(a.shape, np.int16)
    dev.to_host(out.reshape(a.shape), res)
    return res


def _axes(axis) -> tuple:
    """The axes a filter runs along: all three for a volume, the two in-slice axes (ascending) for slices."""
    return (0, 1, 2) if axis is None else tuple(a for a in range(3) if a != axis)


def _median_size(value) -> int:
    return max(3, min(int(2 * value + 1), 5))


def _mean_size(value) -> int:
    size = int(2 * value + 1)
    if size < 1:
        raise RuntimeError("incorrect filter size")      # SciPy's message
    return size


def _median(t: torch.Tensor, size: int, axis) -> torch.Tensor:
    out = torch.empty_like(t)
    with torch.cuda.device(t.device):
        if axis is None:
            _lib.call("b2v_median_filter_i16", _p(t), *t.shape, size, _p(out), _stream())
        else:
            _lib.call("b2v_median_filter_slices_i16", _p(t), *t.shape, size, axis, _p(out), _stream())
    return out


def _mean(t: torch.Tensor, size: int, axis) -> torch.Tensor:
    out, tmp = torch.empty_like(t), torch.empty_like(t)
    with torch.cuda.device(t.device):
        if axis is None:
            _lib.call("b2v_uniform_filter_i16", _p(t), *t.shape, size, _p(out), _p(tmp), _stream())
        else:
            _lib.call("b2v_uniform_filter_slices_i16", _p(t), *t.shape, size, axis, _p(out), _p(tmp), _stream())
    return out


def median_blur_filter(matrix: np.ndarray, value: float) -> np.ndarray:
    a = _i16_image(matrix)
    size = _median_size(value)
    return _on_device(a, lambda t, axis: _median(t, size, axis))


def mean_blur_filter(matrix: np.ndarray, value: float) -> np.ndarray:
    a = _i16_image(matrix)
    size = _mean_size(value)
    return _on_device(a, lambda t, axis: _mean(t, size, axis))


def _corr(t: torch.Tensor, axis: int, weights: np.ndarray, symmetry: int, out_dtype) -> torch.Tensor:
    """One scipy.ndimage.correlate1d pass (b2v_correlate1d) on a device volume."""
    # a copy: the reversed one-tap Gaussian (sigma < 0.125) is a negative-stride view that counts as contiguous
    w = torch.from_numpy(np.array(weights, dtype=np.float64)).to(t.device)
    out = torch.empty(t.shape, dtype=out_dtype, device=t.device)
    with torch.cuda.device(t.device):
        _lib.call("b2v_correlate1d", _p(t), _CODE[t.dtype], *t.shape, axis, _p(w), len(weights) // 2, symmetry, _p(out),
                  _CODE[out_dtype], _stream())
    return out


def _gaussian(t: torch.Tensor, sigma: float, out_dtype, axes=(0, 1, 2)) -> torch.Tensor:
    """ndimage.gaussian_filter(x, sigma) over `axes`: one pass per axis, every pass stored in the output dtype."""
    from scipy.ndimage._filters import _gaussian_kernel1d
    sd = float(sigma)
    lw = int(4.0 * sd + 0.5)                      # truncate = 4.0
    w = _gaussian_kernel1d(sd, 0, lw)[::-1]        # gaussian_filter1d passes the reversed kernel to correlate1d
    for axis in axes:
        t = _corr(t, axis, w, +1, out_dtype)
    return t


def gaussian_blur_filter(matrix: np.ndarray, sigma: float) -> np.ndarray:
    a = _i16_image(matrix)
    return _on_device(a, lambda t, axis: _gaussian(t, sigma, torch.int16, _axes(axis)))


def despeckle_filter(matrix: np.ndarray, value: float) -> np.ndarray:
    return gaussian_blur_filter(matrix, value)


def _slice_minmax(t: torch.Tensor, axis: int) -> torch.Tensor:
    """[min, max] of every slice along `axis` as float64 pairs (b2v_slice_minmax), left on the device."""
    out = torch.empty((t.shape[axis], 2), dtype=torch.float64, device=t.device)
    with torch.cuda.device(t.device):
        _lib.call("b2v_slice_minmax", _p(t), _CODE[t.dtype], *t.shape, axis, _p(out), _stream())
    return out


def _sharpen(t: torch.Tensor, value: float, axis) -> torch.Tensor:
    blurred = _gaussian(_corr_identity_f64(t), 1.0, torch.float64, _axes(axis))
    out = torch.empty_like(t)
    with torch.cuda.device(t.device):
        if axis is None:
            mm = dev.minmax(t).cpu()
            _lib.call("b2v_sharpen_i16", _p(t), _p(blurred), t.numel(), float(value), float(mm[0]), float(mm[1]), _p(out),
                      _stream())
        else:
            mm = _slice_minmax(t, axis)
            _lib.call("b2v_sharpen_slices_i16", _p(t), _p(blurred), *t.shape, axis, float(value), _p(mm), _p(out),
                      _stream())
    return out


def sharpening_filter(matrix: np.ndarray, value: float) -> np.ndarray:
    a = _i16_image(matrix)
    return _on_device(a, lambda t, axis: _sharpen(t, value, axis))


def _corr_identity_f64(t: torch.Tensor) -> torch.Tensor:
    """matrix.astype(float) on the device, through the same kernel (weights [1])."""
    return _corr(t, 0, np.array([1.0]), +1, torch.float64)


def _border(t: torch.Tensor, value: float, normalize: bool, axis) -> torch.Tensor:
    axes = _axes(axis)
    g = _gaussian(_corr_identity_f64(t), value, torch.float64, axes)
    mags = []
    for a in axes:                                # ndimage.sobel(f, axis): derivative along axis, smoothing along the others
        s = _corr(g, a, np.array([-1.0, 0.0, 1.0]), -1, torch.float64)
        for other in axes:
            if other != a:
                s = _corr(s, other, np.array([1.0, 2.0, 1.0]), +1, torch.float64)
        mags.append(s)
    del g
    with torch.cuda.device(t.device):
        _lib.call("b2v_sobel_magnitude", _p(mags[0]), _p(mags[1]), _p(mags[2] if len(mags) == 3 else None), t.numel(),
                  _stream())
    mag = mags[0]
    del mags[1:]
    out = torch.empty_like(t)
    if axis is not None and normalize:
        img_mm, mag_mm = _slice_minmax(t, axis), _slice_minmax(mag, axis)
        with torch.cuda.device(t.device):
            _lib.call("b2v_rescale_cast_slices_i16", _p(mag), *t.shape, axis, _p(mag_mm), _p(img_mm), _p(out), _stream())
        return out
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
    return out


def border_detection_filter(matrix: np.ndarray, value: float = 1.0, normalize: bool = True) -> np.ndarray:
    a = _i16_image(matrix)
    return _on_device(a, lambda t, axis: _border(t, value, normalize, axis))


# ----------------------------------------------------------------------------- the "Apply image filter" action
def apply_image_filter_device(t: torch.Tensor, filter_type, value, dimension="3D", orientation="Axial"):
    """The filtered image that Slice.__apply_image_filter's filter thread computes (slice_.py:2355-2425), on a
    resident int16 volume: filter_type 0 Gaussian, 1 median, 2 mean, 3 sharpening, 4 despeckle, 5 border
    detection; any other value gives None. dimension "3D" filters the volume; anything else filters every
    slice along the orientation's axis (unknown orientations: axial). Returns a new int16 tensor."""
    _dense(t, "t")
    if t.dtype != torch.int16 or t.dim() != 3:
        raise TypeError("apply_image_filter: int16 3-D volume expected")
    if filter_type not in (0, 1, 2, 3, 4, 5):
        return None
    axis = None if dimension == "3D" else ORIENTATION_AXIS.get(orientation, 0)
    if filter_type in (0, 4):
        return _gaussian(t, value, torch.int16, _axes(axis))
    if filter_type == 1:
        return _median(t, _median_size(value), axis)
    if filter_type == 2:
        return _mean(t, _mean_size(value), axis)
    if filter_type == 3:
        return _sharpen(t, value, axis)
    return _border(t, value, True, axis)


def apply_image_filter(matrix: np.ndarray, filter_type, value, dimension="3D", orientation="Axial"):
    """apply_image_filter_device on a host volume: one upload, the filter's launches, one download. Returns
    the int16 result (Slice._pending_filter_result) or None for an unknown filter_type."""
    a = np.asarray(matrix)
    if a.dtype != np.int16 or a.ndim != 3:
        raise TypeError("apply_image_filter: int16 3-D matrix expected")
    if filter_type not in (0, 1, 2, 3, 4, 5):
        return None
    if filter_type == 2:
        _mean_size(value)                         # raises before any device work
    out = apply_image_filter_device(dev.to_device(a), filter_type, value, dimension, orientation)
    res = np.empty(a.shape, np.int16)
    dev.to_host(out, res)
    return res


def image_histogram_device(t: torch.Tensor):
    """(counts, min, max) of a resident int16 image: counts = np.histogram(a, max - min, (min, max))[0] as an int64
    device tensor, min and max as ints. min == max raises np.histogram's ValueError (bins = 0)."""
    _dense(t, "t")
    if t.dtype != torch.int16:
        raise TypeError("image_histogram: int16 image expected")
    mm = dev.minmax(t).cpu()
    i, e = int(mm[0]), int(mm[1])
    r = e - i
    if r < 1:
        raise ValueError("`bins` must be positive, when an integer")
    counts = torch.empty(r, dtype=torch.int64, device=t.device)
    with torch.cuda.device(t.device):
        _lib.call("b2v_histogram_i16", _p(t), t.numel(), i, r, _p(counts), _stream())
    return counts, i, e


def image_histogram(matrix: np.ndarray):
    """(np.histogram(matrix, r, (i, e))[0], i, e) with i, e = matrix.min(), matrix.max() and r = int(e) - int(i), as
    the Slice.matrix setter and _after_filter compute them; i and e are int16 scalars like NumPy's."""
    a = np.asarray(matrix)
    if a.dtype != np.int16:
        raise TypeError("image_histogram: int16 image expected")
    counts, i, e = image_histogram_device(dev.to_device(a))
    return counts.cpu().numpy(), np.int16(i), np.int16(e)


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
