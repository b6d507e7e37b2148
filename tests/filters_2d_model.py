"""NumPy / SciPy statements of the image-filter action (Slice.__apply_image_filter, slice_.py:2355-2425, and the
filters of invesalius/data/filters.py), for the tests of invesalius3_b200.filters:

  loop_2d             the "2D" branch restated: one filters.py statement sequence per slice, slice by slice
  whole_volume_2d     the same result computed over the whole volume the way the device does it: no pass
                      along the slice axis, per-slice minimum / maximum, per-slice normalisation
  filter_3d           the "3D" branch restated
  histogram_by_count  np.histogram(a, r, (i, e)) as unit-bin counts (the device's formulation)
"""
import numpy as np
from scipy import ndimage

AXIS = {"Axial": 0, "Coronal": 1, "Sagittal": 2}


def median_size(value):
    return max(3, min(int(2 * value + 1), 5))


def mean_size(value):
    return int(2 * value + 1)


def _filter(f, filter_type, value):
    """filters.py's six functions on one array (2-D slice or 3-D volume), restated with SciPy calls."""
    if filter_type in (0, 4):
        return ndimage.gaussian_filter(f, sigma=value)
    if filter_type == 1:
        return ndimage.median_filter(f, size=median_size(value))
    if filter_type == 2:
        return ndimage.uniform_filter(f, size=mean_size(value)).astype(f.dtype)
    if filter_type == 3:
        min_val, max_val = f.min(), f.max()
        float_matrix = f.astype(float)
        blurred = ndimage.gaussian_filter(float_matrix, sigma=1.0)
        detail = float_matrix - blurred
        sharpened = float_matrix + value * 0.5 * detail
        return np.clip(sharpened, min_val, max_val).astype(f.dtype)
    float_matrix = ndimage.gaussian_filter(f.astype(float), sigma=value)
    sx = ndimage.sobel(float_matrix, axis=0)
    sy = ndimage.sobel(float_matrix, axis=1)
    if float_matrix.ndim == 3:
        magnitude = np.sqrt(sx**2 + sy**2 + ndimage.sobel(float_matrix, axis=2) ** 2)
    else:
        magnitude = np.sqrt(sx**2 + sy**2)
    min_val, max_val = float(f.min()), float(f.max())
    mag_min = magnitude.min()
    mag_range = magnitude.max() - mag_min
    if mag_range > 0:
        magnitude = (magnitude - mag_min) / mag_range * (max_val - min_val) + min_val
    return magnitude.astype(f.dtype)


def filter_3d(matrix, filter_type, value):
    if filter_type not in range(6):
        return None
    return _filter(matrix, filter_type, value).astype(matrix.dtype)


def loop_2d(matrix, filter_type, value, orientation="Axial"):
    if filter_type not in range(6):
        return None
    axis = AXIS.get(orientation, 0)
    result = np.zeros_like(matrix)
    for i in range(matrix.shape[axis]):
        idx = [slice(None)] * 3
        idx[axis] = i
        result[tuple(idx)] = _filter(matrix[tuple(idx)], filter_type, value)
    return result.astype(matrix.dtype)


def _per_axis(axis, on, off):
    return tuple(off if a == axis else on for a in range(3))


def _slice_stat(a, axis, fn):
    """fn over every slice along `axis`, broadcastable against `a`."""
    return fn(a, axis=tuple(b for b in range(3) if b != axis), keepdims=True)


def whole_volume_2d(matrix, filter_type, value, orientation="Axial"):
    if filter_type not in range(6):
        return None
    axis = AXIS.get(orientation, 0)
    in_slice = [a for a in range(3) if a != axis]
    if filter_type in (0, 4):
        return ndimage.gaussian_filter(matrix, sigma=_per_axis(axis, value, 0))
    if filter_type == 1:
        return ndimage.median_filter(matrix, size=_per_axis(axis, median_size(value), 1))
    if filter_type == 2:
        return ndimage.uniform_filter(matrix, size=_per_axis(axis, mean_size(value), 1)).astype(matrix.dtype)
    lo, hi = _slice_stat(matrix, axis, np.min), _slice_stat(matrix, axis, np.max)
    f = matrix.astype(float)
    if filter_type == 3:
        blurred = ndimage.gaussian_filter(f, sigma=_per_axis(axis, 1.0, 0))
        return np.clip(f + value * 0.5 * (f - blurred), lo, hi).astype(matrix.dtype)
    g = ndimage.gaussian_filter(f, sigma=_per_axis(axis, value, 0))
    terms = []
    for a in in_slice:       # 2-D sobel: the derivative along a, the smoothing along the other in-slice axis only
        s = ndimage.correlate1d(g, [-1, 0, 1], a)
        terms.append(ndimage.correlate1d(s, [1, 2, 1], in_slice[1] if a == in_slice[0] else in_slice[0]))
    magnitude = np.sqrt(terms[0] ** 2 + terms[1] ** 2)
    mag_min = _slice_stat(magnitude, axis, np.min)
    mag_range = _slice_stat(magnitude, axis, np.max) - mag_min
    with np.errstate(divide="ignore", invalid="ignore"):
        scaled = (magnitude - mag_min) / mag_range * (hi.astype(float) - lo.astype(float)) + lo.astype(float)
    return np.where(mag_range > 0, scaled, magnitude).astype(matrix.dtype)


def histogram_by_count(a):
    i, e = int(a.min()), int(a.max())
    c = np.bincount((a.ravel().astype(np.int64) - i), minlength=e - i + 1)
    c[-2] += c[-1]
    return c[:-1]


def image(shape, seed, constant_slices=()):
    """A smooth-plus-noise int16 image; constant_slices: (axis, index, value) triples set to one value."""
    rng = np.random.default_rng(seed)
    a = (ndimage.gaussian_filter(rng.normal(size=shape), 1.0) * 3000 + rng.normal(size=shape) * 200).astype(np.int16)
    for axis, i, v in constant_slices:
        idx = [slice(None)] * 3
        idx[axis] = i
        a[tuple(idx)] = v
    return a
