"""CPU restatement of scipy.ndimage.zoom for spline orders 0-3, modes 'constant' and 'mirror',
prefilter=True, grid_mode=False -- TEST INFRASTRUCTURE ONLY.

Written from the algorithm (a B-spline prefilter with one pole per order, then a separable
B-spline gather), in NumPy, one operation per statement so that every float64 rounding happens
where the device rounds. Vectorised across lines and output voxels; sequential along each line.

  spline_filter(a, order)     the interpolation prefilter over every axis, float64 out
  zoom(a, factors, ...)       the resample, with SciPy's output shape and factor conventions
"""
from __future__ import annotations

import math

import numpy as np

# The poles sqrt(8) - 3 and sqrt(3) - 2, correctly rounded. Evaluating the expressions in float64
# instead loses 7 and 2 ulps to cancellation, which the recursion turns into differences of up to
# thousands of ulps in the coefficients.
POLES = {2: -0.171572875253809902396622551580603843, 3: -0.267949192431122706472553658494127633}


def _filter_axis(c: np.ndarray, order: int, axis: int) -> None:
    """In place along `axis` of the float64 array c: gain, causal init (mirror boundary), forward
    recursion, anticausal init, backward recursion. Lines of length 1 are left as they are."""
    n = c.shape[axis]
    if n == 1:
        return
    v = np.moveaxis(c, axis, 0)                   # a view: v[i] is sample i of every line
    z = POLES[order]
    gain = (1.0 - z) * (1.0 - 1.0 / z)
    v *= gain
    # causal init: c0 = sum over the mirrored line, c0 / (1 - z^(2n-2))
    zn1 = math.pow(z, n - 1)
    c0 = v[0] + zn1 * v[n - 1]
    zi = z
    for i in range(1, n - 1):
        c0 = c0 + zi * (v[i] + zn1 * v[n - 1 - i])
        zi = zi * z
    v[0] = c0 / (1.0 - zn1 * zn1)
    for i in range(1, n):
        v[i] = v[i] + z * v[i - 1]
    v[n - 1] = (z * v[n - 2] + v[n - 1]) * z / (z * z - 1.0)
    for i in range(n - 2, -1, -1):
        v[i] = z * (v[i + 1] - v[i])


def spline_filter(a: np.ndarray, order: int) -> np.ndarray:
    c = np.array(a, dtype=np.float64)
    for axis in range(c.ndim):
        _filter_axis(c, order, axis)
    return c


def weights(x: np.ndarray, order: int):
    """B-spline weights of the order+1 taps starting at `start` for coordinates x (float64 arrays),
    and `start`. The last weight is 1 minus the others, subtracted in order."""
    if order & 1:
        start = np.floor(x)
    else:
        start = np.floor(x + 0.5)
    t = x - start
    w = []
    if order == 1:
        w.append(1.0 - t)
    elif order == 2:
        w1 = 0.75 - t * t
        h = 0.5 - t
        w.append(0.5 * h * h)
        w.append(w1)
    elif order == 3:
        u = 1.0 - t
        w.append(u * u * u / 6.0)
        w.append((t * t * (t - 2.0) * 3.0 + 4.0) / 6.0)
        w.append((u * u * (u - 2.0) * 3.0 + 4.0) / 6.0)
    last = np.ones_like(x)
    for wi in w:
        last = last - wi
    w.append(last)
    return w, start.astype(np.int64) - order // 2


def mirror_index(idx: np.ndarray, n: int) -> np.ndarray:
    """Fold indices into [0, n) by reflection about samples 0 and n-1 (period 2n-2)."""
    if n == 1:
        return np.zeros_like(idx)
    p = 2 * n - 2
    m = np.mod(idx, p)
    return np.where(m >= n, p - m, m)


def output_shape(shape, factors):
    return tuple(int(round(n * f)) for n, f in zip(shape, factors))


def step(n_in: int, n_out: int) -> float:
    """The coordinate step (n_in - 1) / (n_out - 1), or 1 when n_out is 1."""
    return (n_in - 1) / (n_out - 1) if n_out > 1 else 1.0


def _axis_table(n_in: int, n_out: int, order: int, mode: str):
    """Per output index: tap indices [order+1][n_out], weights, and the 'outside' flag."""
    cc = np.arange(n_out, dtype=np.float64) * step(n_in, n_out)
    if mode == "constant":
        outside = cc > n_in - 1                    # strict: exactly n_in - 1 interpolates
    else:
        outside = np.zeros(n_out, bool)
        if n_in == 1:
            cc = np.where(cc > 0, 0.0, cc)
        else:
            p = float(2 * n_in - 2)
            hi = cc > n_in - 1
            f = cc - p * np.trunc(cc / p)
            f = np.where(f >= n_in, p - f, f)
            cc = np.where(hi, f, cc)
    cc = np.where(outside, 0.0, cc)
    w, start = weights(cc, order)
    idx = [mirror_index(start + k, n_in) for k in range(order + 1)]
    return idx, w, outside


def _round_to(t: np.ndarray, dtype) -> np.ndarray:
    dt = np.dtype(dtype)
    if dt.kind == "f":
        return t.astype(dt)
    info = np.iinfo(dt)
    if dt.kind == "u":
        r = np.where(t > 0, t + 0.5, 0.0)
    else:
        r = np.where(t > 0, t + 0.5, t - 0.5)
    r = np.clip(r, info.min, info.max)
    return np.trunc(r).astype(dt)


def zoom(a: np.ndarray, factors, order: int = 3, mode: str = "constant", cval: float = 0.0, out_dtype=None):
    """scipy.ndimage.zoom(a, factors, out_dtype, order, mode, cval) on a 2-D or 3-D array."""
    a = np.asarray(a)
    out_dtype = a.dtype if out_dtype is None else np.dtype(out_dtype)
    if np.ndim(factors) == 0:
        factors = (factors,) * a.ndim
    shape = output_shape(a.shape, factors)
    if all(f == 1 for f in factors):
        return a.astype(out_dtype)
    src = spline_filter(a, order) if order > 1 else a.astype(np.float64)
    tables = [_axis_table(n, m, order, mode) for n, m in zip(a.shape, shape)]
    nd = a.ndim
    t = np.zeros(shape, np.float64)
    outside = np.zeros(shape, bool)
    for ax, (_, _, o) in enumerate(tables):
        outside |= o.reshape([-1 if k == ax else 1 for k in range(nd)])
    # taps in row-major order over the axes; each value times the axis weights in axis order
    for taps in np.ndindex(*(order + 1,) * nd):
        ix = np.ix_(*[tables[ax][0][k] for ax, k in enumerate(taps)])
        coeff = src[ix]
        for ax, k in enumerate(taps):
            coeff = coeff * tables[ax][1][k].reshape([-1 if j == ax else 1 for j in range(nd)])
        t = t + coeff
    t = np.where(outside, float(cval), t)
    return _round_to(t, out_dtype)
