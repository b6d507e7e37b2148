"""CPU restatement of scipy.ndimage.shift (spline orders 0-3, modes 'constant' and 'mirror', prefilter=True)
and of the parallel form of imagedata_utils.FixGantryTilt -- test infrastructure only.

shift() reuses oracle/zoom.py's prefilter, weights, mirror folding and rounding; only the coordinates differ
from zoom's: o + (-shift) per axis, which can be negative, so 'constant' mode writes cval on both sides and
'mirror' folds negative coordinates the way SciPy's map_coordinate does.

FixGantryTilt shifts slice n in place with cval = matrix.min() of the partly shifted volume. Its parallel form:
  cval[n]       = min(min of original slices n.., min over k < n of shifted_min[k])
  shifted_min[k] = min(min of slice k's in-range outputs, cval[k] if slice k has an out-of-range output)
The in-range outputs do not depend on cval and the out-of-range set depends on the shift alone, so every slice
can be interpolated first, then the cvals come from a scan over nz scalars, then the out-of-range outputs are
filled.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import zoom as oz


def coordinates(n: int, s: float, mode: str):
    """Sampled coordinates of the n outputs of an axis shifted by s, and the 'constant' mode outside flags."""
    cc = np.arange(n, dtype=np.float64) + (-np.float64(s))   # SciPy negates the shift, then adds it
    outside = np.zeros(n, bool)
    if mode == "constant":
        outside = (cc < 0) | (cc > n - 1)                    # strict on both sides
    elif n == 1:
        cc = np.zeros(n)
    else:
        p = 2 * n - 2
        lo = (p * np.trunc(-cc / p).astype(np.int64)).astype(np.float64) + cc
        lo = np.where(lo <= 1 - n, lo + p, -lo)
        hi = cc - float(p) * np.trunc(cc / float(p))
        hi = np.where(hi >= n, p - hi, hi)
        cc = np.where(cc < 0, lo, np.where(cc > n - 1, hi, cc))
    return np.where(outside, 0.0, cc), outside


def shift(a: np.ndarray, shift, order: int = 3, mode: str = "constant", cval: float = 0.0, out_dtype=None):
    """scipy.ndimage.shift(a, shift, out_dtype, order, mode, cval) on a 2-D or 3-D array."""
    a = np.asarray(a)
    out_dtype = a.dtype if out_dtype is None else np.dtype(out_dtype)
    shifts = (shift,) * a.ndim if np.ndim(shift) == 0 else tuple(shift)
    src = oz.spline_filter(a, order) if order > 1 else a.astype(np.float64)
    nd = a.ndim
    tables = []
    outside = np.zeros(a.shape, bool)
    for ax, (n, s) in enumerate(zip(a.shape, shifts)):
        cc, out = coordinates(n, s, mode)
        w, start = oz.weights(cc, order)
        tables.append(([oz.mirror_index(start + k, n) for k in range(order + 1)], w))
        outside |= out.reshape([-1 if k == ax else 1 for k in range(nd)])
    t = np.zeros(a.shape, np.float64)
    # taps in row-major order over the axes; each value times the axis weights in axis order
    for taps in np.ndindex(*(order + 1,) * nd):
        coeff = src[np.ix_(*[tables[ax][0][k] for ax, k in enumerate(taps)])]
        for ax, k in enumerate(taps):
            coeff = coeff * tables[ax][1][k].reshape([-1 if j == ax else 1 for j in range(nd)])
        t = t + coeff
    t = np.where(outside, float(cval), t)
    return oz._round_to(t, out_dtype)


def tilt_shifts(nz: int, spacing, tilt) -> list[float]:
    """FixGantryTilt's per-slice y shifts, in its float64 expressions and order."""
    gntan = math.tan(np.radians(tilt))
    return [-(gntan * n * spacing[2]) / spacing[1] for n in range(nz)]


def slice_outside(ny: int, nx: int, sy: float, sx: float) -> np.ndarray:
    """'constant' mode out-of-range outputs of a 2-D slice shifted by (sy, sx)."""
    return coordinates(ny, sy, "constant")[1][:, None] | coordinates(nx, sx, "constant")[1][None, :]


def cval_chain(orig_min, inrange_min, has_out) -> list[int]:
    """Per-slice cvals from the per-slice minima (inrange_min None where a slice has no in-range output)."""
    nz = len(orig_min)
    suffix = [0] * nz
    run = None
    for n in range(nz - 1, -1, -1):
        run = orig_min[n] if run is None else min(run, orig_min[n])
        suffix[n] = run
    cvals, shifted = [], None
    for n in range(nz):
        c = suffix[n] if shifted is None else min(suffix[n], shifted)
        cvals.append(c)
        cand = [v for v in (inrange_min[n], c if has_out[n] else None) if v is not None]
        if cand:
            shifted = min(cand) if shifted is None else min(shifted, *cand)
    return cvals


def fix_gantry_tilt(matrix: np.ndarray, spacing, tilt, interp=None):
    """The parallel form of FixGantryTilt on a copy of `matrix`: returns (result, per-slice cvals).
    interp(slice, (sy, 0), cval) is the 2-D order-3 interpolator (SciPy's shift by default)."""
    if interp is None:
        from scipy import ndimage as ndi

        def interp(sl, sh, cval):
            return ndi.shift(sl, sh, cval=cval)
    nz, ny, nx = matrix.shape
    shifts = tilt_shifts(nz, spacing, tilt)
    out = np.empty_like(matrix)
    outside, inrange_min, orig_min = [], [], []
    for n in range(nz):
        orig_min.append(int(matrix[n].min()))
        out[n] = interp(matrix[n], (shifts[n], 0), 0)
        mask = slice_outside(ny, nx, shifts[n], 0)
        outside.append(mask)
        inrange_min.append(int(out[n][~mask].min()) if not mask.all() else None)
    cvals = cval_chain(orig_min, inrange_min, [m.any() for m in outside])
    for n in range(nz):
        out[n][outside[n]] = cvals[n]
    return out, cvals


def reference_loop(matrix: np.ndarray, spacing, tilt):
    """FixGantryTilt restated as it runs, on a copy of `matrix`, with SciPy's shift: (result, cvals)."""
    from scipy.ndimage import shift as nd_shift
    matrix = matrix.copy()
    angle = np.radians(tilt)
    spacing = spacing[0], spacing[1], spacing[2]
    gntan = math.tan(angle)
    cvals = []
    for n, slice_ in enumerate(matrix):
        offset = gntan * n * spacing[2]
        cvals.append(int(matrix.min()))
        matrix[n] = nd_shift(slice_, (-offset / spacing[1], 0), cval=matrix.min())
    return matrix, cvals
