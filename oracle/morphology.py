"""CPU restatement of the binary morphology kernels (csrc/morphology.cu) — TEST INFRASTRUCTURE ONLY.

binary_morphology(image, op, radius, planar) computes scipy.ndimage.binary_erosion(border_value=True) /
binary_dilation(border_value=False) with the footprint {d : |d|^2 <= radius^2} (skimage's disk per z-slice
when planar, ball otherwise) by the separable bounded squared distance the device uses: per axis,
g <- min over |t| <= r of g[shifted by t] + t^2, clamped at r^2 + 1, with nothing coming from outside the
volume. Whole-array NumPy passes, 3 (2r + 1) of them; tests/test_morphology_model.py pins it to SciPy.
"""
from __future__ import annotations

import numpy as np


def _min_plus(g: np.ndarray, axis: int, r: int, sentinel: int) -> np.ndarray:
    """min over |t| <= r of g[i + t] + t^2 along `axis`; positions outside the volume contribute nothing."""
    out = np.full(g.shape, sentinel, np.uint16)   # g + t^2 <= 2 r^2 + 1 fits for any radius up to 180
    n = g.shape[axis]
    for t in range(-r, r + 1):
        if abs(t) >= n:
            continue
        dst = [slice(None)] * g.ndim
        src = [slice(None)] * g.ndim
        dst[axis] = slice(max(0, -t), n - max(0, t))
        src[axis] = slice(max(0, t), n - max(0, -t))
        np.minimum(out[tuple(dst)], g[tuple(src)] + np.uint16(t * t), out=out[tuple(dst)])
    return np.minimum(out, sentinel)


def binary_morphology(image: np.ndarray, op: str, radius: int, planar: bool) -> np.ndarray:
    """bool result of eroding (op "erosion") or dilating (op "dilation") the non-zero voxels of a 3-D
    `image`; planar: every z-slice on its own with the disk, else the volume with the ball."""
    a = np.asarray(image) != 0
    if a.ndim != 3:
        raise ValueError("3-D image expected")
    if op not in ("erosion", "dilation"):
        raise ValueError(op)
    r = int(radius)
    sentinel = r * r + 1
    src = a if op == "dilation" else ~a     # erosion: the unset voxels are the sources
    g = np.where(src, 0, sentinel).astype(np.uint16)
    for axis in ((2, 1) if planar else (2, 1, 0)):
        g = _min_plus(g, axis, r, sentinel)
    hit = g <= r * r
    return hit if op == "dilation" else ~hit
