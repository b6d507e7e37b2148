"""CPU checker of the volume rendering's data preparation — TEST INFRASTRUCTURE ONLY.

ctypes wrapper of oracle/raycasting.c (built into oracle/libraycasting.so by oracle/raycasting.mk): the flip and
unsigned-short shift of Volume.LoadVolume, the preset convolutions of ApplyConvolution and the histogram of
CalculateHistogram (invesalius/data/volume.py). PARITY WITH VTK UNPINNED: see raycasting.c's header.
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
_LIB = None


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        so, src = _HERE / "libraycasting.so", _HERE / "raycasting.c"
        if not so.exists() or so.stat().st_mtime < src.stat().st_mtime:
            subprocess.run(["make", "-C", str(_HERE), "-f", "raycasting.mk"], check=True, capture_output=True)
        _LIB = C.CDLL(str(so))
    return _LIB


def _ptr(a: np.ndarray):
    return C.c_void_p(a.ctypes.data)


def _volume(matrix, dtype) -> np.ndarray:
    a = np.asarray(matrix)
    if a.dtype != dtype or a.ndim != 3:
        raise TypeError(f"raycasting: a 3-D {np.dtype(dtype).name} volume expected, not {a.dtype} {a.shape}")
    if a.size == 0:
        raise ValueError("raycasting: empty volume")
    return np.ascontiguousarray(a)


def _weights(w) -> np.ndarray:
    w = np.ascontiguousarray(w, dtype=np.float64).reshape(-1)
    if w.size != 25:
        raise ValueError(f"raycasting: a 5x5 kernel has 25 weights, not {w.size}")
    return w


def flip_shift(matrix) -> tuple[np.ndarray, tuple[float, float]]:
    """(u uint16 [dz][dy][dx], (min, max)): the flipped and shifted volume and the scalar range."""
    m = _volume(matrix, np.int16)
    u = np.empty(m.shape, np.uint16)
    rng = np.zeros(2)
    lib().orc_rc_flip_shift(_ptr(m), *(C.c_int64(s) for s in m.shape), _ptr(u), _ptr(rng))
    return u, (float(rng[0]), float(rng[1]))


def convolve(u, weights) -> np.ndarray:
    """One vtkImageConvolve pass with SetKernel5x5(weights) over every slice of a uint16 volume."""
    a = _volume(u, np.uint16)
    w = _weights(weights)
    out = np.empty(a.shape, np.uint16)
    if lib().orc_rc_convolve(_ptr(a), *(C.c_int64(s) for s in a.shape), _ptr(w), _ptr(out)):
        raise ValueError("raycasting: the weights must be finite, non-negative and sum below 65536 / 65535")
    return out


def convolve_chain(u, kernels) -> np.ndarray:
    """ApplyConvolution: one pass per kernel in list order; no kernels gives u back."""
    out = _volume(u, np.uint16).copy()
    for w in kernels:
        out = convolve(out, w)
    return out


def histogram(matrix) -> tuple[np.ndarray, float, float]:
    """(counts int64 [r], min, max) with r = int(max - min): counts[k] = #(m == min + k), max not counted."""
    m = _volume(matrix, np.int16)
    rng = np.zeros(2)
    lib().orc_rc_range(_ptr(m), C.c_int64(m.size), _ptr(rng))
    r = int(rng[1] - rng[0])
    counts = np.empty(r, np.int64)
    lib().orc_rc_histogram(_ptr(m), C.c_int64(m.size), C.c_int(int(rng[0])), C.c_int64(r), _ptr(counts))
    return counts, float(rng[0]), float(rng[1])
