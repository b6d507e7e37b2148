"""CPU checker of the Laplacian surface smoothing — TEST INFRASTRUCTURE ONLY.

ctypes wrapper of oracle/smoothing.c (built into oracle/libsmoothing.so by oracle/smoothing.mk): the
sequential vtkSmoothPolyDataFilter, with its point types and edge lists.
PARITY WITH VTK UNPINNED: see smoothing.c's header and DESIGN.md §5.
"""
from __future__ import annotations

import ctypes as C
import math
import subprocess
from pathlib import Path

import numpy as np

from oracle.connectivity import _faces3

_HERE = Path(__file__).resolve().parent
_LIB = None


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        so, src = _HERE / "libsmoothing.so", _HERE / "smoothing.c"
        if not so.exists() or so.stat().st_mtime < src.stat().st_mtime:
            subprocess.run(["make", "-C", str(_HERE), "-f", "smoothing.mk"], check=True, capture_output=True)
        _LIB = C.CDLL(str(so))
    return _LIB


def _ptr(a: np.ndarray):
    return C.c_void_p(a.ctypes.data)


def cosine(angle: float) -> float:
    """cos of an angle in degrees clamped to [0, 180], as VTK's filter takes it."""
    return math.cos(min(max(float(angle), 0.0), 180.0) * (math.pi / 180.0))


def smooth(vertices, faces, iterations=20, relaxation_factor=0.01, feature_angle=45.0, edge_angle=15.0,
           feature_edge_smoothing=False, boundary_smoothing=True, convergence=0.0) -> dict:
    """The filter on numpy arrays: vertices float32 [V,3], faces int32/int64 [T,3] or [T,4]. Returns the moved
    vertices (float32 [V,3]), types int8 [V], lists (one int32 array per point, in VTK's order) and the
    number of iterations done."""
    v = np.ascontiguousarray(np.array(vertices, dtype=np.float32, copy=True))
    f = _faces3(faces)
    nv, nt = len(v), len(f)
    types = np.zeros(nv, np.int8)
    nlist = np.zeros(nv, np.int32)
    lists = np.zeros(max(6 * nt, 1), np.int32)
    counts = np.zeros(2, np.int64)
    conv = min(max(float(convergence), 0.0), 1.0)
    rc = lib().orc_smooth_run(_ptr(v), C.c_int64(nv), _ptr(f), C.c_int64(nt), C.c_int64(int(iterations)),
                              C.c_double(float(relaxation_factor)), C.c_double(cosine(feature_angle)),
                              C.c_double(cosine(edge_angle)), C.c_int(int(bool(feature_edge_smoothing))),
                              C.c_int(int(bool(boundary_smoothing))), C.c_double(conv), _ptr(types), _ptr(nlist),
                              _ptr(lists), _ptr(counts))
    if rc:
        raise (MemoryError if rc == 3 else ValueError)(f"smoothing: bad faces or iterations (code {rc})")
    ends = np.cumsum(nlist)
    return {"vertices": v, "types": types, "lists": np.split(lists[:counts[1]], ends[:-1]) if nv else [],
            "iterations": int(counts[0])}
