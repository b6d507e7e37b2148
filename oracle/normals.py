"""CPU checker of surface normals and mass properties — TEST INFRASTRUCTURE ONLY.

ctypes wrapper of oracle/normals.c (built into oracle/libnormals.so by oracle/normals.mk): the sequential
vtkPolyDataNormals (consistent order, auto-orientation, feature splitting, cell and point normals) and
vtkMassProperties' volume and area.
PARITY WITH VTK UNPINNED: see normals.c's header and DESIGN.md §5.
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

from oracle.connectivity import _faces3

_HERE = Path(__file__).resolve().parent
_LIB = None


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        so, src = _HERE / "libnormals.so", _HERE / "normals.c"
        if not so.exists() or so.stat().st_mtime < src.stat().st_mtime:
            subprocess.run(["make", "-C", str(_HERE), "-f", "normals.mk"], check=True, capture_output=True)
        _LIB = C.CDLL(str(so))
    return _LIB


def _ptr(a: np.ndarray):
    return C.c_void_p(a.ctypes.data)


def compute_normals(vertices, faces, feature_angle=30.0, auto_orient=False) -> dict:
    """The filter on numpy arrays: vertices float32 [V,3], faces int32/int64 [T,3] or [T,4]. Returns points
    float32 [V + new,3], faces int64 [T,3], point_normals float32 [V + new,3], cell_normals float32 [T,3],
    regions, flips, new_points and waves."""
    v = np.ascontiguousarray(vertices, dtype=np.float32)
    f = _faces3(faces)
    nv, nt = len(v), len(f)
    cap = nv + 3 * nt
    pts, pn = np.zeros((cap, 3), np.float32), np.zeros((cap, 3), np.float32)
    fo, cn = np.zeros((nt, 3), np.int64), np.zeros((nt, 3), np.float32)
    counts = np.zeros(4, np.int64)
    rc = lib().orc_normals(_ptr(v), C.c_int64(nv), _ptr(f), C.c_int64(nt), C.c_double(float(feature_angle)),
                           C.c_int(int(bool(auto_orient))), _ptr(pts), _ptr(fo), _ptr(pn), _ptr(cn), _ptr(counts))
    if rc:
        raise (MemoryError if rc == 3 else ValueError)(f"normals: bad faces or angle (code {rc})")
    n = nv + int(counts[2])
    return {"points": pts[:n].copy(), "faces": fo, "point_normals": pn[:n].copy(), "cell_normals": cn,
            "regions": int(counts[0]), "flips": int(counts[1]), "new_points": int(counts[2]),
            "waves": int(counts[3])}


def mass_properties(vertices, faces, terms: bool = False):
    """(volume, area) as vtkMassProperties gives them; with terms=True also the per-triangle terms float64
    [T,4] (area and the x, y, z projected-volume terms) and classes int8 [T]."""
    v = np.ascontiguousarray(vertices, dtype=np.float32)
    f = _faces3(faces)
    nt = len(f)
    t, c = np.zeros((nt, 4), np.float64), np.zeros(nt, np.int8)
    out = np.zeros(2, np.float64)
    rc = lib().orc_mass_properties(_ptr(v), C.c_int64(len(v)), _ptr(f), C.c_int64(nt), _ptr(t), _ptr(c), _ptr(out))
    if rc:
        raise (MemoryError if rc == 3 else ValueError)(f"mass_properties: bad faces (code {rc})")
    return (float(out[0]), float(out[1]), t, c) if terms else (float(out[0]), float(out[1]))
