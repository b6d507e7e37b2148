"""CPU checker for "Remove non-visible faces" — TEST INFRASTRUCTURE ONLY.

ctypes wrapper of oracle/visibility.c (built into oracle/liboracle.so) with the
plugin's signature on arrays: remove_non_visible_faces(vertices, faces, positions, remove_visible).
PARITY WITH VTK UNPINNED: see visibility.c's header and DESIGN.md §5.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import _faces3, _ptr, lib

RES = 800
CAMERA_DOUBLES = 32
BIG_BOX = 64
DEFAULT_POSITIONS = ((1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1))


def _positions(positions) -> np.ndarray:
    p = np.ascontiguousarray(np.asarray(positions, dtype=np.float64))
    if p.ndim != 2 or p.shape[1] != 3 or not 1 <= len(p) <= 64:
        raise ValueError("positions: 1..64 directions of 3 components expected")
    if not np.isfinite(p).all() or (p == 0).all(axis=1).any():
        raise ValueError("positions: every direction must be finite and non-zero")
    return p


def bounds(vertices: np.ndarray) -> np.ndarray:
    v = np.ascontiguousarray(vertices, dtype=np.float32)
    b = np.zeros(6, np.float64)
    lib().orc_vis_bounds(_ptr(v), C.c_int64(len(v)), _ptr(b))
    return b


def cameras(bnds, positions=DEFAULT_POSITIONS) -> np.ndarray:
    """[views][32] camera records: composite matrix, position, focal point, view-up, clipping range,
    distance, radius (the layout of b2v_visibility_cameras)."""
    p = _positions(positions)
    b = np.ascontiguousarray(bnds, dtype=np.float64)
    out = np.zeros((len(p), CAMERA_DOUBLES), np.float64)
    rc = lib().orc_vis_cameras(_ptr(b), _ptr(p), C.c_int(len(p)), _ptr(out))
    if rc:
        raise ValueError(f"cameras: bad bounds or positions (code {rc})")
    return out


def remove_non_visible_faces(vertices, faces, positions=DEFAULT_POSITIONS, remove_visible=False, debug=False):
    """(vertices float32 [V',3], faces int32 [T',3]); with debug=True also a dict with the cameras, the
    depth buffers float64 [views][800][800], the per-vertex visibility and the count of triangles whose
    pixel box exceeds 64 pixels (summed over the views)."""
    v = np.asarray(vertices)
    if v.dtype != np.float32:
        raise TypeError("vertices: float32 expected")
    if v.ndim != 2 or v.shape[1] != 3 or len(v) == 0:
        raise ValueError("vertices: [V,3] with V >= 1 expected")
    if not np.isfinite(v).all():
        raise ValueError("vertices must be finite")
    v = np.ascontiguousarray(v)
    f = _faces3(faces)
    if len(f) and (f.min() < 0 or f.max() >= len(v)):
        raise ValueError("faces: index out of range")
    p = _positions(positions)
    nv, nt, nviews = len(v), len(f), len(p)
    cams = np.zeros((nviews, CAMERA_DOUBLES), np.float64)
    zbuf = np.zeros((nviews, RES, RES), np.float64) if debug else None
    vis = np.zeros(nv, np.uint8)
    vo = np.zeros((nv, 3), np.float32)
    fo = np.zeros((max(nt, 1), 3), np.int32)
    counts = np.zeros(3, np.int64)
    rc = lib().orc_vis_run(_ptr(v), C.c_int64(nv), _ptr(f), C.c_int64(nt), _ptr(p), C.c_int(nviews),
                           C.c_int(int(bool(remove_visible))), _ptr(cams), _ptr(zbuf), _ptr(vis), _ptr(vo), _ptr(fo),
                           _ptr(counts))
    if rc:
        raise (MemoryError if rc == 3 else ValueError)(f"remove_non_visible_faces: code {rc}")
    out = vo[:counts[0]].copy(), fo[:counts[1]].copy()
    if not debug:
        return out
    return out + ({"cameras": cams, "zbuf": zbuf, "visible": vis.astype(bool), "big_triangles": int(counts[2])},)
