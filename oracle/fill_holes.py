"""CPU checker of the surface hole filler — TEST INFRASTRUCTURE ONLY.

ctypes wrapper of oracle/fill_holes.c (built into oracle/liboracle.so): the
sequential vtkFillHolesFilter, with its boundary lines and per-loop records.
PARITY WITH VTK UNPINNED: see fill_holes.c's header and DESIGN.md §5.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import _faces3, _ptr, lib


FILLED, FAILED, TOO_LARGE = 0, 1, 2
FLT_MAX = float(np.finfo(np.float32).max)


def fill_holes(vertices, faces, hole_size=1.0) -> dict:
    """The filter on numpy arrays: vertices float32 [V,3], faces int32/int64 [T,3] or [T,4]. Returns faces
    (int64 [T + N,3]: the input's, then the new triangles), lines (the number of boundary lines) and, per
    valid loop in order, first_line, npts (int64), radius (float64) and status (int8: 0 filled, 1 failed,
    2 too large)."""
    v = np.ascontiguousarray(vertices, dtype=np.float32)
    f = _faces3(faces)
    hole = float(hole_size)
    if hole != hole:
        raise ValueError("fill_holes: the hole size is NaN")
    hole = min(max(hole, 0.0), FLT_MAX)
    nv, nt = len(v), len(f)
    cap = max(3 * nt, 1)
    tris = np.zeros((cap, 3), np.int64)
    first, npts = np.zeros(cap, np.int64), np.zeros(cap, np.int64)
    radius, status = np.zeros(cap, np.float64), np.zeros(cap, np.int8)
    counts = np.zeros(3, np.int64)
    rc = lib().orc_fill_holes(_ptr(v), C.c_int64(nv), _ptr(f), C.c_int64(nt), C.c_double(hole), _ptr(tris),
                              _ptr(first), _ptr(npts), _ptr(radius), _ptr(status), _ptr(counts))
    if rc:
        raise (MemoryError if rc == 3 else ValueError)(f"fill_holes: bad faces (code {rc})")
    nl, nloops, ntris = (int(x) for x in counts)
    return {"faces": np.concatenate([f, tris[:ntris]]), "lines": nl, "first_line": first[:nloops].copy(),
            "npts": npts[:nloops].copy(), "radius": radius[:nloops].copy(), "status": status[:nloops].copy()}
