"""CPU checker of the surface clean and triangle filter — TEST INFRASTRUCTURE ONLY.

ctypes wrapper of oracle/clean.c (built into oracle/libclean.so by oracle/clean.mk): sequential
vtkCleanPolyData and vtkTriangleFilter on polys and strips. Inputs take the forms the product takes (faces
[T,3] / [T,4] with a leading 3, or an (offsets, connectivity) pair); outputs are int64 cell arrays.
PARITY WITH VTK UNPINNED: see clean.c's header.
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
        so, src = _HERE / "libclean.so", _HERE / "clean.c"
        if not so.exists() or so.stat().st_mtime < src.stat().st_mtime:
            subprocess.run(["make", "-C", str(_HERE), "-f", "clean.mk"], check=True, capture_output=True)
        _LIB = C.CDLL(str(so))
    return _LIB


def _ptr(a: np.ndarray):
    return C.c_void_p(a.ctypes.data)


def cell_array(x):
    """(offsets int64 [n + 1], connectivity int64) of None, faces [T,3] / [T,4] or an (offsets, conn) pair."""
    if x is None:
        return np.zeros(1, np.int64), np.zeros(0, np.int64)
    if isinstance(x, (tuple, list)):
        offs, conn = (np.ascontiguousarray(a, dtype=np.int64) for a in x)
        if offs.size == 0:
            offs = np.zeros(1, np.int64)
        if offs[-1] != conn.size:
            raise ValueError("malformed offsets: the last must be the connectivity's length")
        return offs, conn
    f = np.asarray(x)
    if f.ndim != 2 or f.shape[1] not in (3, 4):
        raise ValueError("faces [T,3] or [T,4] expected")
    if f.shape[1] == 4:
        if (f[:, 0] != 3).any():
            raise ValueError("faces [T,4] must lead with 3")
        f = f[:, 1:]
    return np.arange(0, 3 * len(f) + 1, 3, dtype=np.int64), np.ascontiguousarray(f, dtype=np.int64).reshape(-1)


def _raise(rc: int, what: str):
    if rc == 3:
        raise MemoryError(what)
    raise ValueError(f"{what}: {'malformed offsets' if rc == 4 else 'a point id outside [0, V)'}")


def clean_polydata(points, polys=None, strips=None) -> dict:
    """The clean on numpy arrays: points float32, point_ids, verts / lines / polys / strips as (offsets,
    connectivity) int64 pairs, cell_ids int64."""
    P = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 3)
    po, pc = cell_array(polys)
    so, sc = cell_array(strips)
    np_, ns = len(po) - 1, len(so) - 1
    cap, gcap = max(pc.size + sc.size, 1), np_ + ns + 1
    pts, pid = np.zeros((cap, 3), np.float32), np.zeros(cap, np.int64)
    vconn, lconn, pconn, sconn = (np.zeros(2 * cap, np.int64) for _ in range(4))
    poffs, soffs, cell_ids = (np.zeros(gcap, np.int64) for _ in range(3))
    counts = np.zeros(7, np.int64)
    rc = lib().orc_clean(_ptr(P), C.c_int64(len(P)), _ptr(po), _ptr(pc), C.c_int64(np_), _ptr(so), _ptr(sc),
                         C.c_int64(ns), _ptr(pts), _ptr(pid), _ptr(vconn), _ptr(lconn), _ptr(poffs), _ptr(pconn),
                         _ptr(soffs), _ptr(sconn), _ptr(cell_ids), _ptr(counts))
    if rc:
        _raise(rc, "clean_polydata")
    n, nv_, nl, npc, npk, nsc, nsk = (int(x) for x in counts)
    return {"points": pts[:n].copy(), "point_ids": pid[:n].copy(),
            "verts": (np.arange(nv_ + 1, dtype=np.int64), vconn[:nv_].copy()),
            "lines": (np.arange(0, 2 * nl + 1, 2, dtype=np.int64), lconn[:2 * nl].copy()),
            "polys": (poffs[:npc + 1].copy(), pconn[:npk].copy()),
            "strips": (soffs[:nsc + 1].copy(), sconn[:nsk].copy()),
            "cell_ids": cell_ids[:nv_ + nl + npc + nsc].copy()}


def triangle_filter(points, polys=None, strips=None) -> dict:
    """The triangle filter: faces int64 [T,3] and cell_ids int64 [T]."""
    P = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 3)
    nv = len(P)
    po, pc = cell_array(polys)
    so, sc = cell_array(strips)
    cap = max(pc.size + sc.size, 1)
    tris, cell_ids, nt = np.zeros((cap, 3), np.int64), np.zeros(cap, np.int64), np.zeros(1, np.int64)
    rc = lib().orc_triangle_filter(_ptr(P), C.c_int64(nv), _ptr(po), _ptr(pc), C.c_int64(len(po) - 1), _ptr(so),
                                   _ptr(sc), C.c_int64(len(so) - 1), _ptr(tris), _ptr(cell_ids), _ptr(nt))
    if rc:
        _raise(rc, "triangle_filter")
    return {"faces": tris[:nt[0]].copy(), "cell_ids": cell_ids[:nt[0]].copy()}
