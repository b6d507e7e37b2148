"""CPU checker of the geodesic surface measurement — TEST INFRASTRUCTURE ONLY.

ctypes wrapper of oracle/geodesic.c (built into oracle/libgeodesic.so by oracle/geodesic.mk): the closest points
of vtkPointLocator, the sequential vtkDijkstraGraphGeodesicPath (distances, heap predecessors and trace), the
per-point ambiguity and the device's predecessor rule, and the path length as measures.py sums it.
PARITY WITH VTK UNPINNED: see geodesic.c's header and DESIGN.md.
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
        so, src = _HERE / "libgeodesic.so", _HERE / "geodesic.c"
        if not so.exists() or so.stat().st_mtime < src.stat().st_mtime:
            subprocess.run(["make", "-C", str(_HERE), "-f", "geodesic.mk"], check=True, capture_output=True)
        _LIB = C.CDLL(str(so))
        _LIB.orc_geodesic_trace.restype = C.c_int64
    return _LIB


def _ptr(a: np.ndarray):
    return C.c_void_p(a.ctypes.data)


def _points(vertices) -> np.ndarray:
    return np.ascontiguousarray(vertices, dtype=np.float64).reshape(-1, 3)


def distances(vertices, faces, start: int) -> dict:
    """The whole distance field from `start`: dist float64 [V] (+inf unreached), pre int64 [V] (the heap's
    predecessors, -1 at the start and where unreached), rule int64 [V] (the smallest (d[u], id) attaining
    neighbour) and amb bool [V] (two distinct attaining neighbours share the smallest d[u])."""
    v, f = _points(vertices), _faces3(faces)
    nv = len(v)
    dist, pre, rule = np.empty(nv), np.empty(nv, np.int64), np.empty(nv, np.int64)
    amb = np.zeros(nv, np.uint8)
    rc = lib().orc_geodesic(_ptr(v), C.c_int64(nv), _ptr(f), C.c_int64(len(f)), C.c_int64(int(start)), _ptr(dist),
                            _ptr(pre), _ptr(rule), _ptr(amb))
    if rc:
        raise (MemoryError if rc == 3 else ValueError)(f"geodesic: bad faces or start (code {rc})")
    return {"dist": dist, "pre": pre, "rule": rule, "amb": amb.astype(bool)}


def trace(pre: np.ndarray, start: int, end: int) -> np.ndarray:
    """TraceShortestPath over `pre`: int64 ids from the end to the start (the end alone when unreached)."""
    pre = np.ascontiguousarray(pre, dtype=np.int64)
    ids = np.empty(len(pre), np.int64)
    n = lib().orc_geodesic_trace(_ptr(pre), C.c_int64(len(pre)), C.c_int64(int(start)), C.c_int64(int(end)),
                                 _ptr(ids))
    if n < 0:
        raise ValueError("geodesic trace: the predecessors form a cycle")
    return ids[:n].copy()


def closest_points(vertices, picks) -> np.ndarray:
    v = _points(vertices)
    p = np.ascontiguousarray(picks, dtype=np.float64).reshape(-1, 3)
    ids = np.empty(len(p), np.int64)
    lib().orc_closest_points(_ptr(v), C.c_int64(len(v)), _ptr(p), C.c_int64(len(p)), _ptr(ids))
    return ids


def path_length(points: np.ndarray, total_in: float = 0.0) -> tuple[float, float]:
    """(segment length summed from 0, total_in with the segment added step by step) over float32 points."""
    p = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 3)
    out = np.zeros(2)
    lib().orc_path_length(_ptr(p), C.c_int64(len(p)), C.c_double(float(total_in)), _ptr(out))
    return float(out[0]), float(out[1])


def geodesic_path(vertices, faces, picks) -> dict:
    """The body of _draw_line: for each pair of consecutive picks, the closest points, the heap's path from the
    first to the second and its length. ids: a list of int64 arrays (one per segment, end to start); points:
    float32 [sum, 3] appended in segment order; lengths: float64 per segment; total; ambiguous / unreached:
    bool per segment (ambiguous: some step of the path other than its start is an ambiguous point)."""
    v, f = _points(vertices), _faces3(faces)
    picks = np.ascontiguousarray(picks, dtype=np.float64).reshape(-1, 3)
    out = {"ids": [], "points": np.zeros((0, 3), np.float32), "lengths": np.zeros(0), "total": 0.0,
           "ambiguous": np.zeros(0, bool), "unreached": np.zeros(0, bool)}
    if len(picks) < 2 or len(f) == 0:
        return out
    snap = closest_points(v, picks)
    pts, lengths, amb, unr, total = [], [], [], [], 0.0
    for s, e in zip(snap[:-1], snap[1:]):
        g = distances(v, f, s)
        ids = trace(g["pre"], s, e)
        p = np.asarray(vertices)[ids].astype(np.float32)
        seg, total = path_length(p, total)
        out["ids"].append(ids)
        pts.append(p)
        lengths.append(seg)
        amb.append(bool(g["amb"][ids[ids != s]].any()))
        unr.append(bool(np.isinf(g["dist"][e])))
    out.update(points=np.concatenate(pts), lengths=np.array(lengths), total=total, ambiguous=np.array(amb),
               unreached=np.array(unr))
    return out
