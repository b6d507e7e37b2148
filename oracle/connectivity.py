"""CPU checker of the surface connectivity tools — TEST INFRASTRUCTURE ONLY.

ctypes wrapper of oracle/connectivity.c (built into oracle/liboracle.so):
the traversal of vtkPolyDataConnectivityFilter, and the outputs of polydata_utils.SelectLargestPart,
SplitDisconectedParts and JoinSeedsParts on arrays, assembled from it.
PARITY WITH VTK UNPINNED: see connectivity.c's header and DESIGN.md §5.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import _faces3, _ptr, lib


def traverse(nv: int, faces, seeds=None) -> dict:
    """The filter's state: region int32 [T] (-1: not visited), point_map int32 [V] (-1: not numbered),
    sizes int64 [R], depth (the most waves of one region that marked a cell). seeds=None is the
    all-regions traversal; a sequence of point ids is the seeded one (one region)."""
    f = _faces3(faces)
    nt = len(f)
    s = np.ascontiguousarray(np.asarray([] if seeds is None else seeds, dtype=np.int64).reshape(-1))
    region = np.empty(nt, np.int32)
    pmap = np.empty(nv, np.int32)
    sizes = np.zeros(max(nt, 1), np.int64)
    counts = np.zeros(4, np.int64)
    rc = lib().orc_conn_run(_ptr(f), C.c_int64(nv), C.c_int64(nt), _ptr(s), C.c_int64(len(s)),
                            C.c_int(int(seeds is not None)), _ptr(region), _ptr(pmap), _ptr(sizes), _ptr(counts))
    if rc:
        raise (MemoryError if rc == 3 else ValueError)(f"connectivity: bad faces or seeds (code {rc})")
    return {"region": region, "point_map": pmap, "sizes": sizes[:counts[0]].copy(), "depth": int(counts[3]),
            "points": int(counts[1]), "cells": int(counts[2])}


def _vtk_points(vertices: np.ndarray, pmap: np.ndarray, n: int):
    ids = np.empty(n, np.int64)
    used = np.nonzero(pmap >= 0)[0]
    ids[pmap[used]] = used
    return vertices[ids], ids


def _part(pts, f, st, cells, compact: bool):
    """(vertices, faces int32 [C,3], point ids, cell ids) of the cells `cells` (ascending); pts: the VTK-form
    (vertices, point ids) of the traversal, shared by every part."""
    v, pids = pts
    fo = st["point_map"][f[cells]].astype(np.int32).reshape(-1, 3)
    if compact and len(cells):
        lo, hi = int(fo.min()), int(fo.max()) + 1
        v, pids, fo = v[lo:hi], pids[lo:hi], fo - lo
    elif compact:
        v, pids = v[:0], pids[:0]
    return v, fo, pids, cells.astype(np.int64)


def select_largest_part(vertices, faces, compact=False):
    f = _faces3(faces)
    st = traverse(len(vertices), f)
    pts = _vtk_points(vertices, st["point_map"], st["points"])
    if len(st["sizes"]) == 0:
        return _part(pts, f, st, np.zeros(0, np.int64), compact)
    r = int(np.argmax(st["sizes"]))           # the first region of the largest size
    return _part(pts, f, st, np.nonzero(st["region"] == r)[0], compact)


def split_disconnected_parts(vertices, faces, compact=False):
    f = _faces3(faces)
    st = traverse(len(vertices), f)
    pts = _vtk_points(vertices, st["point_map"], st["points"])
    order = np.argsort(st["region"], kind="stable")
    ends = np.cumsum(st["sizes"])
    return [_part(pts, f, st, order[e - n:e], compact) for n, e in zip(st["sizes"], ends)]


def join_seeds_parts(vertices, faces, seeds, compact=False):
    f = _faces3(faces)
    st = traverse(len(vertices), f, seeds)
    return _part(_vtk_points(vertices, st["point_map"], st["points"]), f, st, np.nonzero(st["region"] == 0)[0],
                 compact)
