"""CPU checker of the surface join — TEST INFRASTRUCTURE ONLY.

The body of join_process_surface (invesalius/data/surface_process.py:228-461) restated sequentially on numpy
arrays, composed of the existing checkers in the reference's order and with the same data passed between
the steps: oracle.clean, oracle.normals, oracle.ca_smoothing, oracle.connectivity and oracle.fill_holes.
It adds no rule of its own beyond the join's: the append, keeping only the triangles of each clean, and the
empty surface. PARITY WITH VTK UNPINNED, as for every checker it calls.
"""
from __future__ import annotations

import numpy as np

import oracle
from oracle import clean as oc, connectivity as ocn, fill_holes as ofh, normals as on


def append(pieces):
    """vtkAppendPolyData: (points float32 [V,3], faces int64 [T,3]), pieces without points skipped."""
    vs, fs, base = [], [], 0
    for v, f in pieces:
        v = np.asarray(v, np.float32).reshape(-1, 3)
        if len(v) == 0:
            continue
        vs.append(v)
        fs.append(np.asarray(f, np.int64).reshape(-1, 3) + base)
        base += len(v)
    if not vs:
        return None, None
    return np.concatenate(vs), np.concatenate(fs)


def clean_triangles(points, faces):
    """oracle.clean with only the triangles kept: (points, faces [T,3], cell_ids of the triangles, the number
    of verts and lines dropped)."""
    c = oc.clean_polydata(points, faces)
    skip = len(c["verts"][0]) - 1 + len(c["lines"][0]) - 1
    return c["points"], c["polys"][1].reshape(-1, 3), c["cell_ids"][skip:], skip


def join(pieces, algorithm, keep_largest, fill_holes, options) -> dict:
    """pieces: (vertices, faces) numpy arrays in append order. Returns points, faces (int64),
    point_normals, cell_normals, volume, area and dropped_cells, as join_surface_device does."""
    points, faces = append(pieces)
    dropped = 0
    if points is not None:
        points, faces, _, dropped = clean_triangles(points, faces)
        if len(faces) == 0:
            points = None
    if algorithm == "ca_smoothing":
        if points is not None:
            n = on.compute_normals(points, faces, 30.0, False)
            points, faces, cell_ids, more = clean_triangles(n["points"], n["faces"])
            dropped += more
            cell_normals = np.ascontiguousarray(n["cell_normals"][cell_ids])
        T, tmax, bmin, steps = (options[k] for k in ("angle", "max distance", "min weight", "steps"))
        if points is not None:
            points = points.copy()
            faces4 = np.ascontiguousarray(np.concatenate([np.full((len(faces), 1), 3, np.int64), faces], 1))
            oracle.ca_smoothing(points, faces4, cell_normals, T, tmax, bmin, steps)
    if keep_largest and points is not None:
        points, faces, _, _ = ocn.select_largest_part(points, faces)
        faces = faces.astype(np.int64)
    if fill_holes and points is not None:
        faces = ofh.fill_holes(points, faces, 300.0)["faces"]
    if points is None:
        z = np.zeros((0, 3), np.float32)
        return {"points": z, "faces": np.zeros((0, 3), np.int64), "point_normals": z.copy(), "cell_normals": z.copy(),
                "volume": 0.0, "area": 0.0, "dropped_cells": dropped}
    volume, area = on.mass_properties(points, faces)
    n = on.compute_normals(points, faces, 80.0, True)
    return {"points": n["points"], "faces": n["faces"], "point_normals": n["point_normals"],
            "cell_normals": n["cell_normals"], "volume": volume, "area": area, "dropped_cells": dropped}
