"""Meshes for the visible-faces tests, and a plain-Python restatement of the plugin's last step (select the
faces of the selected points, then vtkCleanPolyData's merge and first-use numbering) to check both the C
checker and the device against."""
from __future__ import annotations

import numpy as np


def icosphere(radius: float, level: int, center=(0.0, 0.0, 0.0)):
    """Shared-vertex icosphere: float32 [V,3], int32 [T,3] (outward, counter-clockwise)."""
    t = (1.0 + 5 ** 0.5) / 2.0
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t),
         (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
         (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10),
         (8, 6, 7), (9, 8, 1)]
    verts = [np.array(p, np.float64) / np.linalg.norm(p) for p in v]
    for _ in range(level):
        mid = {}

        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                p = verts[a] + verts[b]
                verts.append(p / np.linalg.norm(p))
                mid[k] = len(verts) - 1
            return mid[k]

        nf = []
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        f = nf
    vv = np.array(verts) * radius + np.asarray(center, np.float64)
    return vv.astype(np.float32), np.array(f, np.int32)


def nested_shells(R: float = 1.0, level: int = 4):
    """Outer sphere of radius R, then an inner one of radius R/2 (its ids follow the outer's)."""
    vo, fo = icosphere(R, level)
    vi, fi = icosphere(R / 2, level)
    return np.concatenate([vo, vi]), np.concatenate([fo, fi + len(vo)]), len(fo)


def cube(half: float = 1.0):
    """The 12-triangle cube, 8 shared vertices."""
    h = half
    v = np.array([[x, y, z] for z in (-h, h) for y in (-h, h) for x in (-h, h)], np.float32)
    quads = [(0, 2, 3, 1), (4, 5, 7, 6), (0, 1, 5, 4), (2, 6, 7, 3), (0, 4, 6, 2), (1, 3, 7, 5)]
    f = []
    for a, b, c, d in quads:
        f += [(a, b, c), (a, c, d)]
    return v, np.array(f, np.int32)


def soup(vertices: np.ndarray, faces: np.ndarray, seed: int = 0):
    """STL-style triangle soup: three fresh vertices per face (coincident copies), faces shuffled."""
    rng = np.random.default_rng(seed)
    f = faces[rng.permutation(len(faces))]
    return np.ascontiguousarray(vertices[f.reshape(-1)]), np.arange(3 * len(f), dtype=np.int32).reshape(-1, 3)


def select_and_clean(vertices: np.ndarray, faces3: np.ndarray, visible: np.ndarray, remove_visible: bool):
    """Faces with a selected vertex, then the corner walk of vtkCleanPolyData (float ==, so -0 == +0)."""
    sel = ~visible if remove_visible else visible
    keep = sel[faces3].any(axis=1)
    key_new = {}
    out_v, ids = [], []
    for t in np.flatnonzero(keep):
        row = []
        for k in faces3[t]:
            x, y, z = (float(c) for c in vertices[k])
            key = (x + 0.0, y + 0.0, z + 0.0)
            if key not in key_new:
                key_new[key] = len(out_v)
                out_v.append(vertices[k])
            row.append(key_new[key])
        ids.append(row)
    ov = np.array(out_v, np.float32).reshape(-1, 3)
    of = np.array([r for r in ids if len(set(r)) == 3], np.int32).reshape(-1, 3)
    return ov, of
