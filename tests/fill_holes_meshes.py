"""Meshes for the hole-filling tests, and a plain-Python restatement of vtkFillHolesFilter (written
independently of oracle/fill_holes.c, from the contract in its header) to check the checker."""
from __future__ import annotations

import math

import numpy as np

from visibility_meshes import cube, icosphere

FILLED, FAILED, TOO_LARGE = 0, 1, 2


def _sub(a, b):
    return [a[0] - b[0], a[1] - b[1], a[2] - b[2]]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _norm(v):
    return math.sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2])


def _unit(v):
    n = _norm(v)
    return [x / n for x in v] if n != 0.0 else v


def bounding_radius(pts):
    """vtkSphere::ComputeBoundingSphere with hints {0, 0}, as the contract states it."""
    c, r = list(pts[0]), 0.0
    for p in pts:
        v = _sub(p, c)
        d2 = (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]
        if d2 > r * r:
            d = math.sqrt(d2)
            r = (r + d) / 2.0
            delta = d - r
            c = [(r * c[k] + delta * p[k]) / d for k in range(3)]
    return r


def ear_clip(P, poly):
    """The contract's greedy triangulation: the triangles (point ids), or None when the loop fails."""
    n = len(poly)
    if n < 3:
        return None
    x = [P[p] for p in poly]
    N = [0.0, 0.0, 0.0]
    for i in range(1, n - 1):
        c = _cross(_sub(x[i], x[0]), _sub(x[i + 1], x[0]))
        N = [N[k] + c[k] for k in range(3)]
    N = _unit(N)
    rem = list(range(n))
    out = []
    while len(rem) > 3:
        best, bkey = None, math.inf
        for j, i in enumerate(rem):
            a, b, c = rem[j - 1], i, rem[(j + 1) % len(rem)]
            e = _unit(_cross(_sub(x[c], x[b]), _sub(x[a], x[b])))
            if not ((e[0] * N[0] + e[1] * N[1]) + e[2] * N[2] > 0.0):
                continue
            key = (_norm(_sub(x[b], x[a])) + _norm(_sub(x[c], x[b]))) + _norm(_sub(x[a], x[c]))
            if key < bkey:
                best, bkey = j, key
        if best is None:
            return None
        out.append((poly[rem[best - 1]], poly[rem[best]], poly[rem[(best + 1) % len(rem)]]))
        del rem[best]
    out.append(tuple(poly[i] for i in rem))
    return out


def fill_holes_py(vertices, faces, hole_size=1.0):
    """(faces int64 [T+N,3], lines, [(first_line, npts, radius, status)]) by the contract."""
    P = [tuple(float(c) for c in p) for p in np.asarray(vertices, np.float32)]
    f = [tuple(int(x) for x in row) for row in np.asarray(faces).reshape(-1, 3)]
    links = [[] for _ in P]
    for c, tri in enumerate(f):
        for p in tri:
            links[p].append(c)
    lines = []
    for c, tri in enumerate(f):
        for i in range(3):
            p1, p2 = tri[i], tri[(i + 1) % 3]
            if not any(d != c and p2 in f[d] for d in links[p1]):
                lines.append((p1, p2))
    out = [list(t) for t in f]
    if len(lines) < 3:
        return np.array(out, np.int64).reshape(-1, 3), len(lines), []
    llinks = [[] for _ in P]
    for k, (a, b) in enumerate(lines):
        llinks[a].append(k)
        llinks[b].append(k)
    visited = [False] * len(lines)
    loops = []
    for L in range(len(lines)):
        if visited[L]:
            continue
        visited[L] = True
        start, end, cur = lines[L][0], lines[L][1], L
        poly, valid = [start], True
        while end != start and valid:
            poly.append(end)
            others = [m for m in llinks[end] if m != cur]
            if len(others) != 1:
                valid = False
                continue
            n = others[0]
            visited[n] = True
            end = lines[n][1] if lines[n][0] == end else lines[n][0]
            cur = n
        if not valid:
            continue
        r = bounding_radius([P[p] for p in poly])
        if r <= hole_size:
            tris = ear_clip(P, poly)
            status = FAILED if tris is None else FILLED
            out += [list(t) for t in tris or []]
        else:
            status = TOO_LARGE
        loops.append((L, len(poly), r, status))
    return np.array(out, np.int64).reshape(-1, 3), len(lines), loops


# ---- meshes ------------------------------------------------------------------------------------------------
def without(v, f, drop):
    """f without the faces `drop`."""
    keep = np.ones(len(f), bool)
    keep[list(drop)] = False
    return v, np.ascontiguousarray(f[keep])


def icosphere_minus_one(level=2):
    v, f = icosphere(1.0, level)
    return without(v, f, [len(f) // 3])


def cube_minus_quad():
    v, f = cube(1.0)
    return without(v, f, [0, 1])


def random_deletion(v, f, frac, seed):
    """f with a random fraction of its faces deleted and the rest shuffled: many bow-tie points."""
    rng = np.random.default_rng(seed)
    keep = rng.random(len(f)) >= frac
    g = f[keep]
    return v, np.ascontiguousarray(g[rng.permutation(len(g))])


def bowtie(order=None):
    """A flat 5 x 5 grid with two interior triangles removed that meet at one point only (id 12): two
    triangular holes share that point. The triangle (1, 7, 6) next to the first hole is flipped, so one of
    that hole's lines runs against the other two and whether it is traced as a loop depends on the line ids.
    `order` permutes the remaining faces."""
    n = 5
    y, x = np.mgrid[0:n, 0:n]
    v = np.stack([x, y, np.zeros_like(x)], -1).reshape(-1, 3).astype(np.float32)
    f = []
    for j in range(n - 1):
        for i in range(n - 1):
            a = j * n + i
            f += [(a, a + 1, a + n + 1), (a, a + n + 1, a + n)]
    f = [(1, 6, 7) if t == (1, 7, 6) else t for t in f if t not in [(6, 7, 12), (12, 18, 17)]]
    f = np.array(f, np.int32)
    return v, np.ascontiguousarray(f[np.asarray(order)]) if order is not None else f


def collinear_loop():
    """Two triangles with all four points on one line: one boundary loop whose polygon normal is zero, so
    no ear qualifies."""
    v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [3, 0, 0]], np.float32)
    return v, np.array([(0, 1, 2), (0, 2, 3)], np.int32)


def closed_plus_sliver():
    """A closed icosphere plus the degenerate triangle (p, p, q) over two points that share no edge: exactly
    two boundary lines."""
    v, f = icosphere(1.0, 1)
    q = next(int(x) for x in range(len(v)) if not ((f == 0).any(1) & (f == x).any(1)).any() and x != 0)
    return v, np.concatenate([f, np.array([(0, 0, q)], np.int32)])


def open_tube(n_around: int, n_along: int = 3, radius: float = 1.0):
    """An open cylinder: two boundary loops of n_around points each, at z = 0 and z = n_along - 1."""
    a = np.arange(n_around) * (2 * np.pi / n_around)
    rings = [np.stack([radius * np.cos(a), radius * np.sin(a), np.full(n_around, float(z))], -1)
             for z in range(n_along)]
    v = np.concatenate(rings).astype(np.float32)
    f = []
    for z in range(n_along - 1):
        for i in range(n_around):
            a0, a1 = z * n_around + i, z * n_around + (i + 1) % n_around
            b0, b1 = a0 + n_around, a1 + n_around
            f += [(a0, a1, b1), (a0, b1, b0)]
    return v, np.array(f, np.int32)
