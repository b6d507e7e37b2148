"""Meshes for the smoothing tests, and a plain-Python restatement of vtkSmoothPolyDataFilter (written
independently of oracle/smoothing.c, from the contract in its header) to check the checker."""
from __future__ import annotations

import math

import numpy as np

SIMPLE, FIXED, FEATURE, BOUNDARY = 0, 1, 2, 3

# the reference callers' settings
APPLY_SMOOTH = dict(iterations=20, relaxation_factor=0.4, feature_angle=80.0, feature_edge_smoothing=False,
                    boundary_smoothing=False)
DECIMATE = dict(iterations=15)
MARKER = dict(iterations=7, relaxation_factor=0.2, feature_edge_smoothing=False, boundary_smoothing=False)
FEATURES_ON = dict(iterations=10, relaxation_factor=0.3, feature_angle=30.0, feature_edge_smoothing=True)
SETTINGS = {"apply_smooth": APPLY_SMOOTH, "decimate": DECIMATE, "marker": MARKER, "features_on": FEATURES_ON}


def _cos(angle):
    return math.cos(min(max(float(angle), 0.0), 180.0) * (math.pi / 180.0))


def _normal(P, t):
    v1, v2, v3 = (tuple(float(x) for x in P[p]) for p in t)
    ax, ay, az = v3[0] - v2[0], v3[1] - v2[1], v3[2] - v2[2]
    bx, by, bz = v1[0] - v2[0], v1[1] - v2[1], v1[2] - v2[2]
    n = [ay * bz - az * by, az * bx - ax * bz, ax * by - ay * bx]
    ln = math.sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2])
    return [x / ln for x in n] if ln != 0.0 else n


def _unit(v):
    d = math.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
    return [x / d for x in v] if d != 0.0 else v


def smooth_py(vertices, faces, iterations=20, relaxation_factor=0.01, feature_angle=45.0, edge_angle=15.0,
              feature_edge_smoothing=False, boundary_smoothing=True, convergence=0.0):
    """(vertices float32 [V,3], types, lists, iterations done) by the contract."""
    P0 = np.asarray(vertices, np.float32)
    f = [tuple(int(x) for x in row) for row in np.asarray(faces).reshape(-1, 3)]
    nv = len(P0)
    links = [[] for _ in range(nv)]
    for c, tri in enumerate(f):
        for p in tri:
            links[p].append(c)
    cos_f, cos_e = _cos(feature_angle), _cos(edge_angle)
    typ = [SIMPLE] * nv
    lst = [[] for _ in range(nv)]

    def hit(p, e, other):
        if e != SIMPLE and typ[p] == SIMPLE:
            lst[p] = [other]
            typ[p] = e
        elif (e != SIMPLE and typ[p] in (BOUNDARY, FEATURE)) or (e == SIMPLE and typ[p] == SIMPLE):
            lst[p].append(other)
            if typ[p] != SIMPLE and len(lst[p]) > 2:
                typ[p] = FIXED

    for c, tri in enumerate(f):
        for i in range(3):
            p1, p2 = tri[i], tri[(i + 1) % 3]
            nei = [d for d in links[p1] if d != c and p2 in f[d]]
            if not nei:
                e = BOUNDARY
            elif len(nei) >= 2:
                e = SIMPLE if min(nei) < c else FEATURE
            elif nei[0] > c:
                e = SIMPLE
                if feature_edge_smoothing:
                    n, m = _normal(P0, tri), _normal(P0, f[nei[0]])
                    if n[0] * m[0] + n[1] * m[1] + n[2] * m[2] <= cos_f:
                        e = FEATURE
            else:
                continue
            hit(p1, e, p2)
            hit(p2, e, p1)

    for p in range(nv):
        if typ[p] not in (FEATURE, BOUNDARY):
            continue
        if not boundary_smoothing and typ[p] == BOUNDARY:
            typ[p] = FIXED
        elif len(lst[p]) != 2:
            typ[p] = FIXED
        else:
            a, x, b = (tuple(float(v) for v in P0[q]) for q in (lst[p][0], p, lst[p][1]))
            l1 = _unit([x[k] - a[k] for k in range(3)])
            l2 = _unit([b[k] - x[k] for k in range(3)])
            if l1[0] * l2[0] + l1[1] * l2[1] + l1[2] * l2[2] < cos_e:
                typ[p] = FIXED

    P = P0.copy()
    done = 0
    if f and iterations > 0 and relaxation_factor != 0.0:
        used = np.unique(np.asarray(f).reshape(-1))
        lo, hi = P0[used].astype(np.float64).min(0), P0[used].astype(np.float64).max(0)
        dx, dy, dz = (float(h - l) for h, l in zip(hi, lo))
        conv = min(max(float(convergence), 0.0), 1.0) * math.sqrt(dx * dx + dy * dy + dz * dz)
        max_dist = float("inf")
        while max_dist > conv and done < iterations:
            max_dist = 0.0
            for p in range(nv):
                n = len(lst[p])
                if typ[p] == FIXED or n == 0:
                    continue
                x = [float(v) for v in P[p]]
                d = [0.0, 0.0, 0.0]
                for j in lst[p]:
                    for k in range(3):
                        d[k] += (float(P[j, k]) - x[k]) / n
                y = [x[k] + relaxation_factor * d[k] for k in range(3)]
                dist = (x[0] - y[0]) * (x[0] - y[0]) + (x[1] - y[1]) * (x[1] - y[1]) + (x[2] - y[2]) * (x[2] - y[2])
                max_dist = max(max_dist, dist)
                P[p] = np.array(y, np.float64).astype(np.float32)
            max_dist = math.sqrt(max_dist)
            done += 1
    return P, np.array(typ, np.int8), [np.array(x, np.int32) for x in lst], done


# ---- meshes ------------------------------------------------------------------------------------------------
def grid_patch(n: int, m: int, seed: int = 0, jitter: float = 0.1):
    """An open n x m grid of points, two triangles a square, z jittered."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:m, 0:n]
    v = np.stack([x, y, rng.random((m, n)) * jitter], -1).reshape(-1, 3).astype(np.float32)
    f = []
    for j in range(m - 1):
        for i in range(n - 1):
            a = j * n + i
            f += [(a, a + 1, a + n + 1), (a, a + n + 1, a + n)]
    return v, np.array(f, np.int32)


def fin():
    """Three triangles on one edge (0, 1): a non-manifold fin, plus a fan around the edge's ends."""
    v = np.array([[0, 0, 0], [1, 0, 0], [0.5, 1, 0], [0.5, -1, 0], [0.5, 0, 1], [0.5, 0.3, -1], [1.5, 0.5, 0.2]],
                 np.float32)
    f = np.array([(0, 1, 2), (1, 0, 3), (0, 1, 4), (1, 0, 5), (1, 6, 2)], np.int32)
    return v, f


def with_degenerate(v, f, seed: int = 0):
    """f plus degenerate triangles (a repeated corner, and all three equal) on existing points."""
    rng = np.random.default_rng(seed)
    picks = rng.integers(0, len(v), 4)
    extra = [(picks[0], picks[0], picks[1]), (picks[2], picks[3], picks[3]), (picks[1], picks[1], picks[1])]
    return v, np.concatenate([f, np.array(extra, np.int32)])


def with_unused(v, f, seed: int = 0):
    """v with unused points spliced in: every face id is remapped."""
    rng = np.random.default_rng(seed)
    nv = len(v) + 9
    keep = np.sort(rng.choice(nv, len(v), replace=False))
    out = (rng.random((nv, 3)) * 50).astype(np.float32)
    out[keep] = v
    return out, keep[f].astype(np.int32)


def folded_sheet(n: int = 9):
    """A grid patch folded at 90 degrees along its middle column: a sharp feature line."""
    v, f = grid_patch(n, n, jitter=0.0)
    x = v[:, 0].copy()
    mid = (n - 1) / 2
    v[:, 2] = np.where(x > mid, x - mid, 0.0)
    v[:, 0] = np.minimum(x, mid)
    return v, f


def hexagon_fan(center=(0.1, -0.05, 0.3)):
    """A centre point (id 0) and a ring of six: only the centre is interior."""
    a = np.arange(6) * (np.pi / 3)
    v = np.zeros((7, 3), np.float32)
    v[0] = center
    v[1:, 0], v[1:, 1] = np.cos(a), np.sin(a)
    f = np.array([(0, 1 + i, 1 + (i + 1) % 6) for i in range(6)], np.int32)
    return v, f
