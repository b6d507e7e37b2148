"""An independent NumPy restatement of the surface normals contract (oracle/normals.c's header): consistent
ordering, auto-orientation, cell normals, feature splitting, point normals, and vtkMassProperties. Written
from the contract's text with plain Python containers, it pins the C checker on small meshes so the checker
does not rest on one reading of VTK alone."""
from __future__ import annotations

import math

import numpy as np

from connectivity_meshes import dense_random, fan, strip
from smoothing_meshes import fin, folded_sheet, grid_patch, with_degenerate, with_unused
from visibility_meshes import icosphere

F32 = np.float32


def _links(nv, f):
    links = [[] for _ in range(nv)]
    for t, tri in enumerate(f):
        for p in tri:
            links[p].append(t)
    return links


def _edge_neighbors(links, f, c, p1, p2):
    return [d for d in links[p1] if d != c and p2 in f[d]]


def tri_normal(v, tri):
    v1, v2, v3 = ([float(x) for x in v[p]] for p in tri)
    a = [v3[k] - v2[k] for k in range(3)]
    b = [v1[k] - v2[k] for k in range(3)]
    n = [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]
    ln = math.sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2])
    return [x / ln for x in n] if ln != 0.0 else n


def _x_key(v, p):
    x = float(v[p][0])
    return (1, 0.0, p) if math.isnan(x) else (0, x, p)


def compute_normals(vertices, faces, feature_angle=30.0, auto_orient=False) -> dict:
    v = np.asarray(vertices, np.float32)
    f = [tuple(int(x) for x in t) for t in np.asarray(faces).reshape(-1, 3)]
    nv, nt = len(v), len(f)
    links = _links(nv, f)
    cur = [list(t) for t in f]
    visited = [False] * nt
    flips = regions = waves = 0

    def traverse(seed):
        nonlocal flips
        wave, n = [seed], 0
        while wave:
            n += 1
            nxt = []
            for c in wave:
                for j in range(3):
                    p1, p2 = cur[c][j], cur[c][(j + 1) % 3]
                    for d in _edge_neighbors(links, f, c, p1, p2):
                        if visited[d]:
                            continue
                        l = cur[d].index(p2)
                        if cur[d][(l + 1) % 3] != p1:
                            cur[d].reverse()
                            flips += 1
                        visited[d] = True
                        nxt.append(d)
            wave = nxt
        return n

    if auto_orient:
        seeds = sorted(range(nv), key=lambda p: _x_key(v, p))
    else:
        seeds = range(nt)
    for s in seeds:
        if auto_orient:
            best, cell = 0.0, None
            for d in links[s]:
                if not visited[d]:
                    nx = tri_normal(v, f[d])[0]
                    if abs(nx) > best:
                        best, cell = abs(nx), d
            if cell is None:
                continue
            if tri_normal(v, f[cell])[0] > 0:
                cur[cell].reverse()
                flips += 1
        else:
            if visited[s]:
                continue
            cell = s
        visited[cell] = True
        waves = max(waves, traverse(cell))
        regions += 1

    cn = np.array([tri_normal(v, t) for t in cur], np.float64).astype(F32).reshape(nt, 3)

    # splitting
    cos_angle = math.cos(min(max(float(feature_angle), 0.0), 180.0) * 0.017453292519943295)
    out = [list(t) for t in cur]
    src = list(range(nv))
    for p in range(nv):
        cells = links[p]
        if len(cells) <= 1:
            continue
        group = {}
        for c0 in cells:
            if c0 in group:
                continue
            g = len(set(group.values()))
            group[c0] = g
            t = f[c0]
            s = t.index(p)
            starts = {0: (t[1], t[2]), 1: (t[2], t[0]), 2: (t[1], t[0])}[s]
            for nei in starts:
                c = c0
                while True:
                    en = _edge_neighbors(links, f, c, p, nei)
                    if len(en) != 1 or en[0] in group:
                        break
                    d = en[0]
                    dot = sum(float(cn[c][k]) * float(cn[d][k]) for k in range(3))
                    if not dot > cos_angle:
                        break
                    group[d] = g
                    c = d
                    u = f[c]
                    su = u.index(p)
                    first, other = {0: (u[1], u[2]), 1: (u[2], u[0]), 2: (u[1], u[0])}[su]
                    nei = first if first != nei else other
        ng = len(set(group.values()))
        base = len(src)
        src += [p] * (ng - 1)
        for c in set(cells):
            if group[c] > 0:
                out[c] = [base + group[c] - 1 if q == p else q for q in out[c]]

    # point normals, float32 sums in cell order
    pn = np.zeros((len(src), 3), F32)
    for t in range(nt):
        for q in out[t]:
            for k in range(3):
                pn[q, k] = F32(pn[q, k] + cn[t, k])
    for q in range(len(src)):
        s = pn[q]
        den = F32(math.sqrt(F32(F32(F32(s[0] * s[0]) + F32(s[1] * s[1])) + F32(s[2] * s[2]))))
        if den != 0:
            pn[q] = [F32(x / den) for x in s]
    return {"points": v[np.array(src, np.int64)].reshape(-1, 3), "faces": np.array(out, np.int64).reshape(nt, 3),
            "point_normals": pn, "cell_normals": cn, "regions": regions, "flips": flips,
            "new_points": len(src) - nv, "waves": waves}


def mass_properties(vertices, faces):
    v = np.asarray(vertices, np.float32)
    f = np.asarray(faces).reshape(-1, 3)
    if len(f) == 0:
        return 0.0, 0.0
    w = {k: 0.0 for k in ("x", "y", "z", "xyz", "xy", "xz", "yz")}
    vol, area_sum = [0.0, 0.0, 0.0], 0.0
    for tri in f:
        x, y, z = ([float(v[p][k]) for p in tri] for k in range(3))
        i = [x[1] - x[0], x[2] - x[0], x[2] - x[1]]
        j = [y[1] - y[0], y[2] - y[0], y[2] - y[1]]
        k = [z[1] - z[0], z[2] - z[0], z[2] - z[1]]
        u = [j[0] * k[1] - k[0] * j[1], k[0] * i[1] - i[0] * k[1], i[0] * j[1] - j[0] * i[1]]
        ln = math.sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2])
        u = [c / ln for c in u] if ln != 0.0 else [0.0, 0.0, 0.0]
        a0, a1, a2 = (abs(c) for c in u)
        if a0 > a1 and a0 > a2:
            w["x"] += 1
        elif a1 > a0 and a1 > a2:
            w["y"] += 1
        elif a2 > a0 and a2 > a1:
            w["z"] += 1
        elif a0 == a1 == a2:
            w["xyz"] += 1
        elif a0 == a1 and a0 > a2:
            w["xy"] += 1
        elif a0 == a2 and a0 > a1:
            w["xz"] += 1
        elif a1 == a2 and a0 < a2:
            w["yz"] += 1
        a = math.sqrt(i[1] * i[1] + j[1] * j[1] + k[1] * k[1])
        b = math.sqrt(i[0] * i[0] + j[0] * j[0] + k[0] * k[0])
        c = math.sqrt(i[2] * i[2] + j[2] * j[2] + k[2] * k[2])
        s = 0.5 * (a + b + c)
        area = math.sqrt(abs(s * (s - a) * (s - b) * (s - c)))
        area_sum += area
        avg = [(x[0] + x[1] + x[2]) / 3.0, (y[0] + y[1] + y[2]) / 3.0, (z[0] + z[1] + z[2]) / 3.0]
        for q in (2, 1, 0):
            vol[q] += area * u[q] * avg[q]
    n = float(len(f))
    kx = (w["x"] + (w["xyz"] / 3.0) + ((w["xy"] + w["xz"]) / 2.0)) / n
    ky = (w["y"] + (w["xyz"] / 3.0) + ((w["xy"] + w["yz"]) / 2.0)) / n
    kz = (w["z"] + (w["xyz"] / 3.0) + ((w["xz"] + w["yz"]) / 2.0)) / n
    return abs(kx * vol[0] + ky * vol[1] + kz * vol[2]), area_sum


# ---- meshes ------------------------------------------------------------------------------------------------
def box(lo=(0.0, 0.0, 0.0), hi=(2.0, 3.0, 5.0)):
    """An axis-aligned box, twelve outward triangles over eight corners."""
    v = np.array([[hi[0] if b & 1 else lo[0], hi[1] if b & 2 else lo[1], hi[2] if b & 4 else lo[2]]
                  for b in range(8)], np.float32)
    quads = [(0, 2, 3, 1), (4, 5, 7, 6), (0, 1, 5, 4), (2, 6, 7, 3), (0, 4, 6, 2), (1, 3, 7, 5)]
    f = []
    for a, b, c, d in quads:
        f += [(a, b, c), (a, c, d)]
    return v, np.array(f, np.int32)


def mobius(n: int = 24):
    """A Möbius strip: a non-orientable band of 2n triangles."""
    v = []
    for i in range(n):
        t = 2 * np.pi * i / n
        for s in (-0.3, 0.3):
            r = 1.0 + s * np.cos(t / 2)
            v.append((r * np.cos(t), r * np.sin(t), s * np.sin(t / 2)))
    f = []
    for i in range(n):
        a, b = 2 * i, 2 * i + 1
        if i + 1 < n:
            c, d = a + 2, b + 2
        else:
            c, d = 1, 0                      # the half twist: the ends join crossed
        f += [(a, b, d), (a, d, c)]
    return np.array(v, np.float32), np.array(f, np.int32)


def three_on_an_edge():
    """Three triangles on the edge (0, 1), in mixed orders."""
    v = np.array([[0, 0, 0], [1, 0, 0], [0.5, 1, 0], [0.5, -1, 0.2], [0.5, 0.1, 1]], np.float32)
    return v, np.array([(0, 1, 2), (0, 1, 3), (1, 0, 4)], np.int32)


def randomly_flipped(v, f, seed):
    rng = np.random.default_rng(seed)
    f = f.copy()
    m = rng.random(len(f)) < 0.5
    f[m] = f[m][:, ::-1]
    return v, f


def small_meshes():
    """The small meshes both the checker and the device are pinned on, by name."""
    return {
        "box": box,
        "icosphere": lambda: randomly_flipped(*icosphere(1.0, 2), 1),
        "fan": lambda: fan(12),
        "grid": lambda: grid_patch(9, 7, 3, jitter=0.4),
        "fin": fin,
        "folded_sheet": folded_sheet,
        "mobius": mobius,
        "three_on_an_edge": three_on_an_edge,
        "degenerate": lambda: with_degenerate(*randomly_flipped(*grid_patch(8, 6, 4), 2), seed=5),
        "unused": lambda: with_unused(*randomly_flipped(*icosphere(1.0, 1), 3), seed=3),
        "strip": lambda: strip(41),
        "dense": lambda: dense_random(120, 30, 4),
    }
