"""The clean and triangle filter's C checker (oracle/clean.c) against an independent restatement in this file:
a dict keyed by coordinates for the merge, plain lists for the cells. Also: strips built from a known triangle
list decompose back to those triangles, winding included, without the checker."""
import math
import sys

import numpy as np
import pytest

from oracle import clean as oc


# ---- the restatement -------------------------------------------------------------------------------------------
def _key(P, p):
    x = tuple(float(c) + 0.0 for c in P[p])          # -0.0 + 0.0 == +0.0
    return ("nan", p) if any(c != c for c in x) else x


def model_clean(P, polys, strips):
    po, pc = oc.cell_array(polys)
    so, sc = oc.cell_array(strips)
    cells = [(False, list(pc[po[i]:po[i + 1]])) for i in range(len(po) - 1)]
    cells += [(True, list(sc[so[i]:so[i + 1]])) for i in range(len(so) - 1)]
    ids, first = {}, []
    out = {1: [], 2: [], 3: [], 4: []}
    for g, (strip, pts) in enumerate(cells):
        kept = []
        for p in pts:
            k = _key(P, p)
            if k not in ids:
                ids[k] = len(first)
                first.append(p)
            if not kept or kept[-1] != ids[k]:
                kept.append(ids[k])
        if not strip and len(kept) > 2 and kept[0] == kept[-1]:
            kept.pop()
        n = len(kept)
        cat = (4 if n >= 4 else n) if strip else (3 if n >= 3 else n)
        if cat:
            out[cat].append((g, kept))

    def pair(cs):
        offs = np.cumsum([0] + [len(k) for _, k in cs]).astype(np.int64)
        return offs, np.array([i for _, k in cs for i in k], np.int64)

    first = np.array(first, np.int64)
    return {"points": P[first].reshape(-1, 3), "point_ids": first, "verts": pair(out[1]), "lines": pair(out[2]),
            "polys": pair(out[3]), "strips": pair(out[4]),
            "cell_ids": np.array([g for c in (1, 2, 3, 4) for g, _ in out[c]], np.int64)}


def _sub(a, b):
    return [a[0] - b[0], a[1] - b[1], a[2] - b[2]]


def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _unit(a):
    d = math.sqrt(_dot(a, a))
    return ([c / d for c in a] if d != 0.0 else a), d


def model_ear_cut(P, ids):
    """vtkPolygon::EarCutTriangulation as clean.c's rule 10 states it, on Python floats (IEEE doubles)."""
    n = len(ids)
    x = [[float(c) for c in P[i]] for i in ids]
    ext = [max(p[k] for p in x) - min(p[k] for p in x) for k in range(3)]
    tol = 1e-6 * math.sqrt(_dot(ext, ext))
    nxt, prv = [(i + 1) % n for i in range(n)], [(i - 1) % n for i in range(n)]
    head, m, v = 0, n, 0
    for _ in range(n):
        w = nxt[v]
        d = _sub(x[v], x[w])
        if _dot(d, d) < tol * tol:
            prv[nxt[w]], nxt[v] = v, nxt[w]
            head = v if w == head else head
            m -= 1
        else:
            v = w
    N = [0.0, 0.0, 0.0]
    v = nxt[head]
    while nxt[v] != head:
        c = _cross(_sub(x[v], x[head]), _sub(x[nxt[v]], x[head]))
        N = [N[k] + c[k] for k in range(3)]
        v = nxt[v]
    N, d = _unit(N)
    if d == 0.0:
        return []

    def measure(v):
        v1, v2, v3 = _sub(x[v], x[prv[v]]), _sub(x[nxt[v]], x[v]), _sub(x[prv[v]], x[nxt[v]])
        area = _dot(_cross(v1, v2), N)
        if area < 0.0:
            return -1.0
        if area == 0.0:
            return -sys.float_info.max
        p = (math.sqrt(_dot(v1, v1)) + math.sqrt(_dot(v2, v2))) + math.sqrt(_dot(v3, v3))
        return p * p / area

    def side(sN, o, q):
        e = (sN[0] * (q[0] - o[0]) + sN[1] * (q[1] - o[1])) + sN[2] * (q[2] - o[2])
        return 1 if e > tol else (-1 if e < -tol else 0)

    def meet(a1, a2, b1, b2):
        a, b, c = _sub(a2, a1), _sub(b2, b1), _sub(b1, a1)
        r00, r01, r11, c0, c1 = _dot(a, a), -_dot(a, b), _dot(b, b), _dot(a, c), -_dot(b, c)
        det = r00 * r11 - r01 * r01
        if det == 0.0:
            return True
        u, w = (r11 * c0 - r01 * c1) / det, (-r01 * c0 + r00 * c1) / det
        return 0.0 <= u <= 1.0 and 0.0 <= w <= 1.0

    def removable(v):
        if m <= 3:
            return True
        pv, nx = prv[v], nxt[v]
        sN, d = _unit(_cross(_sub(x[nx], x[pv]), N))
        if d == 0.0:
            return False
        signs = []
        w = nxt[nx]
        while w != pv:
            signs.append((w, side(sN, x[pv], x[w])))
            w = nxt[w]
        for (w0, s0), (w1, s1) in zip(signs, signs[1:]):
            if s1 != s0 and meet(x[pv], x[nx], x[w1], x[w0]):
                return False
        return any(sg < 0 for _, sg in signs)

    queue, v = {}, head
    for _ in range(m):
        k = measure(v)
        if k > 0.0:
            queue[v] = k
        v = nxt[v]
    out = []
    while m > 2 and queue:
        best = min(queue, key=lambda i: (queue[i], i))
        convex = len(queue) == m
        del queue[best]
        if not convex and not removable(best):
            continue
        pv, nx = prv[best], nxt[best]
        out.append([ids[best], ids[nx], ids[pv]])
        m -= 1
        if m < 3:
            break
        head = nx if best == head else head
        nxt[pv], prv[nx] = nx, pv
        for u in (pv, nx):
            queue.pop(u, None)
            k = measure(u)
            if k > 0.0:
                queue[u] = k
    return out


def model_triangles(P, polys, strips):
    po, pc = oc.cell_array(polys)
    so, sc = oc.cell_array(strips)
    tris, ids = [], []
    for i in range(len(po) - 1):
        if po[i + 1] - po[i] == 3:
            tris.append(pc[po[i]:po[i + 1]])
            ids.append(i)
        elif po[i + 1] - po[i] > 3:
            t = model_ear_cut(P, list(pc[po[i]:po[i + 1]]))
            tris += t
            ids += [i] * len(t)
    for i in range(len(so) - 1):
        s = sc[so[i]:so[i + 1]]
        for j in range(len(s) - 2):
            tris.append([s[j + 1], s[j], s[j + 2]] if j % 2 else [s[j], s[j + 1], s[j + 2]])
            ids.append(len(po) - 1 + i)
    return {"faces": np.array(tris, np.int64).reshape(-1, 3), "cell_ids": np.array(ids, np.int64)}


def assert_same(got, want):
    assert got.keys() == want.keys()
    for k in want:
        g, w = got[k], want[k]
        if isinstance(w, tuple):
            for a, b in zip(g, w):
                assert np.array_equal(a, b), k
        elif w.dtype == np.float32:
            assert np.array_equal(g.view(np.uint32), w.view(np.uint32)), k
        else:
            assert np.array_equal(g, w), k


# ---- meshes ----------------------------------------------------------------------------------------------------
def grid_points(n, seed=0):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 4, size=(n, 3)).astype(np.float32)   # many exact coincidences


CASES = {
    "coincident": (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 0, 0], [0, 0, 0], [0, 0, 1]], np.float32),
                   np.array([[0, 1, 2], [3, 4, 5], [2, 1, 5]]), None),
    "signed_zero": (np.array([[0, 0, 0], [-0.0, 0, -0.0], [1, 0, 0], [0, 1, 0]], np.float32),
                    np.array([[0, 2, 3], [1, 3, 2]]), None),
    "nan": (np.array([[np.nan, 0, 0], [np.nan, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32),
            np.array([[0, 2, 3], [1, 2, 3], [0, 3, 2]]), None),
    "collapse": (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 0]], np.float32),
                 np.array([[0, 1, 0], [0, 0, 1], [1, 1, 1], [0, 3, 1], [0, 1, 2], [2, 3, 0]]), None),
    "unused": (np.array([[9, 9, 9], [0, 0, 0], [1, 0, 0], [7, 7, 7], [0, 1, 0]], np.float32),
               np.array([[4, 2, 1]]), None),
    "empty": (np.zeros((3, 3), np.float32), np.zeros((0, 3), np.int64), None),
}


def _strip_pairs():
    P = grid_points(40, 3)
    strips = [[0, 1, 2, 3], [4, 5, 6], [7, 8], [9], [10, 10, 11, 11, 12], [13, 14, 13, 14, 15],
              [16, 17, 18, 19, 20], [], [21, 22, 23, 24, 25, 26, 27]]
    offs = np.cumsum([0] + [len(s) for s in strips]).astype(np.int64)
    conn = np.array([i for s in strips for i in s], np.int64)
    polys = [[0, 1, 2, 3], [5, 5], [6], [], [30, 31, 32, 33, 30], [34, 35, 34]]
    po = np.cumsum([0] + [len(s) for s in polys]).astype(np.int64)
    pc = np.array([i for s in polys for i in s], np.int64)
    return P, (po, pc), (offs, conn)


@pytest.mark.parametrize("name", sorted(CASES))
def test_clean_cases(name):
    P, polys, strips = CASES[name]
    assert_same(oc.clean_polydata(P, polys, strips), model_clean(P, polys, strips))


def test_clean_mixed_cells_and_strips():
    P, polys, strips = _strip_pairs()
    got = oc.clean_polydata(P, polys, strips)
    assert_same(got, model_clean(P, polys, strips))
    assert len(got["cell_ids"]) > 0 and len(got["verts"][1]) and len(got["lines"][1]) and len(got["strips"][1])


@pytest.mark.parametrize("seed", range(4))
def test_clean_random(seed):
    rng = np.random.default_rng(seed)
    P = grid_points(300, seed)
    P[rng.integers(0, 300, 10)] = np.float32(np.nan)
    P[rng.integers(0, 300, 10), 0] = np.float32(-0.0)
    f = rng.integers(0, 300, size=(800, 3))
    sizes = rng.integers(0, 9, 200)
    so = np.cumsum(np.r_[0, sizes]).astype(np.int64)
    sc = rng.integers(0, 300, so[-1])
    assert_same(oc.clean_polydata(P, f, (so, sc)), model_clean(P, f, (so, sc)))


@pytest.mark.parametrize("dtype", [np.int32, np.int64])
def test_clean_forms_agree(dtype):
    P = grid_points(100, 7)
    f = np.random.default_rng(7).integers(0, 100, size=(200, 3)).astype(dtype)
    f4 = np.concatenate([np.full((200, 1), 3, dtype), f], 1)
    pair = (np.arange(0, 601, 3), f.reshape(-1))
    want = oc.clean_polydata(P, f)
    for form in (f4, pair):
        assert_same(oc.clean_polydata(P, form), want)


def test_malformed():
    P = grid_points(10)
    for offs, conn in (([1, 3], [0, 1, 2]), ([0, 2, 1, 3], [0, 1, 2]), ([0, 3], [0, 1, 2, 3])):
        with pytest.raises(ValueError):
            oc.clean_polydata(P, (np.array(offs), np.array(conn)))
    with pytest.raises(ValueError):
        oc.clean_polydata(P, np.array([[0, 1, 10]]))
    with pytest.raises(ValueError):
        oc.triangle_filter(P, None, (np.array([0, 3]), np.array([0, -1, 2])))


def test_triangle_filter_model():
    P, polys, strips = _strip_pairs()
    assert_same(oc.triangle_filter(P, polys, strips), model_triangles(P, polys, strips))


def _frame(seed):
    """a random rotation and offset, so the polygons lie in general planes"""
    q, _ = np.linalg.qr(np.random.default_rng(seed).normal(size=(3, 3)))
    return q, np.random.default_rng(seed + 1).normal(size=3) * 10


def polygon(kind, n, seed=0):
    """(points float32 [n,3], ids): a convex or a concave planar polygon of n points in a rotated plane"""
    rng = np.random.default_rng(seed)
    t = np.sort(rng.uniform(0, 2 * np.pi, n)) if kind != "regular" else np.linspace(0, 2 * np.pi, n, endpoint=False)
    if kind in ("regular", "convex"):
        r = np.ones(n)
    elif kind == "star":
        r = np.where(np.arange(n) % 2 == 0, 1.0, 0.35)
    elif kind == "comb":                                  # deep notches: many non-convex vertices
        r = np.where(np.arange(n) % 4 < 2, 1.0, 0.15)
    else:                                                 # random radii: mildly concave
        r = rng.uniform(0.4, 1.0, n)
    xy = np.stack([r * np.cos(t), r * np.sin(t), np.zeros(n)], 1)
    if kind in ("star", "comb", "concave") and seed % 2:
        xy = xy[::-1].copy()                              # clockwise as well
    q, o = _frame(seed)
    return (xy @ q.T + o).astype(np.float32), np.arange(n)


POLY_KINDS = ["regular", "convex", "star", "comb", "concave"]
POLY_SIZES = [4, 5, 6, 7, 8, 12, 17, 32, 64]


@pytest.mark.parametrize("kind", POLY_KINDS)
@pytest.mark.parametrize("n", POLY_SIZES)
def test_ear_cut_polygons(kind, n):
    for seed in range(3):
        P, ids = polygon(kind, n, seed)
        pair = (np.array([0, n]), ids)
        got = oc.triangle_filter(P, pair)
        assert_same(got, model_triangles(P, pair, None))
        if kind in ("regular", "convex", "star"):
            assert len(got["faces"]) == n - 2
        # every emitted triangle turns the polygon's way
        x = P.astype(np.float64)
        N = sum(np.cross(x[i] - x[0], x[i + 1] - x[0]) for i in range(1, n - 1))
        for a, b, c in got["faces"]:
            assert np.dot(np.cross(x[a] - x[c], x[b] - x[a]), N) >= 0


def test_ear_cut_degenerate_polygons():
    P = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [3, 0, 0], [0, 0, 0], [1, 1, 0], [1, 1, 0], [0, 1, 0]],
                 np.float32)
    polys = (np.array([0, 4, 8, 12]), np.array([0, 1, 2, 3, 4, 1, 5, 6, 0, 1, 5, 7]))
    assert_same(oc.triangle_filter(P, polys), model_triangles(P, polys, None))


@pytest.mark.parametrize("n", [3, 4, 5, 12, 257])
def test_strip_decomposes_to_known_triangles(n):
    """A strip over points 0..n-1 is the triangle list t_i = (i, i+1, i+2) with every odd one flipped; built
    here from that list alone, it must decompose back to it."""
    tris = [(i, i + 1, i + 2) if i % 2 == 0 else (i + 1, i, i + 2) for i in range(n - 2)]
    strip = np.array([tris[0][0], tris[0][1]] + [t[2] for t in tris], np.int64)
    got = oc.triangle_filter(np.zeros((n, 3), np.float32), None, (np.array([0, len(strip)]), strip))
    assert np.array_equal(got["faces"], np.array(tris, np.int64))
    assert np.array_equal(got["cell_ids"], np.zeros(n - 2, np.int64))
    # consistent winding: every interior edge is crossed in opposite directions by its two triangles
    edges = {}
    for t in tris:
        for a, b in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
            edges[(a, b)] = edges.get((a, b), 0) + 1
    assert all(v == 1 for v in edges.values())
