"""The geodesic checker (oracle/geodesic.c) against independent references that rest on no reading of VTK: SciPy's
Dijkstra for the distances and predecessors, a NumPy brute force for the closest points and a Python loop written
like measures.py:1246-1249 for the lengths. CPU only."""
import math

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import dijkstra

from connectivity_meshes import shuffled_spheres, strip
from normals_model import small_meshes
from oracle import geodesic as og
from smoothing_meshes import grid_patch, with_degenerate, with_unused


def half_grid(n: int = 40, seed: int = 0):
    """A grid with some points moved by half a step: many equal path lengths, hence ambiguous points."""
    rng = np.random.default_rng(seed)
    ys, xs = np.mgrid[0:n, 0:n]
    v = np.stack([xs.ravel(), ys.ravel(), np.zeros(n * n)], 1).astype(np.float32)
    v[:, :2] += np.float32(0.5) * (rng.random((n * n, 2)) < 0.3)
    f = []
    for j in range(n - 1):
        for i in range(n - 1):
            a, b, c, d = j * n + i, j * n + i + 1, (j + 1) * n + i, (j + 1) * n + i + 1
            f += [(a, b, d), (a, d, c)] if (i + j) % 2 else [(a, b, c), (b, d, c)]
    return v, np.array(f, np.int32)


def meshes():
    out = {f"small_{k}": g for k, g in small_meshes().items()}
    out.update({
        "grid_patch": lambda: grid_patch(12, 9, 1),
        "grid_patch_degenerate": lambda: with_degenerate(*grid_patch(12, 9, 2), seed=3),
        "grid_patch_unused": lambda: with_unused(*grid_patch(12, 9, 4), seed=5),
        "half_grid": half_grid,
        "shuffled_spheres": lambda: shuffled_spheres(5, 2),
    })
    return out


def scipy_graph(v, f):
    """The undirected edge graph with weights sqrt((dx dx + dy dy) + dz dz) in double, explicit zeros kept."""
    p = np.asarray(v, np.float64)
    f = np.asarray(f, np.int64)[:, -3:]
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    e = np.unique(np.sort(e[e[:, 0] != e[:, 1]], 1), axis=0)
    d = p[e[:, 0]] - p[e[:, 1]]
    w = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
    rows, cols, data = np.r_[e[:, 0], e[:, 1]], np.r_[e[:, 1], e[:, 0]], np.r_[w, w]
    order = np.lexsort((cols, rows))
    indptr = np.searchsorted(rows[order], np.arange(len(p) + 1))
    return sp.csr_matrix((data[order], cols[order], indptr), shape=(len(p), len(p)))


def _starts(nv, seed=0):
    return sorted({0, nv - 1, *np.random.default_rng(seed).integers(0, nv, 3).tolist()})


@pytest.mark.parametrize("name", list(meshes()))
def test_distances_and_predecessors_equal_scipy(name):
    v, f = meshes()[name]()
    g = scipy_graph(v, f)
    for s in _starts(len(v)):
        got = og.distances(v, f, s)
        want, pred = dijkstra(g, indices=s, return_predecessors=True)
        assert np.array_equal(got["dist"].view(np.uint64), want.view(np.uint64))
        pred = np.where(pred < 0, -1, pred)
        plain = ~got["amb"]
        assert np.array_equal(got["pre"][plain], pred[plain])
        assert np.array_equal(got["rule"][plain], pred[plain])
        assert got["pre"][s] == -1 and (got["pre"][np.isinf(got["dist"])] == -1).all()


def test_half_grid_has_ambiguous_points():
    v, f = half_grid()
    g = og.distances(v, f, 0)
    assert g["amb"].sum() > 0
    # on an ambiguous point the heap's pick still attains d[v] with the smallest d[u]
    p = v.astype(np.float64)
    for x in np.flatnonzero(g["amb"]):
        u, r = g["pre"][x], g["rule"][x]
        w = math.sqrt(sum((p[u, k] - p[x, k]) * (p[u, k] - p[x, k]) for k in range(3)))
        assert g["dist"][u] + w == g["dist"][x] and g["dist"][u] == g["dist"][r] and r <= u


@pytest.mark.parametrize("name", ["small_icosphere", "grid_patch_unused", "shuffled_spheres", "half_grid"])
def test_closest_points_equal_brute_force(name):
    v, f = meshes()[name]()
    rng = np.random.default_rng(1)
    picks = np.concatenate([rng.random((20, 3)) * 10 - 2, v[rng.integers(0, len(v), 5)].astype(np.float64)])
    p = v.astype(np.float64)
    want = []
    for q in picks:
        d = q - p
        d2 = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]
        want.append(int(np.flatnonzero(d2 == d2.min())[0]))
    assert og.closest_points(v, picks).tolist() == want


def _length_like_measures(segments):
    total_length = 0.0
    for pts in segments:
        for j in range(len(pts) - 1):
            pt1, pt2 = [float(x) for x in pts[j]], [float(x) for x in pts[j + 1]]
            d2 = (pt1[0] - pt2[0]) ** 2 + (pt1[1] - pt2[1]) ** 2 + (pt1[2] - pt2[2]) ** 2
            total_length += math.sqrt(d2)
    return total_length


@pytest.mark.parametrize("name", ["grid_patch", "half_grid", "shuffled_spheres", "small_strip"])
@pytest.mark.parametrize("npicks", [2, 3, 10])
def test_path_lengths_equal_measures_loop(name, npicks):
    v, f = meshes()[name]()
    picks = v[np.random.default_rng(npicks).integers(0, len(v), npicks)].astype(np.float64) + 0.01
    r = og.geodesic_path(v, f, picks)
    bounds = np.cumsum([0] + [len(i) for i in r["ids"]])
    segs = [r["points"][a:b] for a, b in zip(bounds[:-1], bounds[1:])]
    assert r["total"] == _length_like_measures(segs)
    assert [og.path_length(s)[0] for s in segs] == list(r["lengths"])
    for ids, s in zip(r["ids"], segs):
        assert np.array_equal(s, v[ids])
    assert len(r["ids"]) == npicks - 1


def test_start_equals_end_and_unreached_end():
    v, f = shuffled_spheres(3, 0)
    g = og.distances(v, f, 0)
    assert og.trace(g["pre"], 0, 0).tolist() == [0]
    far = int(np.flatnonzero(np.isinf(g["dist"]))[0])
    assert og.trace(g["pre"], 0, far).tolist() == [far]
    r = og.geodesic_path(v, f, np.stack([v[0], v[0], v[far]]).astype(np.float64))
    assert [i.tolist() for i in r["ids"]] == [[0], [far]]
    assert r["total"] == 0.0 and r["unreached"].tolist() == [False, True]


def test_no_path_without_cells_or_two_picks():
    v, f = grid_patch(4, 4)
    assert og.geodesic_path(v, f[:0], v[:2])["total"] == 0.0
    r = og.geodesic_path(v, f, v[:1])
    assert r["ids"] == [] and len(r["points"]) == 0


def test_long_strip_path():
    v, f = strip(2000)
    last = int(f.max())                                   # the strip's last points are unused
    r = og.geodesic_path(v, f, np.array([v[0], v[last]], np.float64))
    assert len(r["ids"][0]) > 500 and r["ids"][0][0] == last and r["ids"][0][-1] == 0
