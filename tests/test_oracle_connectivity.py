"""The connectivity checker (oracle/connectivity.c) against an independent plain-Python TraverseAndMark,
against scipy's connected components, and against closed forms. CPU only."""
import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

from connectivity_meshes import dense_random, fan, shuffled_spheres, strip, traverse_py
from oracle import connectivity as oc


def _meshes():
    yield "dense", *dense_random(400, 12, 1)
    yield "dense_many", *dense_random(3000, 2000, 2)
    yield "spheres", *shuffled_spheres(9, 3)
    yield "fan", *fan(5000)
    yield "strip", *strip(301)


@pytest.mark.parametrize("name,v,f", list(_meshes()), ids=lambda x: x if isinstance(x, str) else "")
def test_checker_equals_python_restatement(name, v, f):
    st = oc.traverse(len(v), f)
    region, pmap, sizes = traverse_py(len(v), f)
    assert np.array_equal(st["region"], region)
    assert np.array_equal(st["point_map"], pmap)
    assert np.array_equal(st["sizes"], sizes)
    rng = np.random.default_rng(len(f))
    seeds = list(rng.integers(-2, len(v), 5))
    st = oc.traverse(len(v), f, seeds)
    region, pmap, sizes = traverse_py(len(v), f, seeds)
    assert np.array_equal(st["region"], region) and np.array_equal(st["point_map"], pmap)
    assert np.array_equal(st["sizes"], sizes)


@pytest.mark.parametrize("name,v,f", list(_meshes()), ids=lambda x: x if isinstance(x, str) else "")
def test_partition_equals_scipy(name, v, f):
    st = oc.traverse(len(v), f)
    nt, nv = len(f), len(v)
    # cells and points as one graph: cell t is node t, point p is node nt + p
    rows = np.repeat(np.arange(nt), 3)
    g = sp.coo_matrix((np.ones(3 * nt), (rows, nt + f.reshape(-1))), shape=(nt + nv, nt + nv))
    _, lab = connected_components(g, directed=False)
    cell_lab = lab[:nt]
    # regions ordered by their lowest cell id
    first = {}
    for t, l in enumerate(cell_lab):
        first.setdefault(l, len(first))
    want = np.array([first[l] for l in cell_lab], np.int32)
    assert np.array_equal(st["region"], want)
    assert np.array_equal(st["sizes"], np.bincount(want))
    used = np.zeros(nv, bool)
    used[f.reshape(-1)] = True
    assert np.array_equal(st["point_map"] >= 0, used)
    assert sorted(st["point_map"][used]) == list(range(used.sum()))


def test_strip_seeded_at_one_end_numbers_points_in_order():
    v, f = strip(1001)
    st = oc.traverse(len(v), f, [0])
    assert (st["region"] == 0).all()
    assert np.array_equal(st["point_map"][:1003], np.arange(1003))
    assert st["depth"] > 300
    st = oc.traverse(len(v), f)
    assert np.array_equal(st["point_map"][:1003], np.arange(1003))


def test_largest_ties_go_to_lowest_region():
    a, fa = strip(10)
    b, fb = strip(10)
    c, fc = strip(4)
    v = np.concatenate([c, a, b])
    f = np.concatenate([fc, fa + len(c), fb + len(c) + len(a)])
    st = oc.traverse(len(v), f)
    assert list(st["sizes"]) == [4, 10, 10]
    vo, fo, pids, cids = oc.select_largest_part(v, f)
    assert np.array_equal(cids, np.arange(4, 14))
    assert len(vo) == len(pids) == len(np.unique(f))         # the VTK form keeps every used point
    assert np.array_equal(vo[fo], v[f[4:14]])


@pytest.mark.parametrize("name,v,f", list(_meshes()), ids=lambda x: x if isinstance(x, str) else "")
def test_compact_form_is_vtk_form_minus_offset(name, v, f):
    parts = oc.split_disconnected_parts(v, f)
    compact = oc.split_disconnected_parts(v, f, compact=True)
    st = oc.traverse(len(v), f)
    assert len(parts) == len(compact) == len(st["sizes"])
    off = 0
    for (vv, fv, pv, cv), (vc, fc, pc, cc) in zip(parts, compact):
        assert np.array_equal(cv, cc) and np.array_equal(fv - off, fc)
        assert np.array_equal(vv[off:off + len(vc)], vc) and np.array_equal(pv[off:off + len(pc)], pc)
        assert np.array_equal(vc[fc], v[f[cc]])                # the geometry of the input faces
        off += len(vc)
    assert off == st["points"]
    assert np.array_equal(np.sort(np.concatenate([p[3] for p in parts])), np.arange(len(f)))


def test_seeds():
    v, f = shuffled_spheres(6, 7)
    st = oc.traverse(len(v), f)
    # a seed on each of two regions, a negative id and a duplicate
    p0, p1 = f[np.nonzero(st["region"] == 1)[0][0], 0], f[np.nonzero(st["region"] == 4)[0][0], 2]
    vo, fo, pids, cids = oc.join_seeds_parts(v, f, [-1, p1, p0, p1, -7])
    assert np.array_equal(cids, np.nonzero((st["region"] == 1) | (st["region"] == 4))[0])
    assert np.array_equal(vo[fo], v[f[cids]]) and np.array_equal(vo, v[pids])
    region, pmap, _ = traverse_py(len(v), f, [-1, p1, p0, p1, -7])
    assert np.array_equal(oc.traverse(len(v), f, [-1, p1, p0, p1, -7])["point_map"], pmap)
    # the first seed's lowest cell is marked first: its corner 0 is point 0
    c = np.nonzero((f == p1).any(axis=1))[0][0]
    assert pmap[f[c, 0]] == 0 and pmap[p1] <= 2
    # a seed on an unused point, or no seed at all, reaches nothing: an empty mesh
    unused = np.setdiff1d(np.arange(len(v)), f.reshape(-1))[0]
    for seeds in ([unused], [], [-3]):
        vo, fo, pids, cids = oc.join_seeds_parts(v, f, seeds)
        assert vo.shape == (0, 3) and fo.shape == (0, 3) and len(pids) == len(cids) == 0
    with pytest.raises(ValueError):
        oc.join_seeds_parts(v, f, [len(v)])


def test_empty_and_bad_faces():
    v = np.zeros((4, 3), np.float32)
    assert oc.split_disconnected_parts(v, np.zeros((0, 3), np.int32)) == []
    vo, fo, _, _ = oc.select_largest_part(v, np.zeros((0, 3), np.int64))
    assert vo.shape == (0, 3) and fo.shape == (0, 3)
    with pytest.raises(ValueError):
        oc.traverse(4, np.array([[0, 1, 4]], np.int32))
