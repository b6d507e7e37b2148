"""The C checker of the Laplacian surface smoothing (oracle/smoothing.c) against an independent plain-Python
restatement of the contract (tests/smoothing_meshes.py), and against closed forms."""
import math

import numpy as np
import pytest

from connectivity_meshes import dense_random, fan, shuffled_spheres, strip
from oracle import smoothing as osm
from smoothing_meshes import (BOUNDARY, FEATURE, FIXED, SETTINGS, SIMPLE, fin, folded_sheet, grid_patch,
                              hexagon_fan, smooth_py, with_degenerate, with_unused)
from visibility_meshes import icosphere

MESHES = {
    "icosphere": lambda: icosphere(1.0, 2),
    "spheres": lambda: shuffled_spheres(3, 4),
    "dense": lambda: dense_random(120, 40, 3),
    "fan": lambda: fan(30),
    "strip": lambda: strip(41),
    "grid": lambda: grid_patch(7, 6, 1),
    "fin": fin,
    "degenerate": lambda: with_degenerate(*grid_patch(6, 5, 2), seed=5),
    "unused": lambda: with_unused(*icosphere(1.0, 1), seed=3),
    "folded": folded_sheet,
}


def _same(want, got):
    assert np.array_equal(want["vertices"].view(np.uint32), got[0].view(np.uint32))
    assert np.array_equal(want["types"], got[1])
    assert len(want["lists"]) == len(got[2])
    assert all(np.array_equal(a, b) for a, b in zip(want["lists"], got[2]))
    assert want["iterations"] == got[3]


@pytest.mark.parametrize("name", list(MESHES))
@pytest.mark.parametrize("setting", list(SETTINGS))
def test_checker_matches_restatement(name, setting):
    v, f = MESHES[name]()
    kw = SETTINGS[setting]
    _same(osm.smooth(v, f, **kw), smooth_py(v, f, **kw))


@pytest.mark.parametrize("name", ["icosphere", "grid", "folded", "unused"])
def test_checker_matches_restatement_with_convergence(name):
    v, f = MESHES[name]()
    done = []
    for conv in (1e-3, 1e-2):
        want = osm.smooth(v, f, iterations=200, relaxation_factor=0.3, convergence=conv)
        _same(want, smooth_py(v, f, iterations=200, relaxation_factor=0.3, convergence=conv))
        done.append(want["iterations"])
    assert 1 <= done[1] < 200 and done[1] <= done[0]


def test_nothing_to_do_keeps_the_bits():
    v, f = icosphere(1.0, 2)
    for kw in (dict(iterations=0), dict(relaxation_factor=0.0)):
        r = osm.smooth(v, f, **kw)
        assert np.array_equal(r["vertices"].view(np.uint32), v.view(np.uint32)) and r["iterations"] == 0
    r = osm.smooth(v, np.zeros((0, 3), np.int32))
    assert np.array_equal(r["vertices"], v) and r["iterations"] == 0


def test_hexagon_centre_moves_to_ring_mean():
    v, f = hexagon_fan()
    relax = 0.37
    r = osm.smooth(v, f, iterations=1, relaxation_factor=relax, boundary_smoothing=False)
    assert list(r["types"]) == [SIMPLE] + [FIXED] * 6
    assert sorted(r["lists"][0].tolist()) == [1, 2, 3, 4, 5, 6]
    x = v[0].astype(np.float64)
    d = np.zeros(3)
    for j in r["lists"][0]:
        d += (v[j].astype(np.float64) - x) / 6
    want = (x + relax * d).astype(np.float32)
    assert np.array_equal(r["vertices"][0].view(np.uint32), want.view(np.uint32))
    assert np.array_equal(r["vertices"][1:], v[1:])


def test_gauss_seidel_order():
    """Points 5 and 6 of a 4x4 patch are interior neighbours: 6 sees 5's new position."""
    v, f = grid_patch(4, 4, 7, jitter=0.5)
    relax = 0.5
    r = osm.smooth(v, f, iterations=1, relaxation_factor=relax, boundary_smoothing=False)
    assert r["types"][5] == r["types"][6] == SIMPLE and 5 in r["lists"][6] and 6 in r["lists"][5]

    def move(p, P):
        x = P[p].astype(np.float64)
        d = np.zeros(3)
        for j in r["lists"][p]:
            d += (P[j].astype(np.float64) - x) / len(r["lists"][p])
        return (x + relax * d).astype(np.float32)

    after5 = v.copy()
    after5[5] = move(5, v)
    assert np.array_equal(r["vertices"][5], after5[5])
    assert np.array_equal(r["vertices"][6], move(6, after5))
    assert not np.array_equal(r["vertices"][6], move(6, v))       # a Jacobi sweep gives another surface


def test_boundary_smoothing_slides_along_straight_boundary():
    v, f = grid_patch(5, 4, jitter=0.0)
    v[1, 0] = 0.6                                                  # off-centre on the straight bottom row
    r = osm.smooth(v, f, iterations=5, relaxation_factor=0.5)
    assert r["types"][1] == BOUNDARY and sorted(r["lists"][1].tolist()) == [0, 2]
    assert r["vertices"][1, 0] != v[1, 0]
    assert r["vertices"][1, 1] == 0.0 and r["vertices"][1, 2] == 0.0
    assert r["types"][0] == FIXED and np.array_equal(r["vertices"][0], v[0])   # the sharp corner


def test_more_than_two_edge_neighbours_is_fixed():
    v = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [-1, 0, 0], [-1, -1, 0]], np.float32)
    f = np.array([(0, 1, 2), (0, 3, 4)], np.int32)                # a bow tie: four boundary edges at 0
    r = osm.smooth(v, f, iterations=3, relaxation_factor=0.5)
    assert r["types"][0] == FIXED and np.array_equal(r["vertices"][0], v[0])
    v, f = fin()
    r = osm.smooth(v, f, **SETTINGS["features_on"])
    assert r["types"][0] == FIXED and r["types"][1] == FIXED


def test_feature_edges_of_a_fold():
    v, f = folded_sheet(9)
    r = osm.smooth(v, f, iterations=3, relaxation_factor=0.3, feature_angle=30.0, feature_edge_smoothing=True)
    fold = [j * 9 + 4 for j in range(1, 8)]                        # the fold line's inner points
    assert all(r["types"][p] == FEATURE for p in fold)
    off = osm.smooth(v, f, iterations=3, relaxation_factor=0.3)
    assert all(off["types"][p] == SIMPLE for p in fold)


def test_convergence_stops_where_predicted():
    """The centre of a hexagon fan with its ring fixed moves relax (1 - relax)^t |x0 - m| in iteration t;
    the threshold half a factor above iteration k's move stops the sweep after iteration k (k + 1 done)."""
    v, f = hexagon_fan(center=(0.4, 0.1, 0.3))
    relax, k = 0.3, 6
    m = v[1:].astype(np.float64).mean(0)
    dist = float(np.linalg.norm(v[0].astype(np.float64) - m))
    lo, hi = v.astype(np.float64).min(0), v.astype(np.float64).max(0)
    dx, dy, dz = (float(x) for x in hi - lo)
    diag = math.sqrt(dx * dx + dy * dy + dz * dz)
    conv = relax * (1 - relax) ** (k - 0.5) * dist / diag
    r = osm.smooth(v, f, iterations=100, relaxation_factor=relax, boundary_smoothing=False, convergence=conv)
    assert r["iterations"] == k + 1
    assert smooth_py(v, f, iterations=100, relaxation_factor=relax, boundary_smoothing=False,
                     convergence=conv)[3] == k + 1
    assert osm.smooth(v, f, iterations=100, relaxation_factor=relax, boundary_smoothing=False)["iterations"] > 20


def test_bad_input():
    v, f = icosphere(1.0, 0)
    with pytest.raises(ValueError):
        osm.smooth(v, np.concatenate([f, [[0, 1, len(v)]]]).astype(np.int32))
    with pytest.raises(ValueError):
        osm.smooth(v, f, iterations=-1)
