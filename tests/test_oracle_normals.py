"""The surface normals checker (oracle/normals.c) against an independent restatement (normals_model.py) and
against closed forms that rest on no reading of VTK. CPU only."""
import math

import numpy as np
import pytest

import normals_model as nm
from normals_model import small_meshes
from oracle import normals as on
from visibility_meshes import icosphere


def _same(a, b):
    for k in ("points", "point_normals", "cell_normals"):
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), k
    assert np.array_equal(a["faces"], b["faces"])
    for k in ("regions", "flips", "new_points", "waves"):
        assert a[k] == b[k], k


@pytest.mark.parametrize("name", list(small_meshes()))
@pytest.mark.parametrize("angle", [30.0, 80.0, 160.0])
@pytest.mark.parametrize("auto_orient", [False, True])
def test_checker_equals_model(name, angle, auto_orient):
    v, f = small_meshes()[name]()
    _same(on.compute_normals(v, f, angle, auto_orient), nm.compute_normals(v, f, angle, auto_orient))


@pytest.mark.parametrize("name", list(small_meshes()))
def test_mass_properties_equal_model(name):
    v, f = small_meshes()[name]()
    assert on.mass_properties(v, f) == nm.mass_properties(v, f)


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("shape", ["sphere", "box"])
def test_auto_orient_points_outward(seed, shape):
    v, f = icosphere(2.0, 3, center=(5.0, -1.0, 2.0)) if shape == "sphere" else nm.box((1, -2, 0.5), (4, 1, 2))
    centre = v.astype(np.float64).mean(0)
    v, f = nm.randomly_flipped(v, f, seed)
    r = on.compute_normals(v, f, 30.0, True)
    out = r["points"][r["faces"]].astype(np.float64).mean(1) - centre
    assert (np.einsum("ij,ij->i", r["cell_normals"].astype(np.float64), out) > 0).all()
    assert r["regions"] == 1
    plain = on.compute_normals(v, f, 30.0, False)
    assert plain["regions"] == 1                        # consistent, but the orientation of cell 0


def test_box_splits_at_80_degrees():
    v, f = nm.box()
    r = on.compute_normals(v, f, 80.0)
    assert len(r["points"]) == 24 and r["new_points"] == 16
    faces = {tuple(n) for n in r["cell_normals"].tolist()}
    assert len(faces) == 6
    assert all(tuple(n) in faces for n in r["point_normals"].tolist())
    assert np.array_equal(np.sort(r["points"].view(np.uint32), 0),
                          np.sort(np.repeat(v, 3, 0).view(np.uint32), 0))


def test_box_keeps_corners_at_100_degrees():
    v, f = nm.box()
    r = on.compute_normals(v, f, 100.0)
    assert len(r["points"]) == 8 and r["new_points"] == 0
    centre = v.mean(0)
    pn = r["point_normals"]
    assert np.allclose(np.linalg.norm(pn, axis=1), 1.0, atol=1e-6)
    assert (np.sign(pn) == np.sign(v - centre)).all()


def test_box_mass_properties():
    lo, hi = (1.0, -2.0, 0.5), (4.0, 1.0, 2.5)
    volume, area = on.mass_properties(*nm.box(lo, hi))
    dx, dy, dz = (b - a for a, b in zip(lo, hi))
    assert volume == pytest.approx(dx * dy * dz, rel=1e-15)
    assert area == pytest.approx(2 * (dx * dy + dy * dz + dx * dz), rel=1e-15)


def test_icosphere_mass_properties():
    r = 3.0
    volume, area = on.mass_properties(*icosphere(r, 5, center=(1.0, 2.0, -4.0)))
    assert volume == pytest.approx(4 / 3 * math.pi * r ** 3, rel=2e-3)
    assert area == pytest.approx(4 * math.pi * r ** 2, rel=2e-3)
    assert volume < 4 / 3 * math.pi * r ** 3 and area < 4 * math.pi * r ** 2      # inscribed


def test_bad_input():
    v, f = nm.box()
    with pytest.raises(ValueError):
        on.compute_normals(v, np.concatenate([f, [[0, 1, 8]]]).astype(np.int32))
    with pytest.raises(ValueError):
        on.compute_normals(v, f, float("nan"))
    with pytest.raises(ValueError):
        on.mass_properties(v, np.concatenate([f, [[0, -1, 2]]]).astype(np.int32))
    e = on.compute_normals(v, np.zeros((0, 3), np.int32))
    assert len(e["points"]) == 8 and not e["point_normals"].any() and e["regions"] == 0
    assert on.mass_properties(v, np.zeros((0, 3), np.int32)) == (0.0, 0.0)
