"""Laplacian surface smoothing on the device (invesalius3_b200.surface_smoothing) against the C checker
(oracle/smoothing.c), bit for bit: the vertices (as uint32), the point types and the iteration count."""
import numpy as np
import pytest

from connectivity_meshes import dense_random, fan, shuffled_spheres, strip
from oracle import smoothing as osm
from smoothing_meshes import (APPLY_SMOOTH, DECIMATE, SETTINGS, fin, folded_sheet, grid_patch, hexagon_fan,
                              with_degenerate, with_unused)
from visibility_meshes import icosphere

pytestmark = pytest.mark.gpu


def _form(f, dtype, cols):
    f = f.astype(dtype)
    if cols == 4:
        f = np.concatenate([np.full((len(f), 1), 3, dtype), f], 1)
    return f


def _run(v, f, dtype=np.int32, cols=3, **kw):
    """Device against the checker on the same arrays; returns the device result."""
    import torch
    from invesalius3_b200 import surface_smoothing as ss
    vt = torch.from_numpy(np.ascontiguousarray(v)).cuda()
    ft = torch.from_numpy(np.ascontiguousarray(_form(f, dtype, cols))).cuda()
    want = osm.smooth(v, f, **kw)
    got = ss.smooth_polydata_device(vt, ft, **kw)
    assert np.array_equal(got.vertices.cpu().numpy().view(np.uint32), want["vertices"].view(np.uint32))
    assert np.array_equal(got.point_types.cpu().numpy(), want["types"])
    assert got.iterations == want["iterations"]
    assert np.array_equal(vt.cpu().numpy(), v)                     # the input is not modified
    return got


MESHES = {
    "icosphere": lambda: icosphere(1.0, 5),
    "spheres": lambda: shuffled_spheres(9, 3),
    "dense": lambda: dense_random(3000, 2000, 2),
    "fan": lambda: fan(5000),
    "grid": lambda: grid_patch(150, 120, 1),
    "fin": fin,
    "degenerate": lambda: with_degenerate(*grid_patch(60, 50, 2), seed=5),
    "unused": lambda: with_unused(*icosphere(1.0, 3), seed=3),
    "folded": lambda: folded_sheet(41),
}


@pytest.mark.parametrize("name", list(MESHES))
@pytest.mark.parametrize("setting", list(SETTINGS))
def test_small_meshes(name, setting):
    v, f = MESHES[name]()
    _run(v, f, **SETTINGS[setting])


@pytest.mark.parametrize("dtype,cols", [(np.int32, 3), (np.int64, 3), (np.int32, 4), (np.int64, 4)])
def test_face_forms(dtype, cols):
    v, f = with_unused(*shuffled_spheres(4, 8), seed=1)
    _run(v, f, dtype, cols, **APPLY_SMOOTH)
    _run(v, f, dtype, cols, **DECIMATE)


@pytest.mark.parametrize("iterations", [0, 1, 100])
def test_iteration_counts(iterations):
    v, f = grid_patch(80, 70, 4, jitter=0.4)
    got = _run(v, f, iterations=iterations, relaxation_factor=0.2)
    assert got.iterations == iterations
    if iterations == 0:
        assert got.steps == 0


def test_early_stop():
    v, f = hexagon_fan(center=(0.4, 0.1, 0.3))
    got = _run(v, f, iterations=100, relaxation_factor=0.3, boundary_smoothing=False, convergence=1e-3)
    assert 1 < got.iterations < 100
    v, f = icosphere(1.0, 4)
    for conv in (1e-3, 4e-3):
        got = _run(v, f, iterations=500, relaxation_factor=0.3, convergence=conv)
        assert got.iterations < 500


def test_nothing_to_do_and_errors():
    import torch
    from invesalius3_b200 import surface_smoothing as ss
    v, f = icosphere(1.0, 2)
    out = ss.smooth_polydata(v, f, relaxation_factor=0.0)
    assert np.array_equal(out.view(np.uint32), v.view(np.uint32))
    out = ss.smooth_polydata(v, np.zeros((0, 3), np.int64))
    assert np.array_equal(out, v)
    assert ss.smooth_polydata(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32)).shape == (0, 3)
    r = ss.smooth_polydata_device(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), iterations=3)
    assert r.iterations == 3 and r.steps == 3 * r.levels
    np.testing.assert_array_equal(ss.smooth_polydata(v, f, **APPLY_SMOOTH), osm.smooth(v, f, **APPLY_SMOOTH)["vertices"])
    with pytest.raises(ValueError):
        ss.smooth_polydata(v.astype(np.float64), f)
    with pytest.raises(ValueError, match="index"):
        ss.smooth_polydata(v, np.concatenate([f, [[0, 1, len(v)]]]).astype(np.int32))
    with pytest.raises(ValueError):
        ss.smooth_polydata(v, f, iterations=-1)
    bad = _form(f, np.int64, 4)
    bad[3, 0] = 4
    with pytest.raises(ValueError):
        ss.smooth_polydata(v, bad)


def test_open_surface_touching_the_border():
    import torch
    from invesalius3_b200.mesh import marching_cubes
    z, y, x = np.mgrid[0:48, 0:56, 0:64]
    mask = (((x - 8) ** 2 + (y - 20) ** 2 + (z - 30) ** 2) < 26 ** 2).astype(np.uint8) * np.uint8(255)
    V, F = marching_cubes(torch.from_numpy(mask).cuda(), 127, (0.7, 0.8, 1.1), (0, 0, 0), True)
    v, f = V.cpu().numpy(), F.cpu().numpy()
    for kw in (APPLY_SMOOTH, DECIMATE):
        got = _run(v, f, **kw)
    assert (got.point_types.cpu().numpy() == 3).any()              # a boundary, smoothed with VTK's defaults


def test_long_strip():
    v, f = strip(200_000)
    got = _run(v, f, **DECIMATE)                                   # boundary smoothing on: one long chain
    assert got.levels > 90_000
    _run(v, f, **APPLY_SMOOTH)


def test_cranium_bone_surface(cranium):
    import torch
    from invesalius3_b200.mesh import marching_cubes
    full = tuple(int(s) for s in cranium["full_shape"])
    mask = np.unpackbits(cranium["mask_0_bits_full"])[:np.prod(full)].reshape(full) * np.uint8(255)
    sx, sy, sz = (float(s) for s in cranium["spacing"])
    V, F = marching_cubes(torch.from_numpy(mask).cuda(), 127, (sx, sy, sz), (0, 0, 0), True)
    v, f = V.cpu().numpy(), F.cpu().numpy()
    assert len(f) > 100000
    for kw in (APPLY_SMOOTH, DECIMATE):
        _run(v, f, **kw)


def test_phantom_512_bone_surface():
    import torch
    from invesalius3_b200 import device as dev, phantom
    from invesalius3_b200.mesh import marching_cubes
    vol = phantom.ct((512, 512, 512), seed=2)
    mask = dev.threshold(torch.from_numpy(vol).cuda(), 226, 3071)
    del vol
    V, F = marching_cubes(mask, 127, (1.0, 1.0, 1.0), (0, 0, 0), True)
    del mask
    v, f = V.cpu().numpy(), F.cpu().numpy()
    assert len(f) > 5_000_000
    for kw in (APPLY_SMOOTH, DECIMATE):
        _run(v, f, **kw)
