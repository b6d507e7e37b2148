"""Surface hole filling on the device (invesalius3_b200.surface_holes) against the C checker
(oracle/fill_holes.c), exactly: the faces, the boundary-line count and every loop's record (radii as
uint64)."""
import numpy as np
import pytest

import fill_holes_meshes as fm
from connectivity_meshes import dense_random, noise_volume, shuffled_spheres
from oracle import fill_holes as ofh
from oracle import smoothing as osm
from smoothing_meshes import APPLY_SMOOTH, fin, grid_patch, with_degenerate, with_unused
from visibility_meshes import icosphere, nested_shells

pytestmark = pytest.mark.gpu


def _form(f, dtype, cols):
    f = f.astype(dtype)
    if cols == 4:
        f = np.concatenate([np.full((len(f), 1), 3, dtype), f], 1)
    return f


def _run(v, f, hole_size=1.0, dtype=np.int32, cols=3):
    """Device against the checker on the same arrays; returns the device result."""
    import torch
    from invesalius3_b200 import surface_holes as sh
    fin_ = _form(f, dtype, cols)
    vt = torch.from_numpy(np.ascontiguousarray(v)).cuda()
    ft = torch.from_numpy(np.ascontiguousarray(fin_)).cuda()
    want = ofh.fill_holes(v, f, hole_size)
    got = sh.fill_holes_device(vt, ft, hole_size)
    assert got.faces.dtype == ft.dtype and got.faces.shape[1] == cols
    assert np.array_equal(got.faces.cpu().numpy(), _form(want["faces"], dtype, cols))
    assert got.lines == want["lines"]
    assert np.array_equal(got.first_line.cpu().numpy(), want["first_line"])
    assert np.array_equal(got.points.cpu().numpy(), want["npts"])
    assert np.array_equal(got.radius.cpu().numpy().view(np.uint64), want["radius"].view(np.uint64))
    assert np.array_equal(got.status.cpu().numpy(), want["status"])
    assert np.array_equal(vt.cpu().numpy().view(np.uint32), np.ascontiguousarray(v).view(np.uint32))
    assert np.array_equal(ft.cpu().numpy(), fin_)                  # the inputs are not modified
    return got


MESHES = {
    "icosphere_minus_one": fm.icosphere_minus_one,
    "cube_minus_quad": fm.cube_minus_quad,
    "grid": lambda: grid_patch(40, 30, 1),
    "collinear": fm.collinear_loop,
    "sliver": fm.closed_plus_sliver,
    "closed": lambda: icosphere(1.0, 3),
    "dense": lambda: dense_random(3000, 500, 3),
    "fin": fin,
    "degenerate": lambda: with_degenerate(*grid_patch(30, 20, 2), seed=5),
    "unused": lambda: with_unused(*fm.icosphere_minus_one(3), seed=3),
    "tube": lambda: fm.open_tube(300),
}


@pytest.mark.parametrize("name", list(MESHES))
@pytest.mark.parametrize("hole_size", [0.05, 1.0, 1000.0])
def test_small_meshes(name, hole_size):
    _run(*MESHES[name](), hole_size)


@pytest.mark.parametrize("seed", range(6))
def test_random_deletion(seed):
    """Many bow-tie points: chains between points with more than two lines, closed and open."""
    v, f = fm.random_deletion(*icosphere(1.0, 4), 0.1 + 0.1 * seed, seed)
    for h in (0.05, 0.3, 10.0):
        _run(v, f, h)
    v, f = fm.random_deletion(*shuffled_spheres(12, seed), 0.3, seed)
    _run(v, f, 10.0)


@pytest.mark.parametrize("seed", range(16))
def test_bowtie_orders(seed):
    n = len(fm.bowtie()[1])
    _run(*fm.bowtie(np.random.default_rng(seed).permutation(n)), 2.0)


@pytest.mark.parametrize("dtype,cols", [(np.int32, 3), (np.int64, 3), (np.int32, 4), (np.int64, 4)])
def test_face_forms(dtype, cols):
    v, f = fm.random_deletion(*shuffled_spheres(6, 4), 0.25, 7)
    _run(v, f, 10.0, dtype, cols)


def test_long_loop():
    """A tube closed at one end by a fan: one loop of 20 000 points."""
    v, f = fm.open_tube(20_000, 2, radius=100.0)
    centre = len(v)
    v = np.concatenate([v, np.array([[0.0, 0.0, 0.0]], np.float32)])
    cap = np.array([(centre, (i + 1) % 20_000, i) for i in range(20_000)], np.int32)
    f = np.concatenate([f, cap])
    got = _run(v, f, 1000.0)
    assert got.points.cpu().tolist() == [20_000] and got.status.cpu().tolist() == [ofh.FILLED]
    assert len(got.faces) == len(f) + 19_998


def test_errors_and_empty():
    import torch
    from invesalius3_b200 import surface_holes as sh
    v, f = fm.icosphere_minus_one()
    with pytest.raises(ValueError, match="index"):
        sh.fill_holes(v, np.concatenate([f, [[0, 1, len(v)]]]).astype(np.int32))
    with pytest.raises(ValueError):
        sh.fill_holes(v, f, float("nan"))
    with pytest.raises(TypeError):
        sh.fill_holes(v.astype(np.float64), f)
    bad = _form(f, np.int64, 4)
    bad[3, 0] = 4
    with pytest.raises(ValueError):
        sh.fill_holes(v, bad)
    assert sh.fill_holes(v, np.zeros((0, 3), np.int32)).shape == (0, 3)
    out = sh.fill_holes(v, f, -5.0)                                # clamped to 0: the hole is too large
    assert np.array_equal(out, f)
    assert len(sh.fill_holes(v, f, float("inf"))) == len(f) + 1   # clamped to FLT_MAX
    r = sh.fill_holes_device(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda())
    assert r.lines == 3 and r.status.cpu().tolist() == [sh.FILLED]


def _mc(mask):
    import torch
    from invesalius3_b200.mesh import marching_cubes
    V, F = marching_cubes(torch.from_numpy(np.ascontiguousarray(mask)).cuda(), 127, (1.0, 1.0, 1.0), (0, 0, 0), True)
    return V.cpu().numpy(), F.cpu().numpy()


def _cranium_surface(cranium):
    import torch
    from invesalius3_b200.mesh import marching_cubes
    full = tuple(int(s) for s in cranium["full_shape"])
    mask = np.unpackbits(cranium["mask_0_bits_full"])[:np.prod(full)].reshape(full) * np.uint8(255)
    sx, sy, sz = (float(s) for s in cranium["spacing"])
    V, F = marching_cubes(torch.from_numpy(mask).cuda(), 127, (sx, sy, sz), (0, 0, 0), True)
    return V.cpu().numpy(), F.cpu().numpy()


def test_cranium_surface(cranium):
    v, f = _cranium_surface(cranium)
    assert len(f) > 100_000
    for h in (1.0, 300.0, 1000.0):
        got = _run(v, f, h)
    assert got.lines > 0 and len(got.points) > 1


def test_phantom_surfaces():
    import torch
    from invesalius3_b200 import device as dev, phantom
    from invesalius3_b200.mesh import marching_cubes
    vol = phantom.ct((512, 512, 512), seed=2)
    mask = dev.threshold(torch.from_numpy(vol).cuda(), 226, 3071)
    del vol
    V, F = marching_cubes(mask, 127, (1.0, 1.0, 1.0), (0, 0, 0), True)
    v, f = V.cpu().numpy(), F.cpu().numpy()
    got = _run(v, f, 1000.0)                                       # closed: nothing to fill
    assert got.lines == 0 and len(got.faces) == len(f)
    del V, F
    V, F = marching_cubes(mask[128:384].contiguous(), 127, (1.0, 1.0, 1.0), (0, 0, 0), True)
    del mask
    v, f = V.cpu().numpy(), F.cpu().numpy()
    assert len(f) > 5_000_000
    for h in (1.0, 1000.0):
        got = _run(v, f, h)
    assert got.lines > 0 and (got.status.cpu().numpy() == ofh.FILLED).any()


def test_noise_surface():
    v, f = _mc(noise_volume(128, 0.5, 1))
    for h in (1.0, 300.0):
        got = _run(v, f, h)
    assert len(got.points) > 1000


def test_after_removing_non_visible_faces():
    import torch
    from invesalius3_b200.visible_faces import remove_non_visible_faces_device
    v, f, _ = nested_shells(1.0, 4)
    V, F = remove_non_visible_faces_device(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda())
    _run(V.cpu().numpy(), F.cpu().numpy(), 1000.0)


def test_apply_smooth_filter_on_the_cranium(cranium):
    import torch
    from invesalius3_b200 import surface_smoothing as ss
    v, f = _cranium_surface(cranium)
    sm = osm.smooth(v, f, **APPLY_SMOOTH)["vertices"]
    want = ofh.fill_holes(sm, f, 1000.0)["faces"]
    it, rf = APPLY_SMOOTH["iterations"], APPLY_SMOOTH["relaxation_factor"]
    vt, ft = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    gv, gf = ss.apply_smooth_filter_device(vt, ft, it, rf)
    assert np.array_equal(gv.cpu().numpy().view(np.uint32), sm.view(np.uint32))
    assert np.array_equal(gf.cpu().numpy(), want.astype(np.int32)) and len(want) > len(f)
    assert np.array_equal(vt.cpu().numpy(), v) and np.array_equal(ft.cpu().numpy(), f)
    nv, nf = ss.apply_smooth_filter(v, f, it, rf)
    assert np.array_equal(nv.view(np.uint32), sm.view(np.uint32)) and np.array_equal(nf, want)
