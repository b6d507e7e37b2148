"""Remove non-visible faces on the device (invesalius3_b200.visible_faces) against the C checker
(oracle/visibility.c), bit for bit: the camera records, every view's depth buffer, the per-vertex
visibility, the number of triangles drawn by the cooperative (large-triangle) path, and the output arrays."""
import numpy as np
import pytest

from oracle import visibility as ov
from visibility_meshes import cube, icosphere, nested_shells, select_and_clean, soup

pytestmark = pytest.mark.gpu


def _run(v, f, positions=ov.DEFAULT_POSITIONS, remove_visible=False):
    """Device and checker on the same arrays; asserts equality and returns the checker's output."""
    import torch
    from invesalius3_b200 import visible_faces as vf
    dbg = {}
    vt, ft = torch.from_numpy(np.ascontiguousarray(v)).cuda(), torch.from_numpy(np.ascontiguousarray(f)).cuda()
    vo, fo = vf.remove_non_visible_faces_device(vt, ft, positions, remove_visible, _debug=dbg)
    wv, wf, w = ov.remove_non_visible_faces(v, f, positions, remove_visible, debug=True)
    assert np.array_equal(dbg["bounds"], ov.bounds(v))
    assert np.array_equal(dbg["cameras"], w["cameras"])
    zb = dbg["zbuf"].cpu().numpy()
    for k in range(len(zb)):
        assert np.array_equal(zb[k], w["zbuf"][k]), f"depth buffer of view {k}"
    assert np.array_equal(dbg["visible"].cpu().numpy(), w["visible"])
    assert int(dbg["big_triangles"].item()) == w["big_triangles"]
    got_v, got_f = vo.cpu().numpy(), fo.cpu().numpy()
    assert got_f.dtype == f.dtype and got_f.shape[1] == f.shape[1]
    if f.shape[1] == 4:
        assert (got_f[:, 0] == 3).all()
        got_f = got_f[:, 1:]
    assert np.array_equal(got_v.view(np.uint32), wv.view(np.uint32))
    assert np.array_equal(got_f, wf)
    return wv, wf, w


def test_nested_shells():
    v, f, n_outer = nested_shells(1.0, 5)
    wv, wf, w = _run(v, f)
    assert len(wf) == n_outer and np.array_equal(wv[wf], v[f[:n_outer]])
    assert w["visible"][:len(v) // 2].all() and not w["visible"][len(v) // 2:].any()
    wv, wf, w = _run(v, f, remove_visible=True)
    assert np.array_equal(wv[wf], v[f[n_outer:]])


@pytest.mark.parametrize("dtype", [np.int32, np.int64])
@pytest.mark.parametrize("cols", [3, 4])
def test_face_dtypes_and_forms(dtype, cols):
    v, f, _ = nested_shells(3.0, 3)
    f = f.astype(dtype)
    if cols == 4:
        f = np.concatenate([np.full((len(f), 1), 3, dtype), f], 1)
    _run(v, f)
    _run(v, f, remove_visible=True)


def test_cranium_bone_surface(cranium):
    import torch
    from invesalius3_b200.mesh import marching_cubes
    full = tuple(int(s) for s in cranium["full_shape"])
    mask = np.unpackbits(cranium["mask_0_bits_full"])[:np.prod(full)].reshape(full) * np.uint8(255)
    sx, sy, sz = (float(s) for s in cranium["spacing"])
    V, F = marching_cubes(torch.from_numpy(mask).cuda(), 127, (sx, sy, sz), (0, 0, 0), True)
    v, f = V.cpu().numpy(), F.cpu().numpy()
    assert len(f) > 100000
    wv, wf, w = _run(v, f)
    assert 0 < len(wf) < len(f) and 0 < w["visible"].sum() < len(v)
    _run(v, f, remove_visible=True)


def test_phantom_512_bone_surface():
    import torch
    from invesalius3_b200 import device as dev, phantom
    from invesalius3_b200.mesh import marching_cubes
    vol = phantom.ct((512, 512, 512), seed=2)
    mask = dev.threshold(torch.from_numpy(vol).cuda(), 226, 3071)
    del vol
    V, F = marching_cubes(mask, 127, (1.0, 1.0, 1.0), (0, 0, 0), True)
    del mask
    wv, wf, w = _run(V.cpu().numpy(), F.cpu().numpy())
    assert 0 < len(wf) < F.shape[0]


def test_viewport_filling_cube_takes_the_cooperative_path():
    v, f = cube(1.0)
    wv, wf, w = _run(v, f)
    assert w["big_triangles"] > 0 and len(wf) == 12
    # one view straight at a face: its two triangles cover a large part of the viewport
    wv, wf, w = _run(v, f, positions=[(0, 0, 1)])
    assert w["big_triangles"] >= 2 and (w["zbuf"][0] < 1.0).mean() > 0.2
    # a coarse sphere around a dense one: every depth comes from large triangles
    vo, fo = icosphere(2.0, 0)
    vi, fi = icosphere(1.0, 3)
    _run(np.concatenate([vo, vi]), np.concatenate([fo, fi + len(vo)]))


def test_triangle_soup_is_merged():
    v, f = icosphere(1.5, 3)
    sv, sf = soup(v, f, seed=4)
    sv[sv == 0] = -0.0                          # signed zeros merge with their +0 copies
    wv, wf, w = _run(sv, sf)
    assert len(wv) == len(v) and len(wf) == len(f)
    wv, wf, w = _run(sv, sf.astype(np.int64), positions=[(0, 1, 0)])
    assert 0 < len(wf) < len(f)


def test_non_axis_positions():
    v, f, n_outer = nested_shells(1.0, 4)
    pos = [(1, 1, 0), (-0.3, 2, 0.7), (0, 0, -5), (1e-3, 1, 1)]
    wv, wf, w = _run(v, f, positions=pos)
    assert len(wf) <= n_outer
    v2, f2 = icosphere(1.0, 4)
    wv, wf, w = _run(v2, f2, positions=[(0.6, -0.8, 0.2)])
    check_v, check_f = select_and_clean(v2, f2, w["visible"], False)
    assert np.array_equal(wv, check_v) and np.array_equal(wf, check_f)
    assert 0 < len(wf) < len(f2)


def test_numpy_entry_and_errors():
    import torch
    from invesalius3_b200 import visible_faces as vf
    v, f, n_outer = nested_shells(1.0, 3)
    f4 = np.concatenate([np.full((len(f), 1), 3, np.int64), f], 1)
    vo, fo = vf.remove_non_visible_faces(v, f4)
    wv, wf = ov.remove_non_visible_faces(v, f4)
    assert fo.dtype == np.int64 and np.array_equal(vo, wv) and np.array_equal(fo[:, 1:], wf)
    with pytest.raises(ValueError, match="index"):
        vf.remove_non_visible_faces(v, np.concatenate([f, [[0, 1, len(v)]]]).astype(np.int32))
    bad4 = f4.copy()
    bad4[5, 0] = 4
    with pytest.raises(ValueError):
        vf.remove_non_visible_faces(v, bad4)
    vt = torch.from_numpy(v).cuda()
    vt[7, 2] = float("nan")
    with pytest.raises(ValueError, match="finite"):
        vf.remove_non_visible_faces_device(vt, torch.from_numpy(f).cuda())
    with pytest.raises(ValueError):
        vf.remove_non_visible_faces_device(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), [(0, 0, 0)])
