"""Surface normals and mass properties on the device (invesalius3_b200.surface_normals) against the C checker
(oracle/normals.c): points, faces, point and cell normals as bits, and every count; the per-triangle mass
terms and the totals as bits."""
import numpy as np
import pytest

import normals_model as nm
from normals_model import small_meshes
from connectivity_meshes import noise_volume, strip
from oracle import normals as on

pytestmark = pytest.mark.gpu

FORMS = [(np.int32, 3), (np.int64, 3), (np.int32, 4), (np.int64, 4)]


def _form(f, dtype, cols):
    f = f.astype(dtype)
    if cols == 4:
        f = np.concatenate([np.full((len(f), 1), 3, dtype), f], 1)
    return f


def _run(v, f, angle=30.0, auto_orient=False, dtype=np.int32, cols=3):
    import torch
    from invesalius3_b200 import surface_normals as sn
    fin_ = _form(f, dtype, cols)
    vt = torch.from_numpy(np.ascontiguousarray(v)).cuda()
    ft = torch.from_numpy(np.ascontiguousarray(fin_)).cuda()
    want = on.compute_normals(v, f, angle, auto_orient)
    got = sn.compute_normals_device(vt, ft, angle, auto_orient)
    assert got.faces.dtype == ft.dtype and got.faces.shape[1] == cols
    assert np.array_equal(got.faces.cpu().numpy(), _form(want["faces"], dtype, cols))
    for k in ("points", "point_normals", "cell_normals"):
        assert np.array_equal(getattr(got, k).cpu().numpy().view(np.uint32), want[k].view(np.uint32)), k
    assert (got.regions, got.flips, got.new_points, got.waves) == \
        (want["regions"], want["flips"], want["new_points"], want["waves"])
    assert np.array_equal(ft.cpu().numpy(), fin_)                  # the input is not modified
    return got


@pytest.mark.parametrize("name", list(small_meshes()))
@pytest.mark.parametrize("angle", [30.0, 80.0, 160.0])
@pytest.mark.parametrize("auto_orient", [False, True])
@pytest.mark.parametrize("dtype,cols", FORMS)
def test_small_meshes(name, angle, auto_orient, dtype, cols):
    _run(*small_meshes()[name](), angle, auto_orient, dtype, cols)


def _configs():
    forms = FORMS * 2
    return [(a, o, *forms[2 * i + o]) for i, a in enumerate((30.0, 80.0, 160.0)) for o in (False, True)]


def _all_configs(v, f):
    for angle, auto, dtype, cols in _configs():
        got = _run(v, f, angle, auto, dtype, cols)
    return got


def test_long_strip():
    v, f = nm.randomly_flipped(*strip(200_000), 7)
    _all_configs(v, f)
    got = _run(v, f)
    assert got.waves > 1000 and got.flips > 0
    assert _run(v, f, 30.0, True).regions == 0                     # flat in z = 0: no cell has n.x != 0


def _mc(mask, spacing=(1.0, 1.0, 1.0)):
    import torch
    from invesalius3_b200.mesh import marching_cubes
    V, F = marching_cubes(torch.from_numpy(np.ascontiguousarray(mask)).cuda(), 127, spacing, (0, 0, 0), True)
    return V.cpu().numpy(), F.cpu().numpy()


def test_noise_surface_many_regions():
    v, f = nm.randomly_flipped(*_mc(noise_volume(96, 0.12, 1)), 3)
    got = _all_configs(v, f)
    assert got.regions > 20_000


def test_cranium_surface(cranium):
    full = tuple(int(s) for s in cranium["full_shape"])
    mask = np.unpackbits(cranium["mask_0_bits_full"])[:np.prod(full)].reshape(full) * np.uint8(255)
    v, f = _mc(mask, tuple(float(s) for s in cranium["spacing"]))
    assert len(f) > 100_000
    _all_configs(v, f)
    _mass(v, f)


def test_phantom_surface():
    import torch
    from invesalius3_b200 import device as dev, phantom
    vol = phantom.ct((512, 512, 512), seed=2)
    mask = dev.threshold(torch.from_numpy(vol).cuda(), 226, 3071).cpu().numpy()
    del vol
    v, f = _mc(mask)
    del mask
    for angle, auto in ((80.0, True), (30.0, False)):
        got = _run(v, f, angle, auto)
    assert got.new_points > 0
    _mass(v, f)


def _mass(v, f):
    import torch
    from invesalius3_b200 import _lib
    from invesalius3_b200 import surface_normals as sn
    from invesalius3_b200.device import _p, _stream
    vol, area, terms, cls = on.mass_properties(v, f, terms=True)
    vt, ft = torch.from_numpy(np.ascontiguousarray(v)).cuda(), torch.from_numpy(np.ascontiguousarray(f)).cuda()
    got = sn.mass_properties_device(vt, ft)
    assert got == (vol, area)                                       # summed in the checker's order
    assert sn.mass_properties_device(vt, ft) == got
    # the per-triangle terms, as bits, through the workspace layout
    lib = _lib.load()
    nv, nt = len(v), len(f)
    ws = torch.empty(int(lib.b2v_normals_workspace_bytes(nv, nt)), dtype=torch.uint8, device="cuda")
    out = (_lib.C.c_double * 2)()
    _lib.call("b2v_mass_properties", _p(vt), nv, _p(ft), nt, 3, int(ft.dtype == torch.int64), _p(ws), _stream(), out)
    lay = (_lib.C.c_int64 * 4)()
    _lib.call("b2v_normals_layout", nv, nt, lay)
    raw = ws.cpu().numpy()
    t = raw[lay[2]:lay[2] + 32 * nt].view(np.float64).reshape(nt, 4)
    c = raw[lay[3]:lay[3] + nt].view(np.int8)
    assert np.array_equal(t.view(np.uint64), terms.view(np.uint64)) and np.array_equal(c, cls)


@pytest.mark.parametrize("name", list(small_meshes()))
def test_mass_properties_small(name):
    _mass(*small_meshes()[name]())


def test_mass_properties_noise():
    _mass(*_mc(noise_volume(64, 0.5, 2)))


def test_chain_on_device():
    """marching cubes -> smoothing -> hole filling -> normals -> mass properties, on tensors throughout."""
    import torch
    from invesalius3_b200 import surface_normals as sn
    from invesalius3_b200.mesh import marching_cubes
    from invesalius3_b200.surface_holes import fill_holes_device
    from invesalius3_b200.surface_smoothing import smooth_polydata_device
    g = np.mgrid[0:48, 0:48, 0:48].astype(np.float32)
    mask = ((((g - 24) ** 2).sum(0) < 18 ** 2) * 255).astype(np.uint8)
    V, F = marching_cubes(torch.from_numpy(mask).cuda(), 127, (1.0, 1.0, 1.0), (0, 0, 0), True)
    S = smooth_polydata_device(V, F, 20, 0.4, 80.0, 15.0, False, False).vertices
    H = fill_holes_device(S, F[1:].contiguous(), 1000.0).faces     # one triangle gone: a hole to fill
    r = sn.compute_normals_device(S, H, 80.0, True)
    vol, area = sn.mass_properties_device(r.points, r.faces)
    assert all(t.is_cuda for t in (V, F, S, H, r.points, r.faces, r.point_normals, r.cell_normals))
    s, h = S.cpu().numpy(), H.cpu().numpy()
    _run(s, h, 80.0, True)
    want = on.mass_properties(r.points.cpu().numpy(), r.faces.cpu().numpy())
    assert (vol, area) == want
    assert len(h) == len(F) and r.regions == 1


def test_bad_input():
    import torch
    from invesalius3_b200 import surface_normals as sn
    v, f = nm.box()
    with pytest.raises(ValueError, match="index"):
        sn.compute_normals(v, np.concatenate([f, [[0, 1, 8]]]).astype(np.int32))
    with pytest.raises(ValueError):
        sn.compute_normals(v, f, float("nan"))
    with pytest.raises(TypeError):
        sn.compute_normals(v.astype(np.float64), f)
    with pytest.raises(TypeError):
        sn.mass_properties(v, f.astype(np.int16))
    with pytest.raises(ValueError):
        sn.mass_properties(v, np.concatenate([f, [[0, -1, 2]]]).astype(np.int32))
    bad = _form(f, np.int64, 4)
    bad[3, 0] = 4
    with pytest.raises(ValueError):
        sn.compute_normals(v, bad)
    with pytest.raises(ValueError):
        sn.compute_normals_device(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()[:, :2].contiguous())
    pts, faces, pn, cn, flips, new = sn.compute_normals(v, np.zeros((0, 3), np.int32))
    assert pts.shape == (8, 3) and faces.shape == (0, 3) and not pn.any() and (flips, new) == (0, 0)
    assert sn.mass_properties(v, np.zeros((0, 3), np.int32)) == (0.0, 0.0)
    pts, faces, pn, cn, flips, new = sn.compute_normals(v, f, 80.0)
    assert len(pts) == 24 and new == 16
