"""The geodesic measurement on the device (invesalius3_b200.surface_geodesic) against the C checker
(oracle/geodesic.c): distances as bits, closest points, path ids where no step is ambiguous and the device's
rule where one is, float32 points and lengths as bits."""
import math

import numpy as np
import pytest

from connectivity_meshes import noise_volume, strip
from normals_model import small_meshes
from oracle import geodesic as og
from test_gpu_surface_normals import FORMS, _form, _mc
from test_oracle_geodesic import half_grid

pytestmark = pytest.mark.gpu


def _tensors(v, f):
    import torch
    return torch.from_numpy(np.ascontiguousarray(v)).cuda(), torch.from_numpy(np.ascontiguousarray(f)).cuda()


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _check_rule(v, ids, g):
    """Every step of a path is an edge attaining d[v], with the smallest d[u] and then the smallest id."""
    assert g["rule"][ids[:-1]].tolist() == ids[1:].tolist()
    p = np.asarray(v, np.float64)
    for a, b in zip(ids[:-1], ids[1:]):
        d = p[a] - p[b]
        assert g["dist"][b] + math.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]) == g["dist"][a]


def _path(v, f, picks, dtype=np.int32, cols=3, surface=None):
    """The device path against the checker, segment by segment; returns the device result."""
    from invesalius3_b200 import surface_geodesic as sg
    vt, ft = _tensors(v, _form(f, dtype, cols))
    v_before, f_before = vt.clone(), ft.clone()
    s = surface or sg.GeodesicSurface(vt, ft)
    got = s.path(picks)
    want = og.geodesic_path(v, f, picks)
    assert len(got.ids) == len(want["ids"]) == max(len(picks) - 1, 0)
    snap = og.closest_points(v, picks)
    assert np.array_equal(s.closest_points(picks).cpu().numpy(), snap)
    for k, (gi, wi) in enumerate(zip(got.ids, want["ids"])):
        gi = gi.cpu().numpy()
        assert got.ambiguous[k] == want["ambiguous"][k] and got.unreached[k] == want["unreached"][k]
        if not want["ambiguous"][k]:
            assert np.array_equal(gi, wi)
        else:
            assert gi[0] == wi[0] and gi[-1] == wi[-1]
            _check_rule(v, gi, og.distances(v, f, snap[k]))
    pts = got.points.cpu().numpy()
    ids = np.concatenate([i.cpu().numpy() for i in got.ids]) if got.ids else np.zeros(0, np.int64)
    assert np.array_equal(pts.view(np.uint32), np.asarray(v)[ids].astype(np.float32).view(np.uint32))
    # lengths: the checker's sum over the device's own points (equal to the checker's path when unambiguous)
    total, bounds = 0.0, np.cumsum([0] + [len(i) for i in got.ids])
    for k, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        seg, total = og.path_length(pts[a:b], total)
        assert _bits(got.lengths[k]) == _bits(seg)
    assert _bits(got.total) == _bits(total)
    if not any(want["ambiguous"]):
        assert _bits(got.total) == _bits(want["total"])
    assert np.array_equal(vt.cpu().numpy(), v_before.cpu().numpy())      # inputs are not modified
    assert np.array_equal(ft.cpu().numpy(), f_before.cpu().numpy())
    again = s.path(picks)                                                 # a second call: the same result
    assert all(np.array_equal(a.cpu().numpy(), b.cpu().numpy()) for a, b in zip(again.ids, got.ids))
    assert _bits(again.total) == _bits(got.total) and again.ambiguous == got.ambiguous
    return got


def _distances(v, f, starts, dtype=np.int32, cols=3):
    """Full-mode distances bit-equal everywhere; early-exit distances bit-equal wherever d <= d[end]."""
    from invesalius3_b200 import surface_geodesic as sg
    s = sg.GeodesicSurface(*_tensors(v, _form(f, dtype, cols)))
    for st in starts:
        want = og.distances(v, f, st)["dist"]
        assert np.array_equal(_bits(s.distances(st).cpu().numpy()), _bits(want))
        reach = np.flatnonzero(np.isfinite(want))
        for end in (st, reach[len(reach) // 3], reach[-1], int(np.argmax(np.where(np.isinf(want), -1, want)))):
            got = s.distances(st, int(end)).cpu().numpy()
            fin = want <= want[end]
            assert np.array_equal(_bits(got[fin]), _bits(want[fin]))
            assert (got[~fin] >= want[~fin]).all()
    return s


def _picks(v, n, seed):
    rng = np.random.default_rng(seed)
    return v[rng.integers(0, len(v), n)].astype(np.float64) + rng.normal(0, 0.05, (n, 3))


@pytest.mark.parametrize("name", list(small_meshes()))
@pytest.mark.parametrize("vdtype", [np.float32, np.float64])
@pytest.mark.parametrize("dtype,cols", FORMS)
def test_small_meshes(name, vdtype, dtype, cols):
    v, f = small_meshes()[name]()
    v = v.astype(vdtype)
    if vdtype == np.float64:
        v = v + np.float64(1e-9) * np.arange(v.size).reshape(v.shape)    # not representable in float32
    _distances(v, f, [0, len(v) // 2], dtype, cols)
    for n in (2, 3, 10):
        _path(v, f, _picks(v, n, n), dtype, cols)


def test_half_grid_ambiguous_paths():
    v, f = half_grid(60)
    _distances(v, f, [0, 1234])
    amb = 0
    for seed in range(6):
        amb += sum(_path(v, f, _picks(v, 10, seed)).ambiguous)
    assert amb > 0


def test_start_equals_end_unreached_and_no_path():
    import torch
    from invesalius3_b200 import surface_geodesic as sg
    from connectivity_meshes import shuffled_spheres
    v, f = shuffled_spheres(4, 1)
    g = og.distances(v, f, 0)
    far = int(np.flatnonzero(np.isinf(g["dist"]))[0])
    got = _path(v, f, np.stack([v[0], v[0], v[far], v[3]]).astype(np.float64))
    assert [i.tolist() for i in got.ids[:2]] == [[0], [far]] and got.unreached[:2] == [False, True]
    vt, ft = _tensors(v, f)
    assert sg.geodesic_path_device(vt, ft, v[:1]).ids == []
    r = sg.geodesic_path_device(vt, ft[:0], v[:2])
    assert r.ids == [] and r.total == 0.0 and r.points.shape == (0, 3)
    with pytest.raises(ValueError, match="index"):
        sg.GeodesicSurface(vt, torch.cat([ft, torch.tensor([[0, 1, len(v)]], dtype=ft.dtype, device="cuda")]))
    with pytest.raises(TypeError):
        sg.GeodesicSurface(vt.half(), ft)


def test_numpy_mirror():
    from invesalius3_b200 import surface_geodesic as sg
    v, f = small_meshes()["icosphere"]()
    picks = _picks(v, 3, 0)
    r = sg.geodesic_path(v, f, picks)
    want = og.geodesic_path(v, f, picks)
    assert all(np.array_equal(a, b) for a, b in zip(r.ids, want["ids"]))
    assert np.array_equal(r.points, want["points"]) and r.total == want["total"]
    ids = sg.closest_points_device(*_tensors(v, f)[:1], picks).cpu().numpy()
    assert np.array_equal(ids, og.closest_points(v, picks))
    d = sg.geodesic_distances_device(*_tensors(v, f), 3).cpu().numpy()
    assert np.array_equal(_bits(d), _bits(og.distances(v, f, 3)["dist"]))


def test_split_points_surface():
    """Points split by the normals at 80 degrees have no edges across the feature lines."""
    from invesalius3_b200 import surface_normals as sn
    import normals_model as nm
    vt, ft = _tensors(*nm.box())
    r = sn.compute_normals_device(vt, ft.int(), 80.0, True)
    v, f = r.points.cpu().numpy(), r.faces.cpu().numpy()
    assert r.new_points > 0
    _distances(v, f, [0, 5])
    for n in (2, 3, 10):
        _path(v, f, _picks(v, n, n))
    g = og.distances(v, f, 0)
    assert np.isinf(g["dist"]).any()                       # the box's faces are separate parts now


def test_long_strip():
    from invesalius3_b200 import surface_geodesic as sg
    v, f = strip(200_000)
    last = int(f.max())
    s = _distances(v, f, [0])
    got = _path(v, f, np.array([v[0], v[last]], np.float64), surface=s)
    assert len(got.ids[0]) > 50_000
    s.distances(0, last)
    assert s.rounds > 50_000 // 2 and s.buckets > 1


def test_noise_surface():
    v, f = _mc(noise_volume(96, 0.12, 1))
    _distances(v, f, [0, len(v) // 2])
    for n in (2, 3, 10):
        _path(v, f, _picks(v, n, n))


def test_cranium_surface(cranium):
    full = tuple(int(s) for s in cranium["full_shape"])
    mask = np.unpackbits(cranium["mask_0_bits_full"])[:np.prod(full)].reshape(full) * np.uint8(255)
    v, f = _mc(mask, tuple(float(s) for s in cranium["spacing"]))
    assert len(f) > 100_000
    _distances(v, f, [0, len(v) // 2])
    for n in (2, 3, 10):
        _path(v, f, _picks(v, n, n))


def test_phantom_surface():
    import torch
    from invesalius3_b200 import device as dev, phantom
    from invesalius3_b200 import surface_geodesic as sg
    vol = phantom.ct((512, 512, 512), seed=2)
    mask = dev.threshold(torch.from_numpy(vol).cuda(), 226, 3071).cpu().numpy()
    del vol
    v, f = _mc(mask)
    del mask
    vt, ft = _tensors(v, f)
    s = sg.GeodesicSurface(vt, ft)
    start = int(og.closest_points(v, v[:1])[0])
    want = og.distances(v, f, start)["dist"]
    assert np.array_equal(_bits(s.distances(start).cpu().numpy()), _bits(want))
    for n in (2, 3):
        _path(v, f, _picks(v, n, 10 + n), surface=s)
