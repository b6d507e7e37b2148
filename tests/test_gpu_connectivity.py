"""The surface connectivity tools on the device (invesalius3_b200.surface_connectivity) against the C checker
(oracle/connectivity.c), bit for bit: region ids, sizes, PointMap, and the vertices (as uint32), faces and
ids of all three tools in the VTK and the compact form."""
import numpy as np
import pytest

from connectivity_meshes import dense_random, fan, noise_volume, shuffled_spheres, strip
from oracle import connectivity as oc

pytestmark = pytest.mark.gpu


def _form(f, dtype, cols):
    f = f.astype(dtype)
    if cols == 4:
        f = np.concatenate([np.full((len(f), 1), 3, dtype), f], 1)
    return f


def _same_part(got, want, cols):
    gv, gf, gp, gc = (t.cpu().numpy() for t in got)
    wv, wf, wp, wc = want
    if cols == 4:
        assert (gf[:, 0] == 3).all()
        gf = gf[:, 1:]
    assert np.array_equal(gv.view(np.uint32), wv.view(np.uint32))
    assert np.array_equal(gf, wf) and np.array_equal(gp, wp) and np.array_equal(gc, wc)


def _run(v, f, seeds=None, dtype=np.int32, cols=3, parts=True):
    """Device state and tools against the checker on the same arrays; returns the checker's state."""
    import torch
    from invesalius3_b200 import surface_connectivity as sc
    ff = _form(f, dtype, cols)
    vt, ft = torch.from_numpy(np.ascontiguousarray(v)).cuda(), torch.from_numpy(np.ascontiguousarray(ff)).cuda()
    st = oc.traverse(len(v), f, seeds)
    c = sc.connectivity_device(vt, ft, seeds)
    assert np.array_equal(c.region.cpu().numpy(), st["region"])
    assert np.array_equal(c.point_map.cpu().numpy(), st["point_map"])
    assert np.array_equal(c.sizes.cpu().numpy(), st["sizes"])
    assert c.depth == st["depth"]
    assert c.largest == (int(np.argmax(st["sizes"])) if len(st["sizes"]) and st["sizes"].max() > 0 else -1)
    if not parts:
        return st
    for compact in (False, True):
        if seeds is None:
            _same_part(sc.select_largest_part_device(vt, ft, compact), oc.select_largest_part(v, f, compact), cols)
            got = sc.split_disconnected_parts_device(vt, ft, compact)
            want = oc.split_disconnected_parts(v, f, compact)
            assert len(got) == len(want)
            if not want:
                continue
            # every part at once: the VTK form shares one point set, which is compared once
            if compact:
                gv, gp = torch.cat([g[0] for g in got]), torch.cat([g[2] for g in got])
                wv, wp = np.concatenate([w[0] for w in want]), np.concatenate([w[2] for w in want])
            else:
                assert all(g[0] is got[0][0] and g[2] is got[0][2] for g in got)
                gv, gp, wv, wp = got[0][0], got[0][2], want[0][0], want[0][2]
            _same_part((gv, torch.cat([g[1] for g in got]), gp, torch.cat([g[3] for g in got])),
                       (wv, np.concatenate([w[1] for w in want]), wp, np.concatenate([w[3] for w in want])), cols)
            assert [len(g[1]) for g in got] == [len(w[1]) for w in want]
            assert [len(g[0]) for g in got] == [len(w[0]) for w in want]
        else:
            _same_part(sc.join_seeds_parts_device(vt, ft, seeds, compact), oc.join_seeds_parts(v, f, seeds, compact),
                       cols)
    return st


MESHES = {
    "dense": lambda: dense_random(400, 12, 1),
    "dense_many": lambda: dense_random(3000, 2000, 2),
    "spheres": lambda: shuffled_spheres(9, 3),
    "fan": lambda: fan(5000),
    "strip": lambda: strip(301),
}


@pytest.mark.parametrize("name", list(MESHES))
@pytest.mark.parametrize("dtype,cols", [(np.int32, 3), (np.int64, 3), (np.int32, 4), (np.int64, 4)])
def test_small_meshes(name, dtype, cols):
    v, f = MESHES[name]()
    _run(v, f, dtype=dtype, cols=cols)
    rng = np.random.default_rng(len(f))
    _run(v, f, seeds=[int(s) for s in rng.integers(-2, len(v), 5)], dtype=dtype, cols=cols)


def test_seeds_and_empty():
    import torch
    from invesalius3_b200 import surface_connectivity as sc
    v, f = shuffled_spheres(6, 7)
    unused = int(np.setdiff1d(np.arange(len(v)), f.reshape(-1))[0])
    for seeds in ([unused], [], [-3], [-1, int(f[5, 1]), int(f[90, 0]), int(f[5, 1])]):
        _run(v, f, seeds=seeds)
    vo, fo, pids, cids = sc.join_seeds_parts(v, f, [unused])
    assert vo.shape == (0, 3) and fo.shape == (0, 3) and len(pids) == len(cids) == 0
    with pytest.raises(ValueError):
        sc.join_seeds_parts(v, f, [len(v)])
    with pytest.raises(ValueError, match="index"):
        sc.select_largest_part(v, np.concatenate([f, [[0, 1, len(v)]]]).astype(np.int32))
    bad = _form(f, np.int64, 4)
    bad[3, 0] = 4
    with pytest.raises(ValueError):
        sc.split_disconnected_parts(v, bad)
    e = np.zeros((0, 3), np.int32)
    assert sc.split_disconnected_parts(v, e) == []
    vo, fo, _, _ = sc.select_largest_part(v, e)
    assert vo.shape == (0, 3) and fo.shape == (0, 3)
    vo, fo, _, _ = sc.join_seeds_parts(np.zeros((0, 3), np.float32), e, [])
    assert vo.shape == (0, 3)
    c = sc.connectivity_device(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda())
    assert int(c.sizes.sum()) == len(f)


def test_numpy_entries_keep_dtype_and_form():
    from invesalius3_b200 import surface_connectivity as sc
    v, f = shuffled_spheres(5, 11)
    f4 = _form(f, np.int64, 4)
    vo, fo, pids, cids = sc.select_largest_part(v, f4, compact=True)
    wv, wf, wp, wc = oc.select_largest_part(v, f, compact=True)
    assert fo.dtype == np.int64 and fo.shape[1] == 4 and np.array_equal(fo[:, 1:], wf)
    assert np.array_equal(vo, wv) and np.array_equal(pids, wp) and np.array_equal(cids, wc)
    parts = sc.split_disconnected_parts(v, f)
    assert len(parts) == 5 and all(p[1].dtype == np.int32 for p in parts)


def test_long_strip():
    v, f = strip(200_000)
    st = _run(v, f, seeds=[0], parts=False)
    assert st["depth"] > 60_000
    st = _run(v, f, seeds=[len(v) // 2, 0])
    _run(v, f)


def test_noise_surface_many_regions():
    import torch
    from invesalius3_b200.mesh import marching_cubes
    mask = noise_volume(160, 0.03, 5)
    V, F = marching_cubes(torch.from_numpy(mask).cuda(), 127, (1.0, 1.0, 1.0), (0, 0, 0), True)
    st = _run(V.cpu().numpy(), F.cpu().numpy())
    assert len(st["sizes"]) > 80_000


def test_cranium_bone_surface(cranium):
    import torch
    from invesalius3_b200.mesh import marching_cubes
    full = tuple(int(s) for s in cranium["full_shape"])
    mask = np.unpackbits(cranium["mask_0_bits_full"])[:np.prod(full)].reshape(full) * np.uint8(255)
    sx, sy, sz = (float(s) for s in cranium["spacing"])
    V, F = marching_cubes(torch.from_numpy(mask).cuda(), 127, (sx, sy, sz), (0, 0, 0), True)
    v, f = V.cpu().numpy(), F.cpu().numpy()
    assert len(f) > 100000
    st = _run(v, f)
    assert len(st["sizes"]) > 1
    _run(v, f, seeds=[int(f[len(f) // 2, 0])])


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
    st = _run(v, f, parts=False)
    from invesalius3_b200 import surface_connectivity as sc
    for compact in (False, True):
        _same_part(sc.select_largest_part_device(V, F, compact), oc.select_largest_part(v, f, compact), 3)
    _run(v, f, seeds=[int(f[0, 0]), int(f[-1, 2])], parts=False)
    assert len(f) > 5_000_000 and len(st["sizes"]) >= 1
