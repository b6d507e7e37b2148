"""The surface clean and triangle filter on the device (invesalius3_b200.surface_clean) against the C checker
(oracle/clean.c), bit for bit: points, point_ids, every cell array and cell_ids, in every input form. Also the
invariant that cleaning a surface split by compute_normals gives back the pre-split mesh, and the
context-aware smoothing branch (normals -> clean -> ca_smoothing) against the checker chain."""
import numpy as np
import pytest

from connectivity_meshes import noise_volume, strip
from oracle import clean as oc
from test_oracle_clean import CASES, POLY_KINDS, POLY_SIZES, _strip_pairs, grid_points, polygon

pytestmark = pytest.mark.gpu

FORMS = [(np.int32, 3), (np.int64, 3), (np.int32, 4), (np.int64, 4), (np.int32, 0), (np.int64, 0)]


def _form(f, dtype, cols):
    """faces [T,3] in the form (dtype, cols); cols 0: an (offsets, connectivity) pair"""
    f = np.asarray(f).astype(dtype).reshape(-1, 3)
    if cols == 0:
        return np.arange(0, 3 * len(f) + 1, 3, dtype=np.int64), f.reshape(-1)
    if cols == 4:
        f = np.concatenate([np.full((len(f), 1), 3, dtype), f], 1)
    return f


def _dev(x):
    import torch
    if x is None:
        return None
    if isinstance(x, tuple):
        return tuple(_dev(a) for a in x)
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _pair_np(x):
    """a result's cell array as an int64 (offsets, connectivity) pair"""
    if isinstance(x, tuple):
        return x[0].cpu().numpy(), x[1].cpu().numpy().astype(np.int64)
    return oc.cell_array(x.cpu().numpy())


def check_clean(P, polys, strips=None):
    from invesalius3_b200 import surface_clean as sc
    want = oc.clean_polydata(P, polys, strips)
    got = sc.clean_polydata_device(_dev(P), _dev(polys), _dev(strips))
    assert np.array_equal(got.points.cpu().numpy().view(np.uint32), want["points"].view(np.uint32))
    assert np.array_equal(got.point_ids.cpu().numpy(), want["point_ids"])
    assert np.array_equal(got.cell_ids.cpu().numpy(), want["cell_ids"])
    for k in ("verts", "lines", "polys", "strips"):
        g, w = _pair_np(getattr(got, k)), want[k]
        assert np.array_equal(g[0], w[0]) and np.array_equal(g[1], w[1]), k
    if polys is not None and not isinstance(polys, tuple) and len(want["polys"][1]) == 3 * (len(want["polys"][0]) - 1):
        assert got.polys.dtype == _dev(polys).dtype and got.polys.shape[1] == polys.shape[1]
    return got, want


def check_triangles(P, polys, strips=None):
    from invesalius3_b200 import surface_clean as sc
    want = oc.triangle_filter(P, polys, strips)
    got = sc.triangle_filter_device(_dev(P), _dev(polys), _dev(strips))
    assert got.faces.dim() == 2
    assert np.array_equal(got.faces.cpu().numpy()[:, -3:], want["faces"])
    assert np.array_equal(got.cell_ids.cpu().numpy(), want["cell_ids"])
    return got


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("dtype,cols", FORMS)
def test_cases(name, dtype, cols):
    P, polys, strips = CASES[name]
    check_clean(P, _form(polys, dtype, cols), strips)
    check_triangles(P, _form(polys, dtype, cols), strips)


def test_mixed_cells_and_strips():
    P, polys, strips = _strip_pairs()
    check_clean(P, polys, strips)
    check_clean(P, None, strips)
    check_triangles(P, None, strips)
    check_triangles(P, polys, strips)


@pytest.mark.parametrize("seed", range(3))
def test_random(seed):
    rng = np.random.default_rng(seed)
    P = grid_points(3000, seed)
    P[rng.integers(0, 3000, 50)] = np.float32(np.nan)
    P[rng.integers(0, 3000, 50), 1] = np.float32(-0.0)
    f = rng.integers(0, 3000, size=(20000, 3))
    so = np.cumsum(np.r_[0, rng.integers(0, 12, 3000)]).astype(np.int64)
    strips = (so, rng.integers(0, 3000, so[-1]))
    check_clean(P, f, strips)
    check_triangles(P, f, strips)


def _pack(polys):
    """several (points, ids) polygons as one point array and one (offsets, connectivity) pair"""
    pts, conn, offs, base = [], [], [0], 0
    for P, ids in polys:
        pts.append(P)
        conn.append(ids + base)
        offs.append(offs[-1] + len(ids))
        base += len(P)
    return np.concatenate(pts), (np.array(offs, np.int64), np.concatenate(conn))


@pytest.mark.parametrize("dtype", [np.int32, np.int64])
def test_polygons_4_to_64(dtype):
    """convex and concave polygons of 4-64 points, one warp each, every kind and size in one call"""
    P, (offs, conn) = _pack([polygon(k, n, seed) for k in POLY_KINDS for n in POLY_SIZES for seed in range(3)])
    got = check_triangles(P, (offs, conn.astype(dtype)))
    assert got.faces.dtype == (_dev(conn.astype(dtype)).dtype)
    check_clean(P, (offs, conn.astype(dtype)))


def test_long_polygons_and_mixed_cells():
    """polygons past one warp's share (one block each) beside triangles and short polygons"""
    parts = [polygon(k, n, s) for k, n, s in (("comb", 300, 1), ("concave", 1000, 2), ("regular", 257, 0),
                                              ("star", 256, 3), ("convex", 2048, 4))]
    rng = np.random.default_rng(5)
    parts += [polygon(POLY_KINDS[i % 5], int(rng.integers(3, 65)), i) for i in range(3000)]
    P, polys = _pack(parts)
    got = check_triangles(P, polys)
    assert len(got.faces) > 3000


def test_malformed_and_refused():
    from invesalius3_b200 import surface_clean as sc
    P = grid_points(10)
    for offs, conn in (([1, 3], [0, 1, 2]), ([0, 2, 1, 3], [0, 1, 2]), ([0, 3], [0, 1, 2, 3])):
        with pytest.raises(ValueError):
            sc.clean_polydata(P, (np.array(offs), np.array(conn)))
        with pytest.raises(ValueError):
            sc.triangle_filter(P, None, (np.array(offs), np.array(conn)))
    with pytest.raises(ValueError):
        sc.clean_polydata(P, np.array([[0, 1, 10]]))
    with pytest.raises(ValueError):
        sc.clean_polydata(P, np.array([[3, 0, 1, 2], [4, 0, 1, 2]]))
    with pytest.raises(NotImplementedError):
        sc.clean_polydata(P, np.array([[0, 1, 2]]), verts=(np.array([0, 1]), np.array([0])))


def test_long_strip():
    v, f = strip(200_000)
    check_clean(v, f)
    tri = np.asarray(f).reshape(-1, 3)
    # the strip through the mesh's points in order, and the one-cell strip the triangles came from
    s = np.array([tri[0][0], tri[0][1]] + [t[2] for t in tri], np.int64)
    got = check_triangles(v, None, (np.array([0, len(s)]), s))
    assert len(got.faces) == len(tri)
    check_clean(v, None, (np.array([0, len(s)]), s))


def _mc(mask, spacing=(1.0, 1.0, 1.0)):
    import torch
    from invesalius3_b200.mesh import marching_cubes
    return marching_cubes(torch.from_numpy(np.ascontiguousarray(mask)).cuda(), 127, spacing, (0, 0, 0), True)


def _as_strips(f, seed=0):
    """strips of 3 to 7 points cut from the faces' connectivity in order: each is a run of surface points with
    the repeats the faces carry, so the clean keeps some as strips and reduces others, and the triangle
    filter meets odd and even strip positions"""
    conn = np.asarray(f).reshape(-1).astype(np.int64)
    sizes = np.random.default_rng(seed).integers(3, 8, len(conn) // 3 + 1)
    offs = np.concatenate([[0], np.cumsum(sizes)])
    offs = offs[offs < len(conn)]
    return np.concatenate([offs, [len(conn)]]).astype(np.int64), conn


def _presplit_expected(V, F, n):
    """Independent of the clean: the pre-split faces, oriented as the normals left them, relabelled in NumPy by
    first use of each distinct position; and those positions in that order."""
    v, f = V.cpu().numpy(), F.cpu().numpy().reshape(len(F), -1)[:, -3:]
    pts, nf = n.points.cpu().numpy(), n.faces.cpu().numpy().reshape(len(F), -1)[:, -3:]
    rows = np.ascontiguousarray(np.concatenate([v, pts])).view(np.dtype((np.void, 12))).ravel()
    _, cls = np.unique(rows, return_inverse=True)
    cv, cp = cls[:len(v)], cls[len(v):]
    assert np.array_equal(np.sort(cp[nf], 1), np.sort(cv[f], 1))   # same face, split points at their sources
    seq = cp[nf].reshape(-1)
    uniq, first = np.unique(seq, return_index=True)
    order = uniq[np.argsort(first)]
    rank = np.empty(cls.max() + 1, np.int64)
    rank[order] = np.arange(len(order))
    where = np.empty(cls.max() + 1, np.int64)
    where[cp[::-1]] = np.arange(len(cp))[::-1]
    return rank[cp[nf]], pts[where[order]], len(np.unique(cv[f]))


def _surface_checks(V, F, angles=(30.0, 80.0)):
    """V, F device tensors from marching cubes: the clean, the triangle filter, strips cut from the surface,
    and the split-and-clean invariant at each angle."""
    from invesalius3_b200 import surface_normals as sn
    v, f = V.cpu().numpy(), F.cpu().numpy()
    check_clean(v, f)
    check_triangles(v, f)
    strips = _as_strips(f)
    got, want = check_clean(v, None, strips)
    assert len(want["strips"][1]) and len(want["polys"][1])
    check_triangles(v, None, strips)
    for angle in angles:
        n = sn.compute_normals_device(V, F, angle)
        assert n.new_points > 0
        got, _ = check_clean(n.points.cpu().numpy(), n.faces.cpu().numpy())
        faces, points, distinct = _presplit_expected(V, F, n)
        assert got.points.shape[0] == distinct
        assert np.array_equal(got.points.cpu().numpy(), points)
        assert np.array_equal(got.polys.cpu().numpy().astype(np.int64), faces)


def test_noise_surface():
    V, F = _mc(noise_volume(96, 0.12, 1))
    _surface_checks(V, F)


def test_cranium_surface(cranium):
    full = tuple(int(s) for s in cranium["full_shape"])
    mask = np.unpackbits(cranium["mask_0_bits_full"])[:np.prod(full)].reshape(full) * np.uint8(255)
    V, F = _mc(mask, tuple(float(s) for s in cranium["spacing"]))
    assert len(F) > 100_000
    _surface_checks(V, F)
    for dtype, cols in FORMS:
        check_clean(V.cpu().numpy(), _form(F.cpu().numpy(), dtype, cols))


def test_phantom_surface():
    import torch
    from invesalius3_b200 import device as dev, phantom
    vol = phantom.ct((512, 512, 512), seed=2)
    mask = dev.threshold(torch.from_numpy(vol).cuda(), 226, 3071).cpu().numpy()
    del vol
    V, F = _mc(mask)
    del mask
    _surface_checks(V, F)


def test_ca_smoothing_branch(orc, cranium):
    """compute_normals_device -> clean_polydata_device -> ca_smoothing, against the checker chain"""
    from oracle import normals as on
    from invesalius3_b200 import mesh_ops, surface_clean as sc, surface_normals as sn
    full = tuple(int(s) for s in cranium["full_shape"])
    mask = np.unpackbits(cranium["mask_0_bits_full"])[:np.prod(full)].reshape(full) * np.uint8(255)
    V, F = _mc(mask, tuple(float(s) for s in cranium["spacing"]))
    p = (0.7, 3.0, 0.1, 7)
    n = sn.compute_normals_device(V, F, 30.0)
    c = sc.clean_polydata_device(n.points, n.faces)
    skip = len(c.verts[1]) + len(c.lines[1])
    cn = n.cell_normals[c.cell_ids[skip:]].cpu().numpy()
    faces = c.polys.cpu().numpy()
    F4 = np.concatenate([np.full((len(faces), 1), 3, faces.dtype), faces], 1).astype(np.int64)
    got = c.points.cpu().numpy().copy()
    mesh_ops.context_aware_smoothing(got, F4, cn, *p)

    w = on.compute_normals(V.cpu().numpy(), F.cpu().numpy(), 30.0, False)
    wc = oc.clean_polydata(w["points"], w["faces"])
    wf = wc["polys"][1].reshape(-1, 3)
    want = wc["points"].copy()
    orc.ca_smoothing(want, np.concatenate([np.full((len(wf), 1), 3, np.int64), wf], 1),
                     w["cell_normals"][wc["cell_ids"][len(wc["verts"][1]) + len(wc["lines"][1]):]], *p)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
