"""The jump-flooding checker (oracle/voronoi.c) on cases with known answers and against an independent
pure-Python restatement of floodfill.rs:298-507, the plugin restatement of oracle/voronoi.py against
NumPy itself, and the argument checks of invesalius3_b200.voronoi that are raised before any device
work. Jump flooding is approximate, so beyond these cases nothing is compared with a brute-force
Voronoi diagram."""
import math

import numpy as np
import pytest


@pytest.fixture(scope="session")
def vo():
    """The Voronoi checker (oracle/voronoi.py over oracle/voronoi.c)."""
    from oracle import voronoi
    voronoi.lib()
    return voronoi


def f32_dist(z, y, x, sz, sy, sx):
    f = np.float32
    dz, dy, dx = f(z) - f(sz), f(y) - f(sy), f(x) - f(sx)
    return np.sqrt(dz * dz + dy * dy + dx * dx)


# ----------------------------------------------------------------------------- pure-Python restatement
def py_jump_flooding(dist, owners, sites, normalize):
    """floodfill.rs:298-507 in plain Python loops with float32 scalars, in place."""
    nz, ny, nx = dist.shape
    n = len(sites)
    if n == 0 or dist.size == 0:
        return
    own, dd = owners.copy(), dist.copy()
    for i, (z, y, x) in enumerate(sites[:, :3].tolist()):
        if 0 <= z < nz and 0 <= y < ny and 0 <= x < nx:
            own[z, y, x] = i + 1
            dd[z, y, x] = 0.0
    steps = int(math.floor(math.log2(max(nz, ny, nx)))) if max(nz, ny, nx) > 1 else 0
    oz, oy, ox = nz // 2, ny // 2, nx // 2
    for _ in range(steps):
        own2, dd2 = own.copy(), dd.copy()
        for z in range(nz):
            for y in range(ny):
                for x in range(nx):
                    idx0, best = int(own[z, y, x]), dd[z, y, x]
                    for zi in (-1, 0, 1):
                        for yi in (-1, 0, 1):
                            for xi in (-1, 0, 1):
                                if zi == yi == xi == 0:
                                    continue
                                a, b, c = z + zi * oz, y + yi * oy, x + xi * ox
                                if not (0 <= a < nz and 0 <= b < ny and 0 <= c < nx):
                                    continue
                                idx1 = int(own[a, b, c])
                                if idx1 <= 0 or idx1 > n:
                                    continue
                                d1 = f32_dist(z, y, x, *sites[idx1 - 1, :3])
                                if idx0 <= 0 or d1 < best:
                                    idx0, best = idx1, d1
                    own2[z, y, x], dd2[z, y, x] = idx0, best
        own, dd = own2, dd2
        oz, oy, ox = oz // 2, oy // 2, ox // 2
    if normalize:
        cnt = [0] * n
        sums = [[0, 0, 0] for _ in range(n)]
        for (z, y, x), o in np.ndenumerate(own):
            if 0 < o <= n:
                cnt[o - 1] += 1
                for k, c in enumerate((z, y, x)):
                    sums[o - 1][k] += c
        cen = [[s // c for s in sums[i]] if c else [0, 0, 0] for i, c in enumerate(cnt)]   # sums >= 0
        mx = [np.float32(0)] * n
        for (z, y, x), o in np.ndenumerate(own):
            if 0 < o <= n:
                d = f32_dist(z, y, x, *cen[o - 1])
                dd[z, y, x] = d
                mx[o - 1] = max(mx[o - 1], d)
        for (z, y, x), o in np.ndenumerate(own):
            if 0 < o <= n and mx[o - 1] > 0:
                dd[z, y, x] = dd[z, y, x] / mx[o - 1]
    owners[...] = own
    dist[...] = dd


def _random_case(rng, shape, n_sites, prefill):
    hi = np.array(shape) + 2
    sites = rng.integers(-2, hi, size=(n_sites, 3)).astype(np.int32)
    if n_sites > 3:
        sites[-1] = sites[0]                                   # a duplicate: the last one wins
    owners = np.zeros(shape, np.int32)
    dist = np.zeros(shape, np.float32)
    if prefill:
        owners = rng.integers(-3, n_sites + 4, size=shape).astype(np.int32)
        dist = (rng.random(shape) * 20).astype(np.float32)
    return dist, owners, sites


# ----------------------------------------------------------------------------- known answers
@pytest.mark.parametrize("n", [1, 2, 4, 8, 16])
def test_one_site_power_of_two_cube(vo, n):
    rng = np.random.default_rng(n)
    for _ in range(3):
        site = rng.integers(0, n, size=3)
        dist, own = np.zeros((n, n, n), np.float32), np.zeros((n, n, n), np.int32)
        vo.jump_flooding(dist, own, site[None].astype(np.int32), False)
        assert (own == 1).all()
        want = np.array([f32_dist(*p, *site) for p in np.ndindex(n, n, n)], np.float32).reshape(dist.shape)
        assert np.array_equal(dist, want)


def test_per_axis_offsets_leave_voxels_unowned(vo):
    """(1, 1, 7): offsets 3 then 1 along x reach 0..4 only, while z and y (offset 0) visit the voxel itself."""
    dist, own = np.zeros((1, 1, 7), np.float32), np.zeros((1, 1, 7), np.int32)
    vo.jump_flooding(dist, own, np.array([[0, 0, 0]], np.int32), False)
    assert own.ravel().tolist() == [1, 1, 1, 1, 1, 0, 0]
    assert dist.ravel().tolist() == [0, 1, 2, 3, 4, 0, 0]


def test_duplicate_sites_last_wins(vo):
    dist, own = np.zeros((1, 1, 1), np.float32), np.full((1, 1, 1), 9, np.int32)
    vo.jump_flooding(dist, own, np.array([[0, 0, 0], [0, 0, 0], [5, 0, 0], [0, 0, 0], [-1, 0, 0]], np.int32), False)
    assert own.item() == 4 and dist.item() == 0.0


def test_owners_beyond_sites_are_kept(vo):
    """A pre-filled owner above n_sites is never a candidate; its voxel keeps owner and distance unless a
    strictly nearer valid neighbour appears."""
    own = np.full((1, 1, 4), 7, np.int32)
    dist = np.full((1, 1, 4), 0.25, np.float32)
    vo.jump_flooding(dist, own, np.array([[0, 0, 0]], np.int32), True)
    assert own.ravel().tolist() == [1, 7, 7, 7] and dist.ravel().tolist() == [0, 0.25, 0.25, 0.25]
    own[...] = 0
    own[0, 0, 3] = 9
    dist[...] = 5.0
    vo.jump_flooding(dist, own, np.array([[0, 0, 0]], np.int32), False)
    assert own.ravel().tolist() == [1, 1, 1, 1] and dist.ravel().tolist() == [0, 1, 2, 3]


def test_normalize_centroid_truncates(vo):
    """Centroid of x = 0..3 is 6 // 4 = 1 (not 2): distances [1, 0, 1, 2] / 2."""
    dist, own = np.zeros((1, 1, 4), np.float32), np.zeros((1, 1, 4), np.int32)
    vo.jump_flooding(dist, own, np.array([[0, 0, 0]], np.int32), True)
    assert own.ravel().tolist() == [1, 1, 1, 1]
    assert dist.ravel().tolist() == [0.5, 0.0, 0.5, 1.0]


def test_no_sites_or_empty_volume_untouched(vo):
    dist, own = np.full((2, 3, 4), 3.5, np.float32), np.full((2, 3, 4), 2, np.int32)
    vo.jump_flooding(dist, own, np.zeros((0, 3), np.int32), True)
    assert (dist == 3.5).all() and (own == 2).all()
    vo.jump_flooding(np.zeros((0, 3, 4), np.float32), np.zeros((0, 3, 4), np.int32), np.zeros((2, 3), np.int32), True)


# ----------------------------------------------------------------------------- restatement parity
@pytest.mark.parametrize("shape", [(1, 1, 7), (1, 5, 6), (3, 4, 5), (2, 7, 3), (4, 4, 4), (1, 1, 1), (5, 1, 2)])
@pytest.mark.parametrize("normalize", [False, True])
def test_checker_equals_python_restatement(vo, shape, normalize):
    rng = np.random.default_rng(hash((shape, normalize)) % 2 ** 32)
    for n_sites, prefill in ((1, False), (3, False), (6, True), (9, True)):
        dist, own, sites = _random_case(rng, shape, n_sites, prefill)
        d1, o1 = dist.copy(), own.copy()
        vo.jump_flooding(d1, o1, sites, normalize, nthreads=3)
        d2, o2 = dist.copy(), own.copy()
        py_jump_flooding(d2, o2, sites, normalize)
        assert np.array_equal(o1, o2), (shape, n_sites, prefill)
        assert np.array_equal(d1.view(np.uint32), d2.view(np.uint32)), (shape, n_sites, prefill)


def test_checker_thread_count_and_strided_views(vo):
    rng = np.random.default_rng(7)
    dist, own, sites = _random_case(rng, (9, 12, 10), 12, True)
    outs = []
    for nt in (1, 4):
        d, o = dist.copy(), own.copy()
        vo.jump_flooding(d, o, sites, True, nthreads=nt)
        outs.append((d, o))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
    big_d = np.zeros((9, 14, 13), np.float32)
    big_o = np.zeros((9, 14, 13), np.int32)
    big_d[:, 1:13, 2:12], big_o[:, 1:13, 2:12] = dist, own
    wide = np.zeros((12, 5), np.int32)
    wide[:, :3] = sites
    vo.jump_flooding(big_d[:, 1:13, 2:12], big_o[:, 1:13, 2:12], wide, True)
    assert np.array_equal(big_d[:, 1:13, 2:12], outs[0][0]) and np.array_equal(big_o[:, 1:13, 2:12], outs[0][1])
    assert (big_d[:, 0] == 0).all() and (big_o[:, :, :2] == 0).all()


# ----------------------------------------------------------------------------- plugin restatement
def test_non_random_sites_follow_meshgrid_order(vo):
    s = vo.non_random_sites(8, 6, 4, 4, 3, 2, False)
    assert s.dtype == np.int32 and s.shape == (24, 3)
    z, y, x = np.meshgrid(np.arange(2), np.arange(3), np.arange(4))
    want = np.stack(((z.ravel() + 0.5) * 2.0, (y.ravel() + 0.5) * 2.0, (x.ravel() + 0.5) * 2.0), axis=1)
    assert np.array_equal(s, want.astype(np.int32))


def test_image_normalize_restatement_is_float32():
    from oracle import voronoi as vo
    rng = np.random.default_rng(3)
    a = (rng.random((5, 6, 7)) * 3 - 1).astype(np.float32)
    got = vo.image_normalize(a, -1000, 1000)
    lo, hi = a.min(), a.max()
    want = ((a - lo) * (np.float32(2000) / (hi - lo)) + np.float32(-1000)).astype(np.int16)
    assert got.dtype == np.int16 and np.array_equal(got, want)
    assert (vo.image_normalize(np.full((3, 4), 2.5, np.float32), 7, 9) == 7).all()


# ----------------------------------------------------------------------------- argument checks (no device work)
def test_jump_flooding_argument_errors():
    from invesalius3_b200 import voronoi
    d, o, s = np.zeros((2, 3, 4), np.float32), np.zeros((2, 3, 4), np.int32), np.zeros((2, 3), np.int32)
    with pytest.raises(TypeError):
        voronoi.jump_flooding(d.astype(np.float64), o, s, False)
    with pytest.raises(TypeError):
        voronoi.jump_flooding(d, o.astype(np.int64), s, False)
    with pytest.raises(TypeError):
        voronoi.jump_flooding(d, o, s.astype(np.int64), False)
    with pytest.raises(TypeError):
        voronoi.jump_flooding(d[0], o, s, False)
    with pytest.raises(TypeError):
        voronoi.jump_flooding(d, o, s.ravel(), False)
    with pytest.raises(TypeError):
        voronoi.jump_flooding(d, o, s, 1)
    with pytest.raises(ValueError):
        voronoi.jump_flooding(d, o[:, :2], s, False)
    with pytest.raises(ValueError):
        voronoi.jump_flooding(d, o, s[:, :2], False)
    # no sites, or an empty volume: returns before the shape checks, as the crate does
    voronoi.jump_flooding(d, o[:, :2], s[:0, :2], False)
    voronoi.jump_flooding(d[:0], o, s[:, :2], False)


def test_generator_and_normalize_argument_errors():
    from invesalius3_b200 import voronoi
    for shape, grad_input in (((2, 1, 8), np.zeros((2, 1, 8))), ((1, 8, 1), np.zeros((8, 1))),
                              ((0, 8, 8), np.zeros((0, 8, 8)))):
        with pytest.raises(ValueError) as numpy_err:
            np.gradient(grad_input)
        sz, sy, sx = shape
        with pytest.raises(ValueError) as ours:
            voronoi.create_voronoi_non_random(sx, sy, sz, 2, 2, 1)
        assert str(ours.value) == str(numpy_err.value)
    with pytest.raises(ValueError):
        voronoi.create_voronoi(8, -1, 8)
    a = np.ones((3, 4), np.float32)
    with pytest.raises(NotImplementedError):
        voronoi.image_normalize(a.astype(np.float64), 0, 255)
    with pytest.raises(NotImplementedError):
        voronoi.image_normalize(a, 0, 255, np.uint8)
    with pytest.raises(NotImplementedError):
        voronoi.image_normalize(a, np.float64(0), 255)
