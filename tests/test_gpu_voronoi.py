"""Jump flooding and the Voronoi scaffolds on the device (invesalius3_b200.voronoi) against the C checker
(oracle/voronoi.c) and the NumPy / SciPy restatement of the plugin (oracle/voronoi.py), with
np.array_equal; the float32 gaussian_filter against SciPy directly."""
import numpy as np
import pytest
from scipy import ndimage as ndi

from oracle import voronoi as ov

pytestmark = pytest.mark.gpu


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)


def _both(dist, own, sites, normalize):
    """Run the device and the checker on copies of the same inputs; assert equal outputs."""
    from invesalius3_b200 import voronoi
    d1, o1, d2, o2 = dist.copy(), own.copy(), dist.copy(), own.copy()
    voronoi.jump_flooding(d1, o1, sites, normalize)
    ov.jump_flooding(d2, o2, sites, normalize)
    assert _same(o1, o2), (dist.shape, len(sites), normalize)
    assert _same(d1, d2), (dist.shape, len(sites), normalize)
    return d1, o1


def _random_sites(rng, shape, n):
    return rng.integers((0, 0, 0), shape, size=(n, 3)).astype(np.int32)


@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("shape, n", [((7, 9, 11), 5), ((1, 64, 97), 40), ((3, 40, 33), 25), ((256, 256, 256), 1000)])
def test_jump_flooding_shapes(shape, n, normalize):
    rng = np.random.default_rng(n)
    _, own = _both(np.zeros(shape, np.float32), np.zeros(shape, np.int32), _random_sites(rng, shape, n), normalize)
    assert own.min() >= 0


@pytest.mark.parametrize("normalize", [False, True])
def test_jump_flooding_256x512x512(normalize):
    shape = (256, 512, 512)
    _both(np.zeros(shape, np.float32), np.zeros(shape, np.int32), _random_sites(np.random.default_rng(5), shape, 5000),
          normalize)


@pytest.mark.parametrize("normalize", [False, True])
def test_jump_flooding_bad_and_duplicate_sites(normalize):
    rng = np.random.default_rng(11)
    shape = (9, 17, 23)
    sites = _random_sites(rng, shape, 30)
    sites[5] = sites[2]                        # duplicates: the last one wins
    sites[29] = sites[2]
    sites[7] = (-1, 3, 3)                      # negative and out of range: seed nothing
    sites[8] = (3, 17, 3)
    sites[9] = (3, 3, 23)
    sites[10] = (2 ** 31 - 1, -(2 ** 31), 0)
    _both(np.zeros(shape, np.float32), np.zeros(shape, np.int32), sites, normalize)
    # a pre-filled owner may name a site that seeded nothing: its coordinates are still used
    own = np.zeros(shape, np.int32)
    own[4, 8, 11] = 8
    own[0, 0, 0] = 11
    _both(np.zeros(shape, np.float32), own, sites, normalize)


@pytest.mark.parametrize("normalize", [False, True])
def test_jump_flooding_one_and_no_site(normalize):
    from invesalius3_b200 import voronoi
    shape = (16, 16, 16)
    d, o = _both(np.zeros(shape, np.float32), np.zeros(shape, np.int32), np.array([[3, 12, 5]], np.int32), normalize)
    assert (o == 1).all()
    for sites in (np.zeros((0, 3), np.int32), np.zeros((0, 1), np.int32)):
        dist, own = np.full(shape, 2.5, np.float32), np.full(shape, 4, np.int32)
        voronoi.jump_flooding(dist, own, sites, normalize)
        assert (dist == 2.5).all() and (own == 4).all()
    for sz in ((1, 1, 1), (2, 1, 1)):                 # zero and one steps
        _both(np.full(sz, 7.0, np.float32), np.full(sz, 3, np.int32), np.array([[0, 0, 0], [1, 0, 0]], np.int32),
              normalize)


@pytest.mark.parametrize("normalize", [False, True])
def test_jump_flooding_prefilled(normalize):
    rng = np.random.default_rng(21)
    shape = (12, 31, 26)
    n = 20
    for lo, hi in ((-5, n + 6), (n + 1, n + 50)):
        own = rng.integers(lo, hi, size=shape).astype(np.int32)
        dist = (rng.random(shape) * 40).astype(np.float32)
        dist[rng.random(shape) < 0.05] = np.inf
        _both(dist, own, _random_sites(rng, shape, n), normalize)


def test_jump_flooding_strided_views():
    from invesalius3_b200 import voronoi
    rng = np.random.default_rng(31)
    shape = (10, 33, 40)
    sites = np.zeros((15, 5), np.int32)
    sites[:, :3] = _random_sites(rng, shape, 15)
    sites[:, 3:] = -7
    for normalize in (False, True):
        big_d = (rng.random((12, 35, 44)) * 3).astype(np.float32)
        big_o = rng.integers(0, 4, size=(12, 35, 44)).astype(np.int32)
        view = (slice(1, 11), slice(2, 35), slice(3, 43))
        ref_d, ref_o = big_d[view].copy(), big_o[view].copy()
        ov.jump_flooding(ref_d, ref_o, np.ascontiguousarray(sites[:, :3]), normalize)
        keep_d, keep_o = big_d.copy(), big_o.copy()
        voronoi.jump_flooding(big_d[view], big_o[view], sites, normalize)
        assert _same(big_d[view], ref_d) and _same(big_o[view], ref_o)
        keep_d[view], keep_o[view] = ref_d, ref_o
        assert _same(big_d, keep_d) and _same(big_o, keep_o)     # nothing outside the views changed
    # a view with a step along x goes through a host copy
    d = np.zeros((4, 6, 16), np.float32)
    o = np.zeros((4, 6, 16), np.int32)
    ref_d, ref_o = d[:, :, ::2].copy(), o[:, :, ::2].copy()
    s = np.array([[1, 2, 3], [3, 5, 7]], np.int32)
    ov.jump_flooding(ref_d, ref_o, s, True)
    voronoi.jump_flooding(d[:, :, ::2], o[:, :, ::2], s, True)
    assert _same(d[:, :, ::2], ref_d) and _same(o[:, :, ::2], ref_o) and not o[:, :, 1::2].any()


@pytest.mark.parametrize("border", [True, False])
@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("size", [(97, 64, 1), (40, 36, 30)])
def test_create_voronoi(size, normalize, border):
    from invesalius3_b200 import voronoi
    np.random.seed(123)
    want = ov.create_voronoi(*size, 60, normalize, border)
    next_want = np.random.randint(1 << 30)
    np.random.seed(123)
    got = voronoi.create_voronoi(*size, 60, normalize, border)
    assert _same(got, want)
    assert np.random.randint(1 << 30) == next_want     # the global RNG advanced identically


@pytest.mark.parametrize("border", [True, False])
@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("args", [(80, 70, 3, 6, 5, 1), (48, 40, 1, 7, 6, 1), (36, 32, 28, 4, 3, 3)])
def test_create_voronoi_non_random(args, normalize, noise, border):
    from invesalius3_b200 import voronoi
    np.random.seed(7)
    want = ov.create_voronoi_non_random(*args, normalize, noise, border)
    np.random.seed(7)
    got = voronoi.create_voronoi_non_random(*args, normalize, noise, border)
    assert _same(got, want)


def test_create_voronoi_default_size():
    """The tool's default: 256^3 with 1000 sites, borders on, through image_normalize as gui.py:237 does."""
    from invesalius3_b200 import voronoi
    np.random.seed(2024)
    want = ov.create_voronoi()
    np.random.seed(2024)
    got = voronoi.create_voronoi()
    assert _same(got, want)
    assert _same(voronoi.image_normalize(got, min_=-1000, max_=1000), ov.image_normalize(want, min_=-1000, max_=1000))


def test_image_normalize():
    from invesalius3_b200 import voronoi
    rng = np.random.default_rng(41)
    a = (rng.standard_normal((20, 33, 17)) * 3).astype(np.float32)
    for lo, hi in ((-1000, 1000), (0, 255), (0.0, 1.0), (-3.7, 1234.56), (100, -100)):
        assert _same(voronoi.image_normalize(a, lo, hi), ov.image_normalize(a, lo, hi)), (lo, hi)
    sl = a[3]
    assert _same(voronoi.image_normalize(sl, 0, 255), ov.image_normalize(sl, 0, 255))      # np2bitmap, gui.py:28
    assert _same(voronoi.image_normalize(a[:, ::3, 1:], -1000, 1000), ov.image_normalize(a[:, ::3, 1:], -1000, 1000))
    for fill in (np.full((4, 5, 6), 0.75, np.float32), np.zeros((7, 8), np.float32)):
        for lo in (-1000, 0, 2.9, -2.9):
            got = voronoi.image_normalize(fill, lo, 1000)
            assert _same(got, ov.image_normalize(fill, lo, 1000)) and (got == int(lo)).all()


def test_device_api_errors():
    import torch
    from invesalius3_b200 import voronoi
    d = torch.zeros((4, 5, 6), dtype=torch.float32, device="cuda")
    o = torch.zeros((4, 5, 6), dtype=torch.int32, device="cuda")
    s = torch.zeros((2, 3), dtype=torch.int32, device="cuda")
    with pytest.raises(TypeError):
        voronoi.jump_flooding_device(d.double(), o, s, False)
    with pytest.raises(TypeError):
        voronoi.jump_flooding_device(d, o.long(), s, False)
    with pytest.raises(TypeError):
        voronoi.jump_flooding_device(d, o, s.long(), False)
    with pytest.raises(ValueError):
        voronoi.jump_flooding_device(d, o[:, :4].contiguous(), s, False)
    with pytest.raises(ValueError):
        voronoi.jump_flooding_device(d, o, s[:, :2].contiguous(), False)
    with pytest.raises(ValueError):
        voronoi.jump_flooding_device(d, o[:, :, ::2], s, False)
    with pytest.raises(ValueError, match="too small"):
        voronoi.voronoi_borders_device(o[:, :1].contiguous())
    with pytest.raises(ValueError, match="too small"):
        voronoi.voronoi_borders_device(torch.zeros((1, 5, 1), dtype=torch.int32, device="cuda"))
    ro_d, ro_o = np.zeros((2, 3, 4), np.float32), np.zeros((2, 3, 4), np.int32)
    ro_d.flags.writeable = False
    with pytest.raises(ValueError):
        voronoi.jump_flooding(ro_d, ro_o, np.zeros((1, 3), np.int32), False)


@pytest.mark.parametrize("shape", [(1, 64, 97), (1, 5, 300), (9, 40, 33), (2, 3, 4), (60, 70, 50)])
def test_gaussian_filter_float32(shape):
    """filters._gaussian on float32 equals ndimage.gaussian_filter(x.astype(float32), 1.5), including the z
    pass SciPy still runs (over reflected taps) when nz == 1."""
    import torch
    from invesalius3_b200 import device as dev, filters
    rng = np.random.default_rng(sum(shape))
    x = (rng.random(shape) > 0.7).astype(np.float32)
    x[0, 0, :2] = (1e-7, 3.3)
    for sigma in (1.5, 0.7):
        want = ndi.gaussian_filter(x, sigma)
        assert _same(filters._gaussian(dev.to_device(x), sigma, torch.float32).cpu().numpy(), want)
