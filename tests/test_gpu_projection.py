"""GPU MIDA / LMIP / contour-MIP vs the oracle restatement of invesalius_rs/src/mips.rs
(parity unpinned: the reference has no test for these). MIDA and LMIP must be bit-exact
(same float32 operation order, no FMA). Contour-MIP goes through powf, where libm (the
reference) and the device differ by at most one ulp on rare inputs: the int-typed results
may then differ by one unit on a tiny fraction of pixels — tolerance stated in the test."""
import numpy as np
import pytest
from scipy import ndimage

pytestmark = pytest.mark.gpu

SHAPES = [(1, 1, 1), (2, 3, 5), (7, 9, 11), (33, 40, 70), (40, 130, 37)]


@pytest.fixture(scope="module")
def rs():
    from invesalius3_b200 import device, invesalius_rs
    device.require_cuda()
    return invesalius_rs


def _ct_like(shape, seed):
    rng = np.random.default_rng(seed)
    f = ndimage.gaussian_filter(rng.normal(size=shape), 1.0) if min(shape) > 2 else rng.normal(size=shape)
    f = f / (np.abs(f).max() + 1e-9)
    return (f * 1500 + 200 + rng.normal(0, 20, shape)).astype(np.int16)


def _oshape(shape, axis):
    return [(shape[1], shape[2]), (shape[0], shape[2]), (shape[0], shape[1])][axis]


@pytest.mark.parametrize("shape", SHAPES[1:])
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_mida_i16_bit_exact(rs, orc, shape, axis):
    img = _ct_like(shape, 1)
    for wl, ww in [(300, 300), (-18, 406), (40, 1), (3000, 30000)]:
        want = np.zeros(_oshape(shape, axis), np.int16); got = want.copy()
        orc.mida(img, axis, wl, ww, want)
        rs.mida(img, axis, wl, ww, got)
        assert np.array_equal(got, want), (shape, axis, wl, ww, int((got != want).sum()))


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_mida_u8_f64_and_strided(rs, orc, axis):
    rng = np.random.default_rng(3)
    img8 = rng.integers(0, 256, (9, 20, 45)).astype(np.uint8)
    want = np.zeros(_oshape(img8.shape, axis), np.uint8); got = want.copy()
    orc.mida(img8, axis, 120, 80, want); rs.mida(img8, axis, 120, 80, got)
    assert np.array_equal(got, want)
    f = rng.random((9, 20, 45)) * 255.0
    want = np.zeros(_oshape(f.shape, axis), np.uint8); got = want.copy()
    orc.mida(f, axis, 120, 80, want); rs.mida(f, axis, 120, 80, got)
    assert np.array_equal(got, want)
    # a strided slab view, as Slice.get_image_slice passes for CORONAL / SAGITAL (slice_.py:947,1034)
    big = _ct_like((20, 30, 40), 5)
    view = big[:, 5:12, :]
    want = np.zeros(_oshape(view.shape, axis), np.int16); got = want.copy()
    orc.mida(view, axis, 300, 300, want); rs.mida(view, axis, 300, 300, got)
    assert np.array_equal(got, want)


def test_mida_errors(rs):
    img = _ct_like((5, 6, 7), 0)
    with pytest.raises(TypeError):
        rs.mida(img, 0, 300, 300, np.zeros((6, 7), np.uint8))        # dtype pair not offered
    with pytest.raises(TypeError):
        rs.mida(img.astype(np.float32), 0, 300, 300, np.zeros((6, 7), np.int16))
    with pytest.raises(OverflowError):
        rs.mida(img, 0, 40000, 300, np.zeros((6, 7), np.int16))      # wl extracted as i16
    with pytest.raises(ValueError):
        rs.mida(np.full((3, 4, 5), 7, np.int16), 0, 300, 300, np.zeros((4, 5), np.int16))  # range 0 -> NaN panic
    with pytest.raises(ValueError):
        rs.mida(img, 0, 300, 300, np.zeros((7, 6), np.int16))


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_lmip_bit_exact(rs, orc, shape, axis):
    img = _ct_like(shape, 2)
    for tmin, tmax in [(700, 3033), (-100, 100), (5000, 6000)]:
        want = np.zeros(_oshape(shape, axis), np.int16); got = want.copy()
        orc.lmip(img, axis, tmin, tmax, want)
        rs.lmip(img, axis, tmin, tmax, got)
        assert np.array_equal(got, want), (shape, axis, tmin, tmax)
    f = img.astype(np.float64) * 0.5
    want = np.zeros(_oshape(shape, axis), np.float64); got = want.copy()
    orc.lmip(f, axis, 100.0, 900.0, want); rs.lmip(f, axis, 100.0, 900.0, got)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("tmip", [0, 1, 2])
def test_fast_countour_mip(rs, orc, axis, tmip):
    shape = (24, 40, 56)
    img = _ct_like(shape, 4)
    for n in (1.0, 2.0, 0.35):
        want = np.zeros(_oshape(shape, axis), np.int16); got = want.copy()
        orc.fast_countour_mip(img, n, axis, 300, 300, tmip, want)
        rs.fast_countour_mip(img, n, axis, 300, 300, tmip, got)
        diff = np.abs(got.astype(np.int64) - want.astype(np.int64))
        if tmip == 0:
            # max of the contour volume: a 1-ulp powf difference moves a truncated value by
            # at most one unit, on rare pixels
            assert diff.max() <= 1 and (diff != 0).mean() <= 2e-3, (n, diff.max(), (diff != 0).mean())
        else:
            # LMIP / MIDA over the contour volume are discontinuous in their input, so one
            # differing sample can move a pixel further; it must stay a rare event
            assert (diff != 0).mean() <= 2e-3, (n, (diff != 0).mean())


def test_fast_countour_mip_n1_exact(rs, orc):
    """n == 1: pow(x, 1) is exact in every libm, so the whole pipeline must be bit-exact."""
    img = _ct_like((20, 33, 47), 6)
    for axis in (0, 1, 2):
        for tmip in (0, 1, 2):
            want = np.zeros(_oshape(img.shape, axis), np.int16); got = want.copy()
            orc.fast_countour_mip(img, 1.0, axis, 300, 300, tmip, want)
            rs.fast_countour_mip(img, 1.0, axis, 300, 300, tmip, got)
            assert np.array_equal(got, want), (axis, tmip)
    u8 = np.random.default_rng(1).integers(0, 256, (10, 12, 40)).astype(np.uint8)
    want = np.zeros((12, 40), np.uint8); got = want.copy()
    orc.fast_countour_mip(u8, 1.0, 0, 100, 50, 0, want)
    rs.fast_countour_mip(u8, 1.0, 0, 100, 50, 0, got)
    assert np.array_equal(got, want)
    with pytest.raises((ValueError, OverflowError)):
        rs.fast_countour_mip(u8, 1.0, 0, 100, 50, 1, got)  # 700 does not fit u8: reference panics


def test_fcm_volume_and_float64(rs, orc):
    """The contour volume itself (mips.rs:236-242) against the oracle's, every dtype the reference
    dispatches (int16, uint8, float64), shapes with partial 64 x 8 columns and a single plane; the
    float64 projections (mips_py.rs:240-251) for tmip 0 / 1."""
    import torch
    from invesalius3_b200 import projection
    for shape in ((20, 33, 47), (1, 9, 70), (5, 8, 64), (3, 70, 5)):
        img = _ct_like(shape, 9)
        for a in (img, (img // 16 + 64).clip(0, 255).astype(np.uint8), img.astype(np.float64) * 0.37):
            for axis in (0, 1, 2):
                got = projection.fcm_volume(torch.from_numpy(a).cuda(), 1.0, axis).cpu().numpy()
                assert np.array_equal(got, orc.fcm_volume(a, 1.0, axis)), (shape, a.dtype, axis)
    f = _ct_like((20, 33, 47), 6).astype(np.float64) * 0.75
    for axis in (0, 1, 2):
        for tmip in (0, 1):
            want = np.zeros(_oshape(f.shape, axis), np.float64); got = want.copy()
            orc.fast_countour_mip(f, 1.0, axis, 300, 300, tmip, want)
            rs.fast_countour_mip(f, 1.0, axis, 300, 300, tmip, got)
            assert np.array_equal(got, want), (axis, tmip)
    with pytest.raises(NotImplementedError):
        rs.fast_countour_mip(f, 1.0, 0, 300, 300, 2, np.zeros(_oshape(f.shape, 0), np.float64))


def test_mida_1024_slab_properties():
    """Large input: MIDA of a volume whose rays all saturate in the first slice equals that slice."""
    import torch
    from invesalius3_b200 import projection
    g = torch.Generator(device="cuda").manual_seed(1)
    t = torch.randint(1000, 2000, (64, 512, 512), dtype=torch.int16, device="cuda", generator=g)
    t[0, 0, 0] = -1000  # fixes the range; every other first sample has opacity 1 (wl=0, ww=2)
    for axis in (0, 1, 2):
        out = projection.mida(t, axis, 0, 2)
        first = [t[0], t[:, 0], t[:, :, 0]][axis]
        # alpha = 1 at the first sample => colour = fpi; out = trunc(range*fpi + min) within 1 of v
        diff = (out.to(torch.int32) - first.to(torch.int32)).abs()
        diff[0, 0] = 0  # the ray through the planted -1000 voxel does not saturate at once
        assert int(diff.max()) <= 1, axis


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_mida_wide_value_range_and_foreign_minmax(rs, orc, axis):
    """A volume spanning far more than a CT's ~4k values, and a caller-supplied (min, max) that
    does not bound the data (integer and float64 inputs of equal values must then agree)."""
    import torch
    from invesalius3_b200 import projection
    shape = (21, 34, 70)
    wide = (_ct_like(shape, 9).astype(np.int32) * 9).clip(-32768, 32767).astype(np.int16)
    assert int(wide.max()) - int(wide.min()) > 4096
    want = np.zeros(_oshape(shape, axis), np.int16); got = want.copy()
    orc.mida(wide, axis, 300, 2000, want); rs.mida(wide, axis, 300, 2000, got)
    assert np.array_equal(got, want)
    # supplying the true extrema is the same as letting the kernel find them
    img = _ct_like(shape, 10)
    lo, hi = int(img.min()), int(img.max())
    t = torch.from_numpy(img).cuda()
    full = projection.mida(t, axis, 300, 300)
    mm = torch.tensor([float(lo), float(hi)], dtype=torch.float32, device="cuda")
    assert torch.equal(projection.mida(t, axis, 300, 300, minmax=mm), full)
    # forced extrema narrower than the data: integer and float64 inputs of the same values agree
    u8 = np.random.default_rng(11).integers(0, 256, shape).astype(np.uint8)
    t8 = torch.from_numpy(u8).cuda()
    t64 = t8.to(torch.float64)
    for pair in [(20.0, 235.0), (0.0, 255.0), (60.0, 61.0)]:
        mm2 = torch.tensor(pair, dtype=torch.float32, device="cuda")
        outcome = []
        for vol in (t8, t64):
            try:
                outcome.append(projection.mida(vol, axis, 120, 80, minmax=mm2).cpu())
            except ValueError:
                outcome.append(None)
        if outcome[0] is None or outcome[1] is None:
            assert outcome[0] is None and outcome[1] is None, pair
        else:
            assert torch.equal(outcome[0], outcome[1]), pair


@pytest.mark.parametrize("dtype", [np.int16, np.uint8, np.float64])
def test_rays_along_z_in_stretches(rs, orc, dtype):
    """b2v_mida_z_partial / b2v_lmip_z_partial: a ray walked slab by slab with its state handed
    on equals the whole-volume walk bit for bit (the Z-sharded axis-0 projections, here on one
    device, cut at uneven planes including a one-plane slab)."""
    import torch
    from invesalius3_b200 import device as dev, projection
    shape = (23, 19, 150)
    if dtype == np.int16:
        vol = _ct_like(shape, 21)
        windows, ranges = [(300, 600), (40, 1), (3000, 30000)], [(700, 3033), (-200, 100)]
    elif dtype == np.uint8:
        vol = np.random.default_rng(22).integers(0, 256, shape).astype(np.uint8)
        windows, ranges = [(120, 80), (10, 250)], [(100, 200), (0, 255)]
    else:
        vol = np.random.default_rng(23).random(shape) * 255.0
        windows, ranges = [(120, 80)], [(100.5, 200.25)]
    t = torch.from_numpy(vol).cuda()
    cuts = [0, 5, 6, 17, 23]
    bad = []
    mm = dev.minmax(t)
    for wl, ww in windows:
        odt = np.uint8 if dtype == np.float64 else dtype
        want = np.zeros(shape[1:], odt)
        orc.mida(vol, 0, wl, ww, want)
        state = projection.ray_state(t)
        got = None
        for i in range(len(cuts) - 1):
            got = projection.mida_z_partial(t[cuts[i]:cuts[i + 1]].contiguous(), wl, ww, mm, state, i == 0,
                                            i == len(cuts) - 2)
        if not np.array_equal(got.cpu().numpy(), want):
            bad.append(("mida", wl, ww, int((got.cpu().numpy() != want).sum())))
        whole = projection.mida_z_partial(t, wl, ww, mm, projection.ray_state(t), True, True)
        if not np.array_equal(whole.cpu().numpy(), want):
            bad.append(("mida-one-stretch", wl, ww))
    for tmin, tmax in ranges:
        want = np.zeros(shape[1:], dtype)
        orc.lmip(vol, 0, tmin, tmax, want)
        state = projection.ray_state(t)
        got = None
        for i in range(len(cuts) - 1):
            got = projection.lmip_z_partial(t[cuts[i]:cuts[i + 1]].contiguous(), tmin, tmax, state, i == 0,
                                            i == len(cuts) - 2)
        if not np.array_equal(got.cpu().numpy(), want):
            bad.append(("lmip", tmin, tmax, int((got.cpu().numpy() != want).sum())))
    assert not bad, bad


def test_projections_1024_slab_exact(orc):
    """One 64-plane slab of BASELINE config 3 (64 x 1024 x 1024) against the CPU checker / NumPy,
    exactly: MaxIP on the three axes, MIDA and LMIP with rays along every axis."""
    import torch
    from invesalius3_b200 import device as dev, phantom, projection
    vol = phantom.ct((64, 1024, 1024), seed=3)
    t = torch.from_numpy(vol).cuda()
    for axis in (0, 1, 2):
        assert np.array_equal(dev.mip(t, axis, "max").cpu().numpy(), vol.max(axis)), axis
        want = np.zeros(_oshape(vol.shape, axis), np.int16)
        orc.mida(vol, axis, 300, 300, want)
        assert np.array_equal(projection.mida(t, axis, 300, 300).cpu().numpy(), want), ("mida", axis)
        orc.lmip(vol, axis, 700, 3033, want)
        assert np.array_equal(projection.lmip(t, axis, 700, 3033).cpu().numpy(), want), ("lmip", axis)


def test_rays_along_x_partial_blocks(orc):
    """Rays along x equal the oracle bit for bit for MIDA (early exit and full rays) and LMIP, on
    row counts that do not fill the last block of 128 rays and tails shorter than a 32-sample tile."""
    import torch
    from invesalius3_b200 import projection
    for shape in ((9, 37, 200), (4, 33, 64), (3, 5, 72)):
        vol = _ct_like(shape, 21)
        t = torch.from_numpy(vol).cuda()
        want = np.zeros(_oshape(shape, 2), np.int16)
        for wl, ww in ((300, 300), (32000, 2)):
            orc.mida(vol, 2, wl, ww, want)
            assert np.array_equal(projection.mida(t, 2, wl, ww).cpu().numpy(), want), (shape, wl, ww)
        orc.lmip(vol, 2, 700, 3033, want)
        assert np.array_equal(projection.lmip(t, 2, 700, 3033).cpu().numpy(), want), shape
