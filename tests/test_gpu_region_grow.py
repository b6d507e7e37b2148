"""Region growing on the device (invesalius3_b200.region_grow) against the NumPy restatement of
tests/test_region_grow_model.py: masks with np.array_equal, statistics and thresholds with == on
float64."""
import numpy as np
import pytest
from scipy.ndimage import generate_binary_structure

from test_region_grow_model import grow_3d, image_density, lut255, rg_confidence, structure

pytestmark = pytest.mark.gpu

DTYPES = [np.int16, np.uint8, np.float64]


def _phantom(shape, seed, dtype=np.int16):
    from invesalius3_b200 import phantom
    vol = phantom.ct(shape, seed=seed)
    if dtype == np.uint8:
        return np.clip(vol // 16 + 64, 0, 255).astype(np.uint8)
    if dtype == np.float64:
        return vol.astype(np.float64) * 0.37 + 0.125
    return vol


def _outcome(fn):
    """fn()'s result, or OverflowError where a threshold leaves the image's integer range (as the
    crate raises on a uint8 LUT image whose mean + mult * std passes 255)."""
    try:
        return fn()
    except OverflowError:
        return OverflowError


def _same(a, b):
    return a.dtype == b.dtype and np.array_equal(a, b, equal_nan=a.dtype.kind == "f")


# ----------------------------------------------------------------------------- LUT
@pytest.mark.parametrize("dtype", DTYPES)
def test_lut255_matches_piecewise(dtype):
    from invesalius3_b200 import region_grow as rg
    vol = _phantom((23, 41, 37), 1, dtype)
    cases = [(406, -18), (2000, 300), (1, 50), (2, 50), (0, 7), (-3, 7), (81, 50), (255, 128), (100.5, 20.25),
             (3.75, 120.0)]
    for ww, wl in cases:
        lo, hi = wl - 0.5 - (ww - 1) / 2, wl - 0.5 + (ww - 1) / 2
        v = vol.copy()
        flat = v.reshape(-1)
        for k, edge in enumerate((lo, hi, np.floor(lo), np.ceil(hi), wl)):   # voxels exactly on the edges
            flat[k * 7: k * 7 + 5] = np.asarray(edge).astype(dtype) if dtype != np.float64 else edge
        got = rg.get_LUT_value_255(v, ww, wl)
        assert _same(got, lut255(v, ww, wl)), (ww, wl)
    strided = vol[::2, 1:, ::3]
    assert _same(rg.get_LUT_value_255(strided, 406, -18), lut255(np.ascontiguousarray(strided), 406, -18))
    if dtype == np.float64:
        v = vol.copy()
        v.reshape(-1)[:4] = [np.nan, np.inf, -np.inf, -0.0]
        assert _same(rg.get_LUT_value_255(v, 406, -18), lut255(v, 406, -18))


# ----------------------------------------------------------------------------- moments
def _moments_cases(shape):
    n = int(np.prod(shape))
    return [0, 1, 2, 7, 8, 9, 127, 128, 129, 255, 256, 257, 4095, 4097, 16383, 16384, 16385, 16391, 32769, 65537,
            n // 3, n - 1, n]


@pytest.mark.parametrize("dtype", DTYPES)
def test_masked_moments_match_numpy(dtype):
    import torch
    from invesalius3_b200 import region_grow as rg
    shape = (41, 53, 67)
    vol = _phantom(shape, 3, dtype)
    rng = np.random.default_rng(11)
    t = torch.from_numpy(vol).cuda()
    n = vol.size
    for count in _moments_cases(shape):
        sel = np.zeros(n, np.uint8)
        sel[rng.choice(n, count, replace=False)] = rng.integers(128, 256, count)
        sel = sel.reshape(shape)
        m = rg.masked_moments_device(t, torch.from_numpy(sel).cuda(), "gt127")
        v = vol[sel > 127]
        assert m.count == count
        if count == 0:
            assert np.isnan(m.mean) and np.isnan(m.std)
            continue
        assert (m.min, m.max) == (v.min(), v.max()) and m.mean == np.mean(v) and m.std == np.std(v), count
    # sel == value, and the box alone / OR'd, clipped at the faces
    sel = rng.integers(0, 4, shape).astype(np.uint8)
    ts = torch.from_numpy(sel).cuda()
    for box in [(-1, -1, -1, 1, 1, 1), (39, 51, 65, 41, 53, 67), (10, 20, 30, 10, 20, 30), (5, 5, 5, 4, 9, 9),
                (-5, -5, -5, 100, 100, 100)]:
        bm = np.zeros(shape, bool)
        z0, y0, x0, z1, y1, x1 = box
        if z1 >= z0 and y1 >= y0 and x1 >= x0:
            bm[max(z0, 0): z1 + 1, max(y0, 0): y1 + 1, max(x0, 0): x1 + 1] = True
        for s, want_sel in ((ts, (sel == 1) | bm), (None, bm)):
            m = rg.masked_moments_device(t, s, "eq", 1, box)
            v = vol[want_sel]
            assert m.count == v.size, box
            if v.size:
                assert (m.min, m.max, m.mean, m.std) == (v.min(), v.max(), np.mean(v), np.std(v)), box


def test_masked_moments_whole_large_volume():
    import torch
    from invesalius3_b200 import region_grow as rg
    vol = _phantom((256, 512, 512), 2)
    t = torch.from_numpy(vol).cuda()
    full = torch.full(vol.shape, 255, dtype=torch.uint8, device="cuda")
    m = rg.masked_moments_device(t, full, "gt127")
    assert m.count == vol.size and m.mean == np.mean(vol) and m.std == np.std(vol)
    f = vol.astype(np.float64) * 0.37 + 0.125
    bone = (vol > 226).astype(np.uint8) * 200
    m = rg.masked_moments_device(torch.from_numpy(f).cuda(), torch.from_numpy(bone).cuda(), "gt127")
    v = f[bone > 127]
    assert (m.count, m.min, m.max, m.mean, m.std) == (v.size, v.min(), v.max(), np.mean(v), np.std(v))


# ----------------------------------------------------------------------------- confidence
def _seeds(shape, vol):
    dz, dy, dx = shape
    inner = np.argwhere(vol > 226)
    p = inner[len(inner) // 2]
    return [(int(p[2]), int(p[1]), int(p[0])), (0, 0, 0), (dx - 1, dy - 1, dz - 1), (dx // 2, 0, dz // 2),
            (0, dy // 2, dz - 1)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("con", [6, 18, 26])
def test_confidence_matches_checker(orc, dtype, con):
    from invesalius3_b200 import region_grow as rg
    shape = (29, 47, 38)
    vol = _phantom(shape, 5 + con, dtype)
    st = structure(con)
    grower = rg.RegionGrower(vol)
    grown = 0
    for k, p in enumerate(_seeds(shape, _phantom(shape, 5 + con))):
        for iters, mult in ((0, 2.5), (1, 2.5), (2, 1.0), (3, 2.5), (4, 0.7), (3, 4)):
            for wwl in (None, (406, -18), (255, 127)):
                if (k + iters) % 2 and wwl is not None:
                    continue
                kw = dict(use_ww_wl=wwl is not None, ww=wwl and wwl[0], wl=wwl and wwl[1])
                th_w, th_g = [], []
                want = _outcome(lambda: rg_confidence(orc, vol, p, st, iters, mult, thresholds=th_w, **kw))
                got = _outcome(lambda: grower.confidence(p, st, iters, mult, thresholds=th_g, **kw))
                assert th_g == th_w, (p, iters, mult, wwl)
                if want is OverflowError:
                    assert got is OverflowError, (p, iters, mult, wwl)
                    continue
                grown += int(want.sum())
                assert np.array_equal(got, want), (p, iters, mult, wwl)
    assert grown > 10000
    p = _seeds(shape, _phantom(shape, 5 + con))[0]
    got = _outcome(lambda: rg.do_rg_confidence(vol, np.zeros(shape, np.uint8), p, st, 3, 2.5, False))
    want = _outcome(lambda: rg_confidence(orc, vol, p, st, 3, 2.5, False))
    assert got is want is OverflowError or np.array_equal(got, want)


def test_confidence_2d_tool(orc):
    """do_2d_seg's call: a (1, dy, dx) slice with a (1, 3, 3) structure, strided views of a volume."""
    from invesalius3_b200 import region_grow as rg
    vol = _phantom((40, 96, 120), 8)
    for con2d in (1, 2):
        st = np.array(generate_binary_structure(2, con2d), np.uint8).reshape(1, 3, 3)
        for image in (vol[20][None], vol[:, 50, :][None], vol[:, :, 60][None]):
            dy, dx = image.shape[1:]
            for p in ((dx // 2, dy // 2, 0), (0, 0, 0), (dx - 1, dy // 3, 0)):
                for kw in ({}, dict(use_ww_wl=True, ww=406, wl=-18)):
                    want = rg_confidence(orc, np.ascontiguousarray(image), p, st, 3, 2.5, **kw)
                    got = rg.do_rg_confidence(image, np.zeros(image.shape, np.uint8), p, st, 3, 2.5, **kw)
                    assert np.array_equal(got, want), (p, kw)


def test_confidence_large_volume(orc):
    from invesalius3_b200 import region_grow as rg
    vol = _phantom((256, 512, 512), 2)
    st = structure(26)
    p = _seeds(vol.shape, vol)[0]
    for kw in ({}, dict(use_ww_wl=True, ww=406, wl=-18)):
        th_w, th_g = [], []
        want = rg_confidence(orc, vol, p, st, 3, 2.5, thresholds=th_w, **kw)
        got = rg.RegionGrower(vol).confidence(p, st, 3, 2.5, thresholds=th_g, **kw)
        assert th_g == th_w and np.array_equal(got, want), kw
        assert want.sum() > 1000


# ----------------------------------------------------------------------------- dynamic, threshold
@pytest.mark.parametrize("dtype", DTYPES)
def test_dynamic_and_threshold(orc, dtype):
    from invesalius3_b200 import region_grow as rg
    shape = (31, 45, 52)
    vol = _phantom(shape, 12, dtype)
    grower = rg.RegionGrower(vol)
    seeds = _seeds(shape, _phantom(shape, 12))
    for con in (6, 26):
        st = structure(con)
        for p in seeds:
            for kw in (dict(), dict(use_ww_wl=False), dict(ww=2000, wl=300), dict(dev_min=3, dev_max=40, ww=406, wl=-18)):
                kw.setdefault("ww", 406); kw.setdefault("wl", -18)
                want = grow_3d(orc, vol, p, st, "dynamic", **kw)
                got = grower.grow(p, st, "dynamic", **kw)
                assert (got is None) == (want is None) and (got is None or np.array_equal(got, want)), (p, kw)
            x, y, z = p
            v = vol[z, y, x].item()
            for t0, t1 in ((v - 5, v + 300), (v + 1, v + 50), (v - 50, v - 1)):
                if dtype != np.float64:
                    info = np.iinfo(dtype)
                    t0, t1 = (int(min(max(t, info.min), info.max)) for t in (t0, t1))
                want = grow_3d(orc, vol, p, st, "threshold", t0=t0, t1=t1)
                got = rg.region_grow_3d(vol, p, st, "threshold", t0=t0, t1=t1)
                assert (got is None) == (want is None) and (got is None or np.array_equal(got, want)), (p, t0, t1)
    # an early return on a uint8 image: 250 + 25 wraps
    img = np.full((4, 5, 6), 250, np.uint8)
    assert rg.region_grow_3d(img, (1, 1, 1), structure(6), "dynamic", use_ww_wl=False) is None
    kw = dict(use_ww_wl=dtype != np.uint8, ww=406, wl=-18)
    got = _outcome(lambda: rg.region_grow_3d(vol, seeds[0], structure(6), "confidence", **kw))
    want = _outcome(lambda: grow_3d(orc, vol, seeds[0], structure(6), "confidence", **kw))
    assert got is want is OverflowError or np.array_equal(got, want)


# ----------------------------------------------------------------------------- image density
def test_image_density(cranium):
    from invesalius3_b200 import region_grow as rg
    img = cranium["matrix_crop"]
    for i in (0, 1):
        lo, hi = cranium[f"thr_{i}"]
        body = ((img >= lo) & (img <= hi)).astype(np.uint8) * 255
        padded = np.zeros(tuple(s + 1 for s in img.shape), np.uint8)
        padded[1:, 1:, 1:] = body
        got = rg.calc_image_density(img, padded[1:, 1:, 1:])
        want = image_density(img, body)
        assert [type(g) for g in got] == [type(w) for w in want] and got == want
    assert rg.calc_image_density(img, np.zeros(img.shape, np.uint8)) == (0, 0, 0, 0)
    for dtype in DTYPES:
        vol = _phantom((37, 64, 59), 21, dtype)
        body = np.where(_phantom((37, 64, 59), 21) > 100, 255, 0).astype(np.uint8)
        body[0] = 128
        got, want = rg.calc_image_density(vol, body), image_density(vol, body)
        assert [type(g) for g in got] == [type(w) for w in want] and got == want


# ----------------------------------------------------------------------------- errors, residency
def test_errors():
    from invesalius3_b200 import region_grow as rg
    vol = np.zeros((4, 5, 6), np.int16)
    vol[0, 0, 0] = -32768
    vol[0, 0, 1] = 32767
    st = structure(6)
    with pytest.raises(OverflowError):             # mean -/+ 2.5 std leaves int16
        rg.do_rg_confidence(vol, None, (0, 0, 0), st, 1, 2.5)
    with pytest.raises(IndexError):
        rg.do_rg_confidence(vol, None, (6, 0, 0), st, 1, 2.5)
    with pytest.raises(IndexError):
        rg.region_grow_3d(vol, (0, 5, 0), st, "dynamic")
    with pytest.raises(OverflowError):
        rg.region_grow_3d(vol, (0, -1, 0), st, "threshold", t0=0, t1=1)
    with pytest.raises(ValueError):
        rg.region_grow_3d(vol, (0, 0, 0), st, "magic")


def test_grower_uploads_the_image_once(monkeypatch):
    from invesalius3_b200 import device as dev
    from invesalius3_b200 import region_grow as rg
    moved = []
    to_device = dev.to_device

    def rec_to_device(a, device=None):
        moved.append(a.shape)
        return to_device(a, device)

    monkeypatch.setattr(dev, "to_device", rec_to_device)
    vol = _phantom((30, 40, 50), 4)
    st = structure(6)
    g = rg.RegionGrower(vol)
    p = _seeds(vol.shape, vol)[0]
    for kw in ({}, dict(use_ww_wl=True, ww=406, wl=-18), dict(use_ww_wl=True, ww=406, wl=-18)):
        assert g.confidence(p, st, 3, 2.5, **kw).shape == vol.shape
    assert g.grow(p, st, "dynamic", ww=406, wl=-18) is not None
    assert g.grow(p, st, "threshold", t0=-1000, t1=32767) is not None
    assert moved == [vol.shape]
    g.image_density(np.full(vol.shape, 255, np.uint8))
    assert moved == [vol.shape, vol.shape]
