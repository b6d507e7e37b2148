"""The region growing tool restated in NumPy (the checker of tests/test_gpu_region_grow.py), and
the pairwise summation order the device reproduces, pinned to the NumPy in use.

  pairwise_sum     NumPy's pairwise_sum (numpy/_core/src/umath/loops_utils.h.src) over a float64 list
  lut255           get_LUT_value_255, the reference's np.piecewise (imagedata_utils.py:540-552)
  rg_confidence    do_rg_confidence (styles.py:3220-3251) with the config as arguments
  grow_3d          the growth part of do_3d_seg (styles.py:3157-3203)
  image_density    Slice.calc_image_density (slice_.py:2288-2297)

The flood is the CPU oracle's restatement of floodfill.rs. The thresholds reach it as the crate's
wrapper converts them for int16 (int(), then a range check); uint8 is treated the same way and
float64 gets float() (the crate's wrapper raises TypeError on both, see INTEGRATION.md)."""
import numpy as np
import pytest
from scipy.ndimage import generate_binary_structure


# ----------------------------------------------------------------------------- the checker
def pairwise_sum(a, lo=0, n=None):
    n = len(a) if n is None else n
    if n < 8:
        r = -0.0
        for i in range(n):
            r += a[lo + i]
        return r
    if n <= 128:
        r = [a[lo + k] for k in range(8)]
        i = 8
        while i < n - n % 8:
            for k in range(8):
                r[k] += a[lo + i + k]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for j in range(i, n):
            res += a[lo + j]
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise_sum(a, lo, n2) + pairwise_sum(a, lo + n2, n - n2)


def pw_mean_std(v):
    f = np.asarray(v).astype(np.float64).ravel().tolist()
    n = len(f)
    m = pairwise_sum(f) / n
    return m, float(np.sqrt(pairwise_sum([(a - m) * (a - m) for a in f]) / n))


def lut255(data, window, level):
    shape = data.shape
    data_ = data.ravel()
    data = np.piecewise(
        data_,
        [data_ <= (level - 0.5 - (window - 1) / 2), data_ > (level - 0.5 + (window - 1) / 2)],
        [0, 255, lambda data_: ((data_ - (level - 0.5)) / (window - 1) + 0.5) * (255)],
    )
    data.shape = shape
    return data


def _int_or_float(t, dtype):
    if dtype == np.float64:
        return float(t)
    t = int(t)
    lo, hi = (-32768, 32767) if dtype == np.int16 else (0, 255)
    if not lo <= t <= hi:
        raise OverflowError("out of range integral type conversion attempted")
    return t


def flood(orc, image, p, t0, t1, bstruct, out):
    t0, t1 = _int_or_float(t0, image.dtype), _int_or_float(t1, image.dtype)
    orc._floodfill_threshold_core(image, [p], t0, t1, 1, np.ascontiguousarray(bstruct, np.uint8), out)


def rg_confidence(orc, image, p, bstruct, iters, mult, use_ww_wl=False, ww=None, wl=None, thresholds=None):
    x, y, z = p
    if use_ww_wl:
        image = lut255(image, ww, wl)
    sel = np.zeros(image.shape, bool)
    sel[max(z - 1, 0): z + 2, max(y - 1, 0): y + 2, max(x - 1, 0): x + 2] = True
    out = np.zeros(image.shape, np.uint8)
    for _ in range(iters):
        var = np.std(image[sel])
        mean = np.mean(image[sel])
        t0, t1 = mean - var * mult, mean + var * mult
        if thresholds is not None:
            thresholds.append((t0, t1))
        flood(orc, image, (x, y, z), t0, t1, bstruct, out)
        sel |= out == 1
    return out


def grow_3d(orc, image, p, bstruct, method, t0=None, t1=None, dev_min=25, dev_max=25, use_ww_wl=True, ww=None, wl=None,
            confid_iters=3, confid_mult=2.5):
    x, y, z = p
    if method == "confidence":
        return rg_confidence(orc, image, p, bstruct, confid_iters, confid_mult, use_ww_wl, ww, wl)
    if method == "dynamic":
        if use_ww_wl:
            image = lut255(image, ww, wl)
        v = image[z, y, x]
        with np.errstate(over="ignore"):
            t0, t1 = v - dev_min, v + dev_max
    if image[z, y, x] < t0 or image[z, y, x] > t1:
        return None
    out = np.zeros(image.shape, np.uint8)
    flood(orc, image, p, t0, t1, bstruct, out)
    return out


def image_density(matrix, mask_body):
    values = matrix[mask_body > 127]
    if len(values):
        return values.min(), values.max(), values.mean(), values.std()
    return 0, 0, 0, 0


def structure(con):
    """CON3D of styles.py: 6 -> 1, 18 -> 2, 26 -> 3."""
    return np.array(generate_binary_structure(3, {6: 1, 18: 2, 26: 3}[con]), dtype=np.uint8)


# ----------------------------------------------------------------------------- pairwise order
def _sizes():
    s = set(range(1, 10)) | {127, 128, 129, 255, 256, 257, 1_000_003}
    for k in range(3, 18):
        s |= {2 ** k - 1, 2 ** k + 1}
    return sorted(s)


@pytest.mark.parametrize("dtype", [np.int16, np.uint8, np.float64])
def test_pairwise_order_is_numpys(dtype):
    rng = np.random.default_rng(3)
    for n in _sizes():
        if dtype == np.uint8:
            v = rng.integers(0, 256, n).astype(dtype)
        elif dtype == np.int16:
            v = rng.normal(300, 900, n).astype(dtype)
        else:
            v = rng.normal(300, 900, n) * rng.choice([1e-3, 1.0, 1e5], n)
        m, s = pw_mean_std(v)
        assert np.mean(v) == m and np.std(v) == s, (dtype, n)


def test_pairwise_order_matters():
    """A plain left-to-right sum differs from NumPy's on these values: the test above has teeth."""
    rng = np.random.default_rng(5)
    v = rng.normal(0, 1, 4099) * 10.0 ** rng.integers(-8, 8, 4099)
    seq = 0.0
    for a in v.tolist():
        seq += a
    assert pairwise_sum(v.tolist()) == np.sum(v) != seq


# ----------------------------------------------------------------------------- checker sanity
def test_lut255_hand_values():
    v = np.array([-100, 9, 10, 11, 50, 90, 91, 200], np.int16)
    got = lut255(v, 81, 50)            # lo = 9.5, hi = 89.5
    assert got.dtype == np.int16
    assert got.tolist() == [0, 0, int(((10 - 49.5) / 80 + 0.5) * 255), int(((11 - 49.5) / 80 + 0.5) * 255),
                            int((0.5 / 80 + 0.5) * 255), 255, 255, 255]
    assert lut255(v, 1, 50).tolist() == [0, 0, 0, 0, 255, 255, 255, 255]     # v <= 49.5 | v > 49.5
    assert lut255(v, 0, 50).tolist() == [0, 0, 0, 0, 255, 255, 255, 255]     # overlap at (49, 50]: 255 wins


def test_confidence_hand_case(orc):
    """A bright 5x5x5 cube (100) in 0 with a 200 core: the box about a cube voxel sees 100s and 0s."""
    img = np.zeros((9, 9, 9), np.int16)
    img[2:7, 2:7, 2:7] = 100
    st = structure(6)
    th = []
    out = rg_confidence(orc, img, (4, 4, 4), st, 1, 0.5, thresholds=th)
    assert th == [(100.0, 100.0)]
    assert out.sum() == 125 and (out[2:7, 2:7, 2:7] == 1).all()
    th = []
    out = rg_confidence(orc, img, (2, 2, 2), st, 1, 2.5, thresholds=th)    # a corner: 8 of 27 are 100
    m, s = pw_mean_std(np.where(np.arange(27) < 8, 100, 0))
    assert th[0][0] == m - s * 2.5 and out.sum() == 9 ** 3                  # 0 .. 100 all in range


def test_confidence_walls(orc):
    """From the second iteration on, voxels grown by the first are walls: the flood can only start
    at the seed's still-unfilled neighbours, so a region that the first iteration cut off from the
    seed's neighbourhood stays out even when the wider thresholds would take it."""
    img = np.full((1, 7, 12), 10, np.int16)     # the seed's region: columns 0-4
    img[0, 2, 0] = 16                           # in the seed's box
    img[0, :, 4] = 15
    img[0, :, 5:] = 19                          # beyond it
    st = np.array(generate_binary_structure(2, 1), np.uint8).reshape(1, 3, 3)
    th = []
    out = rg_confidence(orc, img, (1, 3, 0), st, 2, 4.0, thresholds=th)
    assert 3 < th[0][0] < 10 and 16 < th[0][1] < 19
    assert out[0, :, :5].all() and not out[0, :, 5:].any()
    assert th[1][0] <= 10 and th[1][1] >= 19     # the 19s are in range, yet every path to them is walled
    out1 = np.zeros_like(out)
    flood(orc, img, (1, 3, 0), *th[1], st, out1)
    assert out1.sum() == img.size                # a fresh flood with those thresholds takes everything


def test_dynamic_wraps_and_returns_early(orc):
    img = np.full((3, 4, 5), 250, np.uint8)
    st = structure(6)
    # uint8 scalar arithmetic: 250 + 25 wraps to 19 < 250, so the reference returns early
    assert grow_3d(orc, img, (1, 1, 1), st, "dynamic", use_ww_wl=False) is None
    img[:] = 100
    out = grow_3d(orc, img, (1, 1, 1), st, "dynamic", use_ww_wl=False)
    assert out.sum() == img.size
    assert grow_3d(orc, img, (1, 1, 1), st, "threshold", t0=101, t1=200) is None


def test_image_density_hand_case():
    m = np.arange(24, dtype=np.int16).reshape(2, 3, 4)
    mask = np.zeros(m.shape, np.uint8)
    mask[1] = 200
    mn, mx, mean, std = image_density(m, mask)
    assert (mn, mx, mean) == (12, 23, 17.5) and type(mn) is np.int16 and type(mean) is np.float64
    assert image_density(m, np.zeros_like(mask)) == (0, 0, 0, 0)
