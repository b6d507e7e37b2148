"""The CPU restatement of scipy.ndimage.zoom (oracle/zoom.py) against SciPy itself, bit for bit, and the
argument checks of invesalius3_b200.resample that run before any device work.

The restatement is pinned: its prefilter equals spline_filter1d / spline_filter and its zoom equals
scipy.ndimage.zoom with np.array_equal on every case below, so the device tests compare against it."""
import numpy as np
import pytest
from scipy import ndimage as ndi

from oracle import zoom as oz

ORDERS = [0, 1, 2, 3]
LENGTHS = [1, 2, 3, 4, 5, 6, 7, 8, 15, 16, 17, 31, 32, 33, 64, 100, 127, 128, 255, 256, 301, 512, 513]
FACTORS = [0.5, 1 / 3, 0.25, 1.7]


def _data(shape, dtype, rng):
    dtype = np.dtype(dtype)
    if dtype == np.uint8:
        return (rng.random(shape) > 0.5).astype(np.uint8) * 255           # a 0/255 mask: overshoots at order >= 2
    if dtype == np.int16:
        return rng.choice(np.array([-32768, 32767, -1024, 0, 3071], np.int16), size=shape)   # the int16 limits
    return (rng.standard_normal(shape) * 1000).astype(dtype)


@pytest.mark.parametrize("order", [2, 3])
def test_prefilter_equals_spline_filter1d(order):
    rng = np.random.default_rng(order)
    for n in LENGTHS:
        a = rng.integers(-32768, 32768, size=(4, n)).astype(np.int16)
        ref = ndi.spline_filter1d(a, order, axis=1, output=np.float64, mode="constant")
        mine = a.astype(np.float64)
        oz._filter_axis(mine, order, 1)
        assert np.array_equal(ref, mine), n
        assert np.array_equal(ref, ndi.spline_filter1d(a, order, axis=1, output=np.float64, mode="mirror"))


@pytest.mark.parametrize("order", [2, 3])
@pytest.mark.parametrize("dtype", [np.int16, np.uint8, np.float32, np.float64])
def test_prefilter_equals_spline_filter(order, dtype):
    a = _data((9, 1, 23), dtype, np.random.default_rng(7))
    for shape in [(9, 1, 23), (1, 40, 33), (6, 7)]:
        a = _data(shape, dtype, np.random.default_rng(len(shape)))
        ref = ndi.spline_filter(a, order, output=np.float64, mode="constant")
        assert np.array_equal(ref, oz.spline_filter(a, order))


@pytest.mark.parametrize("order", ORDERS)
def test_zoom_lines_every_length(order):
    """2-D arrays of 3 rows: every line length, every factor, float64 and int16 outputs."""
    rng = np.random.default_rng(10 + order)
    for n in LENGTHS:
        a = rng.integers(-32768, 32768, size=(3, n)).astype(np.int16)
        for f in FACTORS:
            for out in (np.float64, np.int16):
                ref = ndi.zoom(a, (1, f), out, order=order)
                mine = oz.zoom(a, (1, f), order=order, out_dtype=out)
                assert ref.shape == mine.shape and np.array_equal(ref, mine), (n, f, out)


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("mode", ["constant", "mirror"])
@pytest.mark.parametrize("dtype", [np.int16, np.uint8, np.float32, np.float64])
def test_zoom_volumes(order, mode, dtype):
    rng = np.random.default_rng(order * 10 + len(mode))
    cases = [((31, 20, 17), 1 / 3), ((9, 40, 33), 0.25), ((13, 6, 5), 1.7), ((1, 64, 64), 0.5), ((2, 3, 3), 0.5),
             ((3, 1, 5), (1 / 3, 1.7, 0.5)), ((64, 65), (0.5, 1 / 3)), ((1, 1), 1.7), ((3, 1), 0.5), ((301, 7), 0.5)]
    for shape, f in cases:
        a = _data(shape, dtype, rng)
        ref = ndi.zoom(a, f, a.dtype, order=order, mode=mode, cval=-3.0)
        mine = oz.zoom(a, f, order=order, mode=mode, cval=-3.0)
        assert ref.dtype == mine.dtype and ref.shape == mine.shape, (shape, f)
        assert np.array_equal(ref, mine), (shape, f)


def test_integer_outputs_round_half_away_and_clip():
    """A 0/255 mask overshoots below 0 and above 255 at order 2 and comes out as 0 and 255; int16
    results are rounded, not truncated."""
    m = np.zeros((1, 9, 9), np.uint8)
    m[0, 3:6, 3:6] = 255
    f64 = ndi.zoom(m, (1, 1.7, 1.7), np.float64, order=2)
    assert f64.min() < -20 and f64.max() > 275
    u8 = ndi.zoom(m, (1, 1.7, 1.7), np.uint8, order=2)
    assert np.array_equal(u8, oz.zoom(m, (1, 1.7, 1.7), order=2))
    assert np.array_equal(u8, np.clip(np.where(f64 > 0, np.floor(f64 + 0.5), 0), 0, 255))
    a = np.random.default_rng(3).integers(-2000, 2000, size=(1, 31, 31)).astype(np.int16)
    t = ndi.zoom(a, (1, 0.5, 0.5), np.float64, order=2)
    i16 = ndi.zoom(a, (1, 0.5, 0.5), np.int16, order=2)
    assert i16.size == 256
    assert np.array_equal(i16, np.where(t > 0, np.floor(t + 0.5), np.ceil(t - 0.5)))
    assert not np.array_equal(i16, np.trunc(t))
    assert np.array_equal(i16, oz.zoom(a, (1, 0.5, 0.5), order=2))


def test_constant_mode_edge_rule():
    """The last output sample's coordinate (m - 1) * ((n - 1) / (m - 1)) can round past n - 1; SciPy's
    'constant' mode then writes cval (a strict test: exactly n - 1 interpolates), 'mirror' interpolates.
    The first sample's coordinate is 0 and always interpolates. On these samples the result does not
    depend on the coefficients, so they are pinned exactly."""
    past = exact = below = 0
    for n in range(2, 400):
        a = np.full((1, n), 1540, np.int16)
        for f in FACTORS:
            m = oz.output_shape(a.shape, (1, f))[1]
            if m < 2:
                continue
            cc = (m - 1) * oz.step(n, m)
            for order in (0, 2, 3):
                const = ndi.zoom(a, (1, f), np.int16, order=order, mode="constant", cval=-7.0)
                mirror = ndi.zoom(a, (1, f), np.int16, order=order, mode="mirror", cval=-7.0)
                assert const[0, 0] == 1540 and mirror[0, -1] == 1540
                assert const[0, -1] == (-7 if cc > n - 1 else 1540), (n, f, cc)
                assert np.array_equal(const, oz.zoom(a, (1, f), order=order, mode="constant", cval=-7.0))
            past += cc > n - 1
            exact += cc == n - 1
            below += cc < n - 1
    assert past and exact and below
    # the case of a 301-slice series at half resolution
    row = np.full(301, 1540, np.int16)
    assert 149 * (300 / 149) == 300.00000000000006
    assert ndi.zoom(row, 0.5, np.int16, order=2)[-1] == 0
    assert ndi.zoom(row, 0.5, np.int16, order=2, mode="mirror")[-1] == 1540
    assert oz.zoom(row[None], (1, 0.5), order=2)[0, -1] == 0


def test_output_shape_and_identity():
    from invesalius3_b200 import resample
    for shape, f in [((301, 512, 512), 0.5), ((5, 7), 1 / 3), ((2, 3, 5), 1.7), ((1, 1), 0.5)]:
        assert resample.output_shape(shape, f) == ndi.zoom(np.zeros(shape), f, order=0).shape
    a = np.arange(12, dtype=np.int16).reshape(3, 4)
    for z in (1, (1.0, 1)):
        r = resample.zoom(a, z, order=2)                     # SciPy returns the input unchanged
        assert np.array_equal(r, ndi.zoom(a, z, order=2)) and r is not a
    assert np.array_equal(resample.zoom(a, 1, np.float32), a.astype(np.float32))


def test_unbuilt_arguments_raise():
    from invesalius3_b200 import resample
    a = np.zeros((4, 4), np.int16)
    with pytest.raises(NotImplementedError):
        resample.zoom(a, 0.5, order=2, prefilter=False)
    with pytest.raises(NotImplementedError):
        resample.zoom(a, 0.5, order=2, grid_mode=True)
    with pytest.raises(NotImplementedError):
        resample.zoom(a.astype(np.int32), 0.5)
    with pytest.raises(NotImplementedError):
        resample.zoom(a.astype(np.complex128), 0.5)
    with pytest.raises(NotImplementedError):
        resample.zoom(a, 0.5, np.uint16)
    with pytest.raises(NotImplementedError):
        resample.zoom(np.zeros(8, np.int16), 0.5)
    with pytest.raises(RuntimeError):
        resample.zoom(a, (0.5, 0.5, 0.5))
    with pytest.raises(RuntimeError):
        resample.zoom(a, 0.5, output=np.zeros((3, 3), np.int16))
