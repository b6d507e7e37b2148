"""The CPU restatement of scipy.ndimage.shift and of FixGantryTilt's parallel form (tests/shift_model.py)
against SciPy and the sequential loop, bit for bit, and the argument checks of invesalius3_b200.resample that
run before any device work."""
import io
import lzma
from pathlib import Path

import numpy as np
import pytest
from scipy import ndimage as ndi

import shift_model as sm

DTYPES = [np.int16, np.uint8, np.float32, np.float64]
SPACING = (0.957, 0.957, 1.5)
TILTS = [-20, 12, 0, 45, -70]


def _shifts(n):
    return [0.0, -0.0, 1e-12, -1e-12, 0.5, -0.5, 0.999999, -0.999999, 1, -1, 3, -7, n - 1, -(n - 1), n, -n,
            n + 2.5, -(2 * n + 0.3), 5 * n + 0.7, -5 * n - 0.2]


def _data(shape, dtype, rng):
    dtype = np.dtype(dtype)
    if dtype == np.uint8:
        return (rng.random(shape) > 0.5).astype(np.uint8) * 255    # a 0/255 mask: undershoots below 0 at orders 2, 3
    if dtype == np.int16:
        return rng.choice(np.array([-32768, 32767, -1024, 0, 3071], np.int16), size=shape)
    return (rng.standard_normal(shape) * 1000).astype(dtype)


def cranium_matrix():
    src = Path(__file__).resolve().parent / "golden" / "cranium_thr_matrix.npy.xz"
    return np.load(io.BytesIO(lzma.decompress(src.read_bytes())))


@pytest.mark.parametrize("order", [0, 1, 2, 3])
@pytest.mark.parametrize("mode", ["constant", "mirror"])
def test_shift_lines_every_length(order, mode):
    """Lines of 1-130 samples as rows and as columns, every edge shift, the four dtypes in turn."""
    rng = np.random.default_rng(order * 2 + len(mode))
    for n in range(1, 131):
        dtype = DTYPES[n % 4]
        for a, axis in ((_data((3, n), dtype, rng), 1), (_data((n, 2), dtype, rng), 0)):
            for s in _shifts(n):
                sh = (0, s) if axis == 1 else (s, 0)
                ref = ndi.shift(a, sh, order=order, mode=mode, cval=-3.0)
                mine = sm.shift(a, sh, order=order, mode=mode, cval=-3.0)
                assert ref.dtype == mine.dtype and np.array_equal(ref, mine), (n, dtype, axis, s)


@pytest.mark.parametrize("order", [0, 1, 2, 3])
@pytest.mark.parametrize("mode", ["constant", "mirror"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_shift_volumes(order, mode, dtype):
    rng = np.random.default_rng(order * 10 + len(mode))
    cases = [((9, 14, 11), (0.3, -1.7, 2.25)), ((1, 20, 17), (0.0, 4.5, -0.5)), ((5, 1, 7), (-2, 0.25, 1e-12)),
             ((6, 8, 9), (7, -8, 9.5)), ((4, 5, 6), 0.75), ((13, 3, 2), (-12.999999, 1.5, -0.0))]
    for shape, sh in cases:
        a = _data(shape, dtype, rng)
        ref = ndi.shift(a, sh, order=order, mode=mode, cval=-3.0)
        assert np.array_equal(ref, sm.shift(a, sh, order=order, mode=mode, cval=-3.0)), (shape, sh)


@pytest.mark.parametrize("order", [2, 3])
def test_uint8_outputs_undershoot(order):
    """A 0/255 mask shifted by half a sample rings below 0 and above 255; uint8 outputs clip."""
    m = np.zeros((9, 12), np.uint8)
    m[3:6, 4:8] = 255
    f64 = ndi.shift(m, (0.5, -0.5), np.float64, order=order)
    assert f64.min() < 0 and f64.max() > 255
    for src in (m, m.astype(np.float32)):
        for mode in ("constant", "mirror"):
            ref = ndi.shift(src, (0.5, -0.5), np.uint8, order=order, mode=mode)
            assert np.array_equal(ref, sm.shift(src, (0.5, -0.5), order=order, mode=mode, out_dtype=np.uint8))


def test_constant_mode_is_strict_on_both_sides():
    row = np.array([[10, 20, 30, 40, 50]], np.float64)
    assert ndi.shift(row, (0, 1e-12), order=1, cval=-1)[0, 0] == -1
    assert ndi.shift(row, (0, -1e-12), order=1, cval=-1)[0, 4] == -1
    assert np.array_equal(sm.shift(row, (0, 1e-12), order=1, cval=-1), ndi.shift(row, (0, 1e-12), order=1, cval=-1))
    assert np.array_equal(sm.shift(row, (0, -1e-12), order=1, cval=-1),
                          ndi.shift(row, (0, -1e-12), order=1, cval=-1))


def test_gantry_tilt_chain_equals_loop():
    """The parallel form (SciPy as the interpolator) equals the sequential loop on the Cranium matrix, and the
    running cval takes more than one value there."""
    m = cranium_matrix()
    distinct = []
    for tilt in TILTS:
        ref, ref_cvals = sm.reference_loop(m, SPACING, tilt)
        got, cvals = sm.fix_gantry_tilt(m, SPACING, tilt)
        assert np.array_equal(ref, got) and ref_cvals == cvals, tilt
        distinct.append(len(set(cvals)))
    assert max(distinct) > 1, distinct


def test_tilt_shifts_follow_the_reference():
    from invesalius3_b200 import resample
    for sp, tilt in ((SPACING, -20), ((0.5, 0.5, 1.0), 15), ((0.3, 0.7, 2.5), 3.3), (SPACING, 0)):
        got = resample.tilt_shifts(40, sp, tilt)
        assert got.dtype == np.float64 and got.shape == (40, 2)
        assert got[:, 0].tolist() == sm.tilt_shifts(40, sp, tilt) and not got[:, 1].any()


def test_unbuilt_and_bad_arguments_raise():
    from invesalius3_b200 import resample
    a = np.zeros((4, 4), np.int16)
    with pytest.raises(NotImplementedError):
        resample.shift(a, 0.5, prefilter=False)
    with pytest.raises(NotImplementedError):
        resample.shift(a, 0.5, order=4)
    with pytest.raises(NotImplementedError):
        resample.shift(a, 0.5, mode="nearest")
    with pytest.raises(NotImplementedError):
        resample.shift(a.astype(np.int32), 0.5)
    with pytest.raises(NotImplementedError):
        resample.shift(a, 0.5, np.uint16)
    with pytest.raises(NotImplementedError):
        resample.shift(np.zeros(8, np.int16), 0.5)
    with pytest.raises(RuntimeError):
        resample.shift(a, (0.5, 0.5, 0.5))
    with pytest.raises(RuntimeError):
        resample.shift(a, 0.5, output=np.zeros((3, 3), np.int16))
    vol = np.zeros((3, 4, 5), np.int16)
    with pytest.raises(RuntimeError):
        resample.fix_gantry_tilt(vol[0], SPACING, 10)
    with pytest.raises(ValueError, match="zero-size"):
        resample.fix_gantry_tilt(np.zeros((3, 0, 5), np.int16), SPACING, 10)
    resample.fix_gantry_tilt(np.zeros((0, 4, 5), np.int16), SPACING, 10)   # the loop has no slice to shift
    ro = vol.copy()
    ro.flags.writeable = False
    with pytest.raises(ValueError, match="read-only"):
        resample.fix_gantry_tilt(ro, SPACING, 10)
    with pytest.raises(NotImplementedError):
        resample.fix_gantry_tilt(vol.astype(np.float32), SPACING, 10)
    with pytest.raises(NotImplementedError):
        resample.make_orthogonal(vol.astype(np.float32), SPACING, (1, 1, 1))
