"""scipy.ndimage.shift, FixGantryTilt and make_orthogonal on the device (invesalius3_b200.resample) against
SciPy, the sequential FixGantryTilt loop and the CPU restatements of tests/shift_model.py, with
np.array_equal."""
import numpy as np
import pytest
from scipy import ndimage as ndi

import shift_model as sm
from test_shift_model import SPACING, TILTS, cranium_matrix

pytestmark = pytest.mark.gpu


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)


@pytest.mark.parametrize("order", [0, 1, 2, 3])
@pytest.mark.parametrize("mode", ["constant", "mirror"])
def test_shift_odd_shapes(order, mode):
    from invesalius3_b200 import resample
    rng = np.random.default_rng(order * 2 + len(mode))
    cases = [((17, 33, 47), (0.3, -1.7, 2.25)), ((5, 3, 1), (1e-12, -0.5, 0.0)), ((1, 20, 301), (0.0, 4.5, -300)),
             ((301, 2, 5), (-150.5, 0.999999, -1e-12)), ((33, 65), (-0.0, 64.5)), ((1, 1), 0.5), ((7, 130), (-6, 131)),
             ((40, 64, 3), 12.75)]
    for shape, sh in cases:
        for dtype in (np.int16, np.uint8, np.float32, np.float64):
            a = (rng.standard_normal(shape) * 900).astype(dtype) if dtype != np.uint8 else \
                ((rng.random(shape) > 0.5) * 255).astype(np.uint8)
            ref = ndi.shift(a, sh, order=order, mode=mode, cval=-5.0)
            assert _same(resample.shift(a, sh, order=order, mode=mode, cval=-5.0), ref), (shape, sh, dtype)
            if a.ndim == 3 and a.size < 40000:
                assert _same(sm.shift(a, sh, order=order, mode=mode, cval=-5.0), ref)


def test_shift_strided_output_and_device_api():
    import torch
    from invesalius3_b200 import device as dev
    from invesalius3_b200 import phantom, resample
    vol = phantom.ct((30, 70, 90), seed=4)
    for view in (vol[::2, 3:, 1:-1], vol[:, :, ::3], vol[5]):
        for order in (1, 3):
            sh = (2.5, -0.25, 7.0)[-view.ndim:]
            ref = ndi.shift(view, sh, order=order)
            assert _same(resample.shift(view, sh, order=order), ref)
            out = np.full(view.shape, 7, np.float32)
            r = resample.shift(view, sh, out, order=order)
            assert r is out and _same(out, ndi.shift(view, sh, np.float32, order=order))
    t = dev.to_device(vol)
    for out in (torch.int16, torch.uint8, torch.float32, torch.float64):
        got = resample.shift_device(t, (-1.5, 3.25, 0.5), 3, out, cval=-1000.0).cpu().numpy()
        assert _same(got, ndi.shift(vol, (-1.5, 3.25, 0.5), got.dtype, order=3, cval=-1000.0))
    with pytest.raises(NotImplementedError):
        resample.shift_device(t, 0.5, 4, torch.int16)
    with pytest.raises(NotImplementedError):
        resample.shift_device(t, 0.5, 3, torch.int16, mode="wrap")


@pytest.mark.parametrize("tilt", TILTS)
def test_fix_gantry_tilt_cranium(tilt, tmp_path):
    """On a copy and on an np.memmap of the Cranium matrix: equal to the loop at each tilt; the device's cvals
    equal the loop's."""
    import torch
    from invesalius3_b200 import device as dev
    from invesalius3_b200 import resample
    m = cranium_matrix()
    ref, ref_cvals = sm.reference_loop(m, SPACING, tilt)
    a = m.copy()
    assert resample.fix_gantry_tilt(a, SPACING, tilt) is None
    assert _same(a, ref)
    mm = np.memmap(tmp_path / "matrix.dat", dtype=np.int16, mode="w+", shape=m.shape)
    mm[:] = m
    resample.fix_gantry_tilt(mm, SPACING, tilt)
    assert _same(np.asarray(mm), ref)
    for slab in (1, 3, 0):
        t = dev.to_device(m)
        cvals = resample.fix_gantry_tilt_device(t, SPACING, tilt, slab=slab)
        torch.cuda.synchronize()
        assert _same(t.cpu().numpy(), ref), slab
        assert cvals.cpu().tolist() == ref_cvals, slab


def test_fix_gantry_tilt_phantom_256x512x512():
    from invesalius3_b200 import phantom, resample
    vol = phantom.ct((256, 512, 512), seed=6)
    want, _ = sm.fix_gantry_tilt(vol, (0.5, 0.5, 1.0), 15)
    resample.fix_gantry_tilt(vol, (0.5, 0.5, 1.0), 15)
    assert _same(vol, want)


def test_fix_gantry_tilt_small_volumes():
    """Single rows and columns, one slice, and tilts that push whole slices out of range."""
    from invesalius3_b200 import resample
    rng = np.random.default_rng(12)
    for shape, sp, tilt in [((6, 1, 9), (1, 1, 1), 30), ((5, 7, 1), (1, 0.5, 2), -40), ((1, 8, 8), SPACING, 10),
                            ((9, 4, 6), (1, 0.2, 3), 60), ((12, 31, 17), (0.4, 0.4, 1.25), -89)]:
        m = rng.integers(-1200, 3000, size=shape).astype(np.int16)
        ref, _ = sm.reference_loop(m, sp, tilt)
        a = m.copy()
        resample.fix_gantry_tilt(a, sp, tilt)
        assert _same(a, ref), (shape, tilt)


def test_make_orthogonal_cranium():
    from invesalius3_b200 import resample
    m = cranium_matrix()
    new = (1.0, 1.0, 1.0)
    zooms = [i / j for (i, j) in zip(SPACING, new)]
    ref = ndi.zoom(m, zooms[::-1], output=m.dtype, mode="constant", cval=m.min())
    assert _same(resample.make_orthogonal(m, SPACING, new), ref)
    u8 = np.where(m[:40, :90, :70] > 300, 255, 3).astype(np.uint8)
    ref = ndi.zoom(u8, (1.5, 0.8, 0.8), output=u8.dtype, mode="constant", cval=u8.min())
    assert _same(resample.make_orthogonal(u8, (0.8, 0.8, 1.5), (1.0, 1.0, 1.0)), ref)


def test_fix_gantry_tilt_errors():
    import torch
    from invesalius3_b200 import device as dev
    from invesalius3_b200 import resample
    t = dev.to_device(np.zeros((4, 5, 6), np.int16))
    with pytest.raises(NotImplementedError):
        resample.fix_gantry_tilt_device(t.to(torch.float32), SPACING, 10)
    with pytest.raises(ValueError):
        resample.fix_gantry_tilt_device(t[0], SPACING, 10)
    with pytest.raises(ValueError):
        resample.fix_gantry_tilt_device(t[:, :, ::2], SPACING, 10)
