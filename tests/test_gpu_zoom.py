"""scipy.ndimage.zoom on the device (invesalius3_b200.resample) against the CPU restatement
(oracle/zoom.py) and SciPy, with np.array_equal. The restatement equals SciPy bit for bit
(tests/test_zoom_model.py), so at the largest sizes the device is compared with SciPy alone."""
import os

import numpy as np
import pytest
from scipy import ndimage as ndi

from oracle import zoom as oz

pytestmark = pytest.mark.gpu

FACTORS = [0.5, 1 / 3, 0.25, 1.7]


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)


def _check(a, f, order, out=None, mode="constant", cval=0.0):
    from invesalius3_b200 import resample
    ref = ndi.zoom(a, f, out, order=order, mode=mode, cval=cval)
    got = resample.zoom(a, f, out, order=order, mode=mode, cval=cval)
    assert _same(got, ref), (a.shape, f, order, out, mode)
    assert _same(got, oz.zoom(a, f, order=order, mode=mode, cval=cval, out_dtype=out))


@pytest.mark.parametrize("order", [0, 1, 2, 3])
@pytest.mark.parametrize("mode", ["constant", "mirror"])
def test_int16_limits(order, mode):
    rng = np.random.default_rng(order)
    shapes = [(17, 33, 47), (5, 3, 1), (2, 1, 7), (3, 45, 16), (1, 20, 301), (301, 2, 5), (7, 40, 64)]
    for shape in shapes:
        a = rng.choice(np.array([-32768, 32767, -32767, 32766, 0, -1024, 3071], np.int16), size=shape)
        for f in FACTORS:
            _check(a, f, order, mode=mode, cval=-5.0)
    _check(a, (0.5, 1.7, 1 / 3), order, np.float64, mode=mode)


@pytest.mark.parametrize("order", [0, 1, 2, 3])
def test_uint8_mask_overshoot(order):
    """A 0/255 mask overshoots at orders 2 and 3; the uint8 output clips to 0 and 255."""
    rng = np.random.default_rng(10 + order)
    m = ((rng.random((40, 37, 66)) > 0.6) * 255).astype(np.uint8)
    for f in FACTORS:
        _check(m, f, order)
    if order >= 2:
        f64 = ndi.zoom(m, 1.7, np.float64, order=order)
        assert f64.min() < 0 and f64.max() > 255


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("order", [0, 1, 2, 3])
def test_float_inputs(dtype, order):
    rng = np.random.default_rng(20 + order)
    a = (rng.standard_normal((19, 28, 35)) * 500).astype(dtype)
    for f in FACTORS:
        _check(a, f, order, mode="constant", cval=2.5)
        _check(a, f, order, mode="mirror")
    for out in (np.int16, np.uint8, np.float32, np.float64):
        _check(a, 0.5, order, out)


@pytest.mark.parametrize("order", [2, 3])
def test_slices_512(order):
    from invesalius3_b200 import phantom, resample
    vol = phantom.ct((3, 512, 512), seed=5)
    for k in range(3):
        sl = vol[k]
        for f in FACTORS:
            _check(sl, f, order)
        if order == 2:
            assert _same(resample.resize_slice(sl, 0.5), ndi.zoom(sl, 0.5, sl.dtype, order=2))
    _check(vol[1].astype(np.float32), 0.25, 3)    # the thumbnails: zoom(np_image[i], 0.25), order 3


def test_device_api_dtypes_and_identity():
    import torch
    from invesalius3_b200 import device as dev
    from invesalius3_b200 import resample
    a = np.random.default_rng(4).integers(-3000, 3000, size=(9, 30, 31)).astype(np.int16)
    t = dev.to_device(a)
    for out in (torch.int16, torch.uint8, torch.float32, torch.float64):
        got = resample.zoom_device(t, 1 / 3, 2, out).cpu().numpy()
        assert _same(got, ndi.zoom(a, 1 / 3, got.dtype, order=2))
    same = resample.zoom_device(t, 1, 3, torch.int16)
    assert same.data_ptr() != t.data_ptr() and torch.equal(same, t)
    assert resample.zoom_device(t, (0.01, 1, 1), 2, torch.int16).shape == (0, 30, 31)
    with pytest.raises(NotImplementedError):
        resample.zoom_device(t, 0.5, 4, torch.int16)
    with pytest.raises(NotImplementedError):
        resample.zoom_device(t, 0.5, 2, torch.int16, mode="nearest")


def test_padded_mask_views_and_mmap(tmp_path):
    """resize_image_array on the padded mask.matrix memmap, on its strided [1:, 1:, 1:] view, and with
    as_mmap=True (surface.py:1352-1353)."""
    from invesalius3_b200 import phantom, resample
    img = phantom.ct((45, 96, 80), seed=8)
    mm = np.memmap(tmp_path / "mask.dat", dtype=np.uint8, mode="w+", shape=(46, 97, 81))
    mm[1:, 1:, 1:] = np.where(img > 200, 255, 0).astype(np.uint8)
    mm[1:, 0, 0] = 1
    for res in (2, 3):
        for arr in (mm, mm[1:, 1:, 1:], img, img[::2, 3:, 1:-1]):
            ref = ndi.zoom(arr, 1.0 / res, arr.dtype, order=2)
            got = resample.resize_image_array(arr, 1.0 / res)
            assert _same(got, ref)
            m = resample.resize_image_array(arr, 1.0 / res, True)
            assert isinstance(m, np.memmap) and m.filename and _same(np.asarray(m), ref)
            fname = m.filename
            del m
            os.unlink(fname)


@pytest.mark.parametrize("factor", [0.5, 1 / 3])
def test_volume_256x512x512(factor):
    from invesalius3_b200 import phantom, resample
    vol = phantom.ct((256, 512, 512), seed=9)
    ref = ndi.zoom(vol, factor, vol.dtype, order=2)
    assert _same(resample.resize_image_array(vol, factor), ref)
