"""The image-filter action on the device (invesalius3_b200.filters.apply_image_filter, the 2-D mode of the six
filters, image_histogram) against SciPy / NumPy, bit for bit. The oracle of the "2D" branch is the reference's
per-slice loop restated with SciPy calls (tests/filters_2d_model.py)."""
import numpy as np
import pytest
from scipy import ndimage

import filters_2d_model as fm
from test_filters_2d_model import CASES, ORIENTATIONS

pytestmark = pytest.mark.gpu


def _odd_volume():
    return fm.image((9, 14, 17), 7, constant_slices=[(0, 3, 250), (1, 5, -40), (2, 8, 1111), (2, 16, 0)])


@pytest.mark.parametrize("orientation", ORIENTATIONS)
@pytest.mark.parametrize("filter_type,value", CASES)
def test_2d_branch_equals_slice_loop(filter_type, value, orientation):
    import torch
    from invesalius3_b200 import device as dev, filters
    vol = _odd_volume()
    want = fm.loop_2d(vol, filter_type, value, orientation)
    got = filters.apply_image_filter(vol, filter_type, value, "2D", orientation)
    assert got.dtype == np.int16 and np.array_equal(got, want)
    t = dev.to_device(vol)
    out = filters.apply_image_filter_device(t, filter_type, value, "2D", orientation)
    assert out.dtype == torch.int16 and np.array_equal(out.cpu().numpy(), want)
    assert np.array_equal(t.cpu().numpy(), vol)          # the input is left alone


@pytest.mark.parametrize("filter_type,value", CASES)
def test_3d_branch_equals_scipy(filter_type, value):
    from invesalius3_b200 import filters
    vol = fm.image((11, 13, 10), 3, constant_slices=[(0, 4, 77)])
    assert np.array_equal(filters.apply_image_filter(vol, filter_type, value, "3D"), fm.filter_3d(vol, filter_type, value))


@pytest.mark.parametrize("shape", [(5, 1, 9), (5, 2, 9), (5, 3, 9), (6, 8, 1), (6, 8, 2), (6, 3, 3), (1, 3, 2), (4, 1, 1)])
def test_thin_slices(shape):
    """In-slice dimensions of 1, 2 and 3: thinner than the windows and than the Gaussian radius at sigma 10."""
    from invesalius3_b200 import filters
    vol = fm.image(shape, sum(shape), constant_slices=[(1, 0, 9)])
    for orientation in ORIENTATIONS:
        for filter_type, value in CASES:
            want = fm.loop_2d(vol, filter_type, value, orientation)
            got = filters.apply_image_filter(vol, filter_type, value, "2D", orientation)
            assert np.array_equal(got, want), (shape, orientation, filter_type, value)


def test_dispatch_like_the_reference():
    from invesalius3_b200 import filters
    vol = _odd_volume()
    for ft in (6, -1, None):
        assert filters.apply_image_filter(vol, ft, 1.0, "2D") is None
    # any dimension but "3D" is the 2-D branch; an unknown orientation is axial
    want = fm.loop_2d(vol, 5, 1.0, "Axial")
    for dimension, orientation in (("2D", "Oblique"), ("2d", "Axial"), ("", None)):
        assert np.array_equal(filters.apply_image_filter(vol, 5, 1.0, dimension, orientation), want)
    with pytest.raises(RuntimeError, match="incorrect filter size"):
        filters.apply_image_filter(vol, 2, -3.0, "3D")


def test_constant_slices():
    """Per-slice mag_range == 0 (a cast without normalisation) and sharpening clipped to [v, v]."""
    from invesalius3_b200 import filters
    vol = fm.image((6, 9, 10), 4)
    vol[:, 4, :] = -123
    vol[2] = 5
    vol[:, :, 0] = 0
    for orientation in ORIENTATIONS:
        for filter_type, value in ((3, 1.0), (3, 10.0), (5, 1.0), (5, 0.1)):
            want = fm.loop_2d(vol, filter_type, value, orientation)
            assert np.array_equal(filters.apply_image_filter(vol, filter_type, value, "2D", orientation), want)
    flat = np.full((3, 4, 5), 321, np.int16)
    for filter_type in range(6):
        assert np.array_equal(filters.apply_image_filter(flat, filter_type, 1.0, "2D", "Coronal"),
                              fm.loop_2d(flat, filter_type, 1.0, "Coronal"))


def test_2d_functions_are_drop_ins():
    """filters.py's six functions on one 2-D slice, strided views included, as the reference's loop calls them."""
    from invesalius3_b200 import filters
    matrix = fm.image((12, 15, 11), 9)
    sl = matrix[:, 7, :]
    assert np.array_equal(filters.median_blur_filter(sl, 3.0), ndimage.median_filter(sl, size=5))
    fns = {0: lambda a, v: filters.gaussian_blur_filter(a, sigma=v), 1: filters.median_blur_filter,
           2: filters.mean_blur_filter, 3: filters.sharpening_filter, 4: filters.despeckle_filter,
           5: lambda a, v: filters.border_detection_filter(a, value=v)}
    for sl in (matrix[4], matrix[:, 7, :], matrix[:, :, 3], np.ascontiguousarray(matrix[:, :, 10])):
        for filter_type, value in CASES:
            got = fns[filter_type](sl, value)
            assert got.shape == sl.shape and np.array_equal(got, fm._filter(sl, filter_type, value)), (filter_type, value)
    sl = matrix[5]
    f = ndimage.gaussian_filter(sl.astype(float), sigma=2.0)
    want = np.sqrt(ndimage.sobel(f, axis=0) ** 2 + ndimage.sobel(f, axis=1) ** 2).astype(np.int16)
    assert np.array_equal(filters.border_detection_filter(sl, 2.0, normalize=False), want)


def test_launches_do_not_grow_with_slices():
    """The 2-D branch filters every slice in the same launches."""
    from invesalius3_b200 import _lib, filters
    lib = _lib.load()
    counts = {}
    for nz in (3, 40):
        vol = fm.image((nz, 20, 24), nz)
        for filter_type in range(6):
            lib.b2v_launch_count_reset()
            filters.apply_image_filter(vol, filter_type, 1.0, "2D", "Axial")
            counts[nz, filter_type] = lib.b2v_launch_count()
    for filter_type in range(6):
        assert counts[3, filter_type] == counts[40, filter_type], counts


def test_image_histogram():
    import torch
    from invesalius3_b200 import device as dev, filters, phantom
    ct = phantom.ct((64, 96, 80), seed=2)
    two = np.where(fm.image((7, 8, 9), 1) > 0, 3071, -1024).astype(np.int16)
    wide = fm.image((5, 6, 7), 2)
    wide[0, 0, 0], wide[4, 5, 6] = -32768, 32767          # 65535 bins: more than shared memory holds
    for a in (ct, two, wide, ct[:, 3, :], ct[10:20, 5:50, 7:70]):
        i, e = a.min(), a.max()
        want = np.histogram(a, int(e) - int(i), (i, e))[0]
        h, lo, hi = filters.image_histogram(a)
        assert (lo, hi) == (i, e) and type(lo) is np.int16 and h.dtype == want.dtype and np.array_equal(h, want)
        counts, lo, hi = filters.image_histogram_device(dev.to_device(np.ascontiguousarray(a)))
        assert (lo, hi) == (int(i), int(e)) and counts.dtype == torch.int64 and np.array_equal(counts.cpu().numpy(), want)
    flat = np.full((4, 5, 6), -7, np.int16)
    with pytest.raises(ValueError, match="`bins` must be positive"):
        np.histogram(flat, 0, (flat.min(), flat.max()))
    with pytest.raises(ValueError, match="`bins` must be positive"):
        filters.image_histogram(flat)


@pytest.mark.parametrize("orientation", ORIENTATIONS)
def test_full_size(orientation):
    """256 x 512 x 512: border detection (Gaussian, 2-D sobel, per-slice normalisation) on the CT phantom, and the
    median (about 40 s per orientation in SciPy at this size) on a 64 x 256 x 256 phantom."""
    from invesalius3_b200 import filters, phantom
    vol = phantom.ct((256, 512, 512), seed=2)
    assert np.array_equal(filters.apply_image_filter(vol, 5, 1.0, "2D", orientation), fm.loop_2d(vol, 5, 1.0, orientation))
    del vol
    small = phantom.ct((64, 256, 256), seed=3)
    assert np.array_equal(filters.apply_image_filter(small, 1, 3.0, "2D", orientation),
                          fm.loop_2d(small, 1, 3.0, orientation))
