"""The whole-volume formulation of the "2D" image-filter branch (tests/filters_2d_model.py, what the device
computes: no pass along the slice axis, per-slice statistics and normalisation) against the per-slice SciPy loop,
bit for bit, the unit-bin histogram against np.histogram, and the argument checks of invesalius3_b200.filters
that run before any device work."""
import numpy as np
import pytest
from scipy import ndimage

import filters_2d_model as fm

ORIENTATIONS = ["Axial", "Coronal", "Sagittal"]
# the dialog's reachable values: sigma 0.1-10, mean "kernel size" -> size 2 value + 1, median always capped at 5
CASES = [(0, 0.1), (0, 1.0), (0, 2.5), (0, 10.0), (1, 1.0), (1, 1.5), (1, 3.0), (2, 0.5), (2, 1.0), (2, 3.0),
         (2, 15.0), (3, 1.0), (3, 2.5), (4, 1.0), (4, 10.0), (5, 0.1), (5, 1.0), (5, 2.5), (5, 10.0)]


@pytest.mark.parametrize("orientation", ORIENTATIONS)
@pytest.mark.parametrize("filter_type,value", CASES)
def test_whole_volume_equals_slice_loop(filter_type, value, orientation):
    vol = fm.image((7, 10, 13), 5, constant_slices=[(0, 2, 300), (1, 4, -7), (2, 6, 1200)])
    want = fm.loop_2d(vol, filter_type, value, orientation)
    assert np.array_equal(fm.whole_volume_2d(vol, filter_type, value, orientation), want)


@pytest.mark.parametrize("shape", [(5, 1, 9), (5, 2, 9), (5, 3, 9), (6, 8, 1), (6, 8, 2), (1, 3, 2), (4, 1, 1)])
def test_thin_slices(shape):
    """In-slice dimensions of 1, 2 and 3, thinner than every window and Gaussian radius."""
    vol = fm.image(shape, sum(shape))
    for orientation in ORIENTATIONS + ["Oblique"]:
        for filter_type, value in CASES:
            want = fm.loop_2d(vol, filter_type, value, orientation)
            got = fm.whole_volume_2d(vol, filter_type, value, orientation)
            assert np.array_equal(got, want), (shape, orientation, filter_type, value)


def test_slice_axis_is_skipped_not_filtered_at_length_one():
    """A Gaussian pass along a length-1 axis is not the identity on int16, so a slice is not a (1, ny, nx) volume."""
    vol = fm.image((3, 40, 41), 11)
    s = 1.3
    per_slice = np.stack([ndimage.gaussian_filter(v, sigma=s) for v in vol])
    assert np.array_equal(ndimage.gaussian_filter(vol, sigma=(0, s, s)), per_slice)
    assert not all(np.array_equal(ndimage.gaussian_filter(v[None], sigma=s)[0], w) for v, w in zip(vol, per_slice))


def test_unknown_filter_and_orientation():
    vol = fm.image((4, 5, 6), 1)
    assert fm.loop_2d(vol, 6, 1.0) is None and fm.filter_3d(vol, -1, 1.0) is None
    assert np.array_equal(fm.loop_2d(vol, 0, 1.0, "Oblique"), fm.loop_2d(vol, 0, 1.0, "Axial"))


def test_histogram_is_unit_bins():
    from invesalius3_b200 import phantom
    for a in (phantom.ct((24, 40, 56), seed=2), np.array([[[5, 9], [9, 9]]], np.int16),
              np.array([-32768, 32767, 0], np.int16), fm.image((6, 7, 8), 3)):
        i, e = a.min(), a.max()
        r = int(e) - int(i)
        assert np.array_equal(np.histogram(a, r, (i, e))[0], fm.histogram_by_count(a))
    a = np.full((3, 4, 5), 17, np.int16)
    with pytest.raises(ValueError, match="`bins` must be positive"):
        np.histogram(a, int(a.max()) - int(a.min()), (a.min(), a.max()))


def test_argument_checks_before_device_work():
    from invesalius3_b200 import filters
    vol = np.zeros((4, 5, 6), np.int16)
    for fn in (filters.median_blur_filter, filters.mean_blur_filter, filters.gaussian_blur_filter,
               filters.sharpening_filter, filters.despeckle_filter, filters.border_detection_filter):
        with pytest.raises(TypeError):
            fn(vol.astype(np.float32), 1.0)
        with pytest.raises(TypeError):
            fn(vol[0].astype(np.float64), 1.0)
        with pytest.raises(TypeError):
            fn(vol[0, 0], 1.0)                      # 1-D
    for m in (vol, vol[:, 2, :]):
        with pytest.raises(RuntimeError, match="incorrect filter size"):
            filters.mean_blur_filter(m, -1.0)
    with pytest.raises(RuntimeError, match="incorrect filter size"):
        filters.apply_image_filter(vol, 2, -1.0, "2D", "Coronal")
    for ft in (6, -1, None, "0"):
        assert filters.apply_image_filter(vol, ft, 1.0) is None
        assert filters.apply_image_filter(vol, ft, 1.0, "2D", "Sagittal") is None
    with pytest.raises(TypeError):
        filters.apply_image_filter(vol.astype(np.uint8), 0, 1.0)
    with pytest.raises(TypeError):
        filters.apply_image_filter(vol[0], 0, 1.0, "2D")
    with pytest.raises(TypeError):
        filters.image_histogram(vol.astype(np.float64))
