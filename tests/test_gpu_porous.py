"""The TPMS and Blobs scaffolds and the float64 image_normalize on the device (invesalius3_b200.porous) against the
NumPy / SciPy checker (oracle/porous.py): float64 results compared on their int64 views, int16 exactly."""
import numpy as np
import pytest
from scipy import ndimage as ndi

from oracle import porous as op

pytestmark = pytest.mark.gpu

SURFACES = op.SURFACES
DEFAULT = (-10.0, 10.0, -10.0, 10.0, -10.0, 10.0)


def _bits_equal(a, b):
    return (a.dtype == b.dtype == np.float64 and a.shape == b.shape
            and np.array_equal(a.view(np.int64), b.view(np.int64)))


def _i16_equal(a, b):
    return a.dtype == b.dtype == np.int16 and a.shape == b.shape and np.array_equal(a, b)


@pytest.mark.parametrize("method", SURFACES)
@pytest.mark.parametrize("args", [
    (-10.0, 10.0, -10.0, 10.0, 1.0, 1.0, 250, 250, 1),       # the dialog's preview
    (-10, 10, -7.5, 12.25, 3.0, -4.5, 97, 83, 71),
    (5.0, -5.0, 0.1, 0.1, -1000.0, 1000.0, 2, 1, 33),
    (*DEFAULT, 250, 250, 250),
])
def test_schwarzp_f64(method, args):
    from invesalius3_b200 import porous
    assert _bits_equal(porous.create_schwarzp(method, *args), op.create_schwarzp(method, *args))


def test_schwarzp_unknown_method_and_errors():
    from invesalius3_b200 import porous
    assert porous.create_schwarzp("Blobs", *DEFAULT, 8, 8, 8) is None
    assert porous.create_schwarzp_i16("Voronoi", *DEFAULT, 8, 8, 8) is None
    assert porous.create_schwarzp("Gyroid", *DEFAULT, 0, 5, 5).shape == (5, 5, 0)
    with pytest.raises(ValueError):
        porous.create_schwarzp_i16("Gyroid", *DEFAULT, 0, 5, 5)
    bad = ("Gyroid", "a", 10, -10, 10, -10, 10, 4, 4, 4)
    with pytest.raises(Exception) as numpy_error:   # whatever np.ogrid raises
        op.create_schwarzp(*bad)
    with pytest.raises(numpy_error.type):
        porous.create_schwarzp(*bad)
    with pytest.raises(numpy_error.type):
        porous.create_schwarzp_i16(*bad)


@pytest.mark.parametrize("method", SURFACES)
def test_schwarzp_i16_default(method):
    from invesalius3_b200 import porous
    args = (*DEFAULT, 250, 250, 250)
    want = op.image_normalize(op.create_schwarzp(method, *args), -1000, 1000)
    assert _i16_equal(porous.create_schwarzp_i16(method, *args), want)
    assert _i16_equal(porous.create_schwarzp_i16(method, *args, min_=0, max_=255),
                      op.image_normalize(op.create_schwarzp(method, *args), 0, 255))


@pytest.mark.parametrize("method", SURFACES)
def test_schwarzp_i16_constant_field(method):
    """All bounds equal: every voxel has one value, and image_normalize fills with min_."""
    from invesalius3_b200 import porous
    args = (2.5, 2.5, 2.5, 2.5, 2.5, 2.5, 250, 250, 250)
    got = porous.create_schwarzp_i16(method, *args)
    assert _i16_equal(got, op.image_normalize(op.create_schwarzp(method, *args), -1000, 1000))
    assert (got == -1000).all()
    with pytest.raises(OverflowError):
        porous.create_schwarzp_i16(method, *args[:6], 3, 3, 3, min_=40000, max_=50000)
    # a min_ that int16 cannot hold only matters for a constant image
    vary = (*DEFAULT, 5, 5, 5)
    assert _i16_equal(porous.create_schwarzp_i16(method, *vary, min_=40000, max_=50000),
                      op.image_normalize(op.create_schwarzp(method, *vary), 40000, 50000))


@pytest.mark.parametrize("method", ["Schwarz D", "P_W_Hybrid"])
def test_schwarzp_i16_full_size(method):
    """The spin controls' largest volume, 1000^3: the checker never holds the float64 field."""
    from invesalius3_b200 import porous
    args = (*DEFAULT, 1000, 1000, 1000)
    got = porous.create_schwarzp_i16(method, *args)
    assert _i16_equal(got, op.schwarzp_i16_slabs(method, *args, slab=25))


@pytest.mark.parametrize("sigma", [0.0, 0.1, 1.5, 5.0, 10.0])
@pytest.mark.parametrize("shape", [(1, 250, 250), (37, 50, 61), (250, 250, 250), (100, 1000, 1000)])
def test_blobs(shape, sigma):
    from invesalius3_b200 import porous
    sz, sy, sx = shape
    np.random.seed(1234)
    got = porous.create_blobs(sx, sy, sz, sigma)
    state = np.random.get_state()
    np.random.seed(1234)
    want = op.create_blobs(sx, sy, sz, sigma)
    assert all(np.array_equal(a, b) for a, b in zip(state, np.random.get_state()))
    assert _bits_equal(got, want)
    want_i16 = op.image_normalize(want, -1000, 1000)
    del got, want
    np.random.seed(1234)
    assert _i16_equal(porous.create_blobs_i16(sx, sy, sz, sigma), want_i16)
    assert all(np.array_equal(a, b) for a, b in zip(state, np.random.get_state()))


def test_blobs_against_scipy_directly():
    from invesalius3_b200 import porous
    np.random.seed(5)
    got = porous.create_blobs(61, 50, 37, 5)
    np.random.seed(5)
    assert _bits_equal(got, ndi.gaussian_filter(np.random.random((37, 50, 61)), sigma=5))


@pytest.mark.parametrize("bounds", [(0, 255), (-1000, 1000), (-12.5, 300.75), (np.float32(-3.3), 7.7)])
@pytest.mark.parametrize("shape", [(250, 250), (1, 250, 250), (23, 41, 57)])
def test_image_normalize_f64(shape, bounds):
    from invesalius3_b200 import porous
    a = np.random.default_rng(9).normal(size=shape) * 300
    assert _i16_equal(porous.image_normalize(a, *bounds), op.image_normalize(a, *bounds))


def test_image_normalize_f64_edges():
    from invesalius3_b200 import porous, voronoi
    c = np.full((17, 19), -4.25)
    assert _i16_equal(porous.image_normalize(c, 3, 9), op.image_normalize(c, 3, 9))
    with pytest.raises(ValueError):
        porous.image_normalize(np.empty((0, 4)), 0, 255)
    with pytest.raises(OverflowError):
        porous.image_normalize(c, 70000, 80000)
    nan = np.arange(12.0).reshape(3, 4)
    nan[1, 2] = np.nan
    with np.errstate(invalid="ignore"):
        assert _i16_equal(porous.image_normalize(nan, 0, 255), op.image_normalize(nan, 0, 255))
    f32 = np.random.default_rng(2).random((9, 8), dtype=np.float32)
    assert _i16_equal(porous.image_normalize(f32, 0, 255), voronoi.image_normalize(f32, 0, 255))
    with pytest.raises(NotImplementedError):
        voronoi.image_normalize(c, 0, 255)
