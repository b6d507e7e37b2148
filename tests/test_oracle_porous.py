"""The porous-scaffold checker (oracle/porous.py) pinned on the CPU: its broadcast TPMS against the 1-D-table order
that b2v_tpms_f64 evaluates (include/b2v.h), its Gaussian against scipy.ndimage.gaussian_filter and its normalise
against the formula, all bit for bit (int64 views for float64)."""
import numpy as np
import pytest
from scipy import ndimage as ndi

from oracle import porous as op


def _bits_equal(a, b):
    return a.dtype == b.dtype == np.float64 and a.shape == b.shape and np.array_equal(a.view(np.int64),
                                                                                       b.view(np.int64))


def table_model(method, init_x, end_x, init_y, end_y, init_z, end_z, sx, sy, sz):
    """The device's evaluation: cos / sin of the 1-D axes, then each product and sum in the header's order."""
    z, y, x = op.axes(init_x, end_x, init_y, end_y, init_z, end_z, sx, sy, sz)
    cx, snx = np.cos(x.ravel())[None, None, :], np.sin(x.ravel())[None, None, :]
    cy, sny = np.cos(y.ravel())[None, :, None], np.sin(y.ravel())[None, :, None]
    cz, snz = np.cos(z.ravel())[:, None, None], np.sin(z.ravel())[:, None, None]
    if method == "Schwarz P":
        return (cx + cy) + cz
    if method == "Schwarz D":
        return (((snx * sny) * snz + (snx * cy) * cz) + (cx * sny) * cz) + (cx * cy) * snz
    if method == "Gyroid":
        return (cx * sny + cy * snz) + cz * snx
    if method == "Neovius":
        return 3.0 * ((cx + cy) + cz) + ((4.0 * cx) * cy) * cz
    if method == "iWP":
        return ((cx * cy + cy * cz) + cz * cx) - (cx * cy) * cz
    return (4.0 * ((cx * cy + cy * cz) + cz * cx) - ((3.0 * cx) * cy) * cz) + 2.4


ARGS = [
    (-10, 10, -10, 10, -10, 10, 25, 25, 25),
    (-10.0, 10.0, -10.0, 10.0, 1.0, 1.0, 250, 250, 1),       # the preview
    (0, 1, 0, 1, 0, 1, 1, 1, 1),
    (0.5, 0.5, -3.3, 7.1, 2.0, 2.0, 2, 3, 2),               # equal bounds
    (10, -10, 4.2, -4.2, 3, -7.5, 17, 9, 5),                # reversed
    (-1000.0, 1000.0, -0.1, 0.1, -123.4, 567.8, 31, 7, 11),
    (-np.pi, np.pi, -2 * np.pi, 2 * np.pi, 0.3, 0.3, 97, 83, 1),
    (-10, 10, -10, 10, -10, 10, 0, 4, 4),                   # empty
]


@pytest.mark.parametrize("method", op.SURFACES)
@pytest.mark.parametrize("args", ARGS)
def test_broadcast_form_equals_table_order(method, args):
    want = table_model(method, *args)
    got = op.create_schwarzp(method, *args)
    assert got.shape == (args[8], args[7], args[6])
    assert _bits_equal(got, want)


def test_unknown_method():
    assert op.create_schwarzp("Voronoi", -10, 10, -10, 10, -10, 10, 4, 4, 4) is None


@pytest.mark.parametrize("method", ["Schwarz D", "P_W_Hybrid", "Gyroid"])
@pytest.mark.parametrize("slab", [1, 4, 64])
def test_slabs_equal_whole_normalise(method, slab):
    args = (-10, 10, -7.5, 9.25, -3, 12, 29, 23, 19)
    want = op.image_normalize(op.create_schwarzp(method, *args), -1000, 1000)
    assert np.array_equal(op.schwarzp_i16_slabs(method, *args, slab=slab), want)


def test_slabs_constant_field():
    got = op.schwarzp_i16_slabs("iWP", 2.0, 2.0, 2.0, 2.0, 2.0, 2.0, 5, 6, 7, slab=3)
    assert got.dtype == np.int16 and (got == -1000).all()


@pytest.mark.parametrize("sigma", [0.0, 1e-16, 0.1, 0.124, 0.125, 1.5, 5.0, 10.0])
@pytest.mark.parametrize("shape", [(1, 25, 31), (7, 5, 11), (13, 12, 3)])
def test_gaussian_equals_scipy(shape, sigma):
    rng = np.random.default_rng(7)
    a = rng.random(shape)
    assert _bits_equal(op.gaussian(a, sigma), ndi.gaussian_filter(a, sigma))


def test_blobs_draw_and_state():
    np.random.seed(11)
    got = op.create_blobs(13, 9, 5, 1.5)
    state = np.random.get_state()
    np.random.seed(11)
    want = ndi.gaussian_filter(np.random.random((5, 9, 13)), 1.5)
    assert _bits_equal(got, want)
    assert all(np.array_equal(a, b) for a, b in zip(state, np.random.get_state()))


def _formula(image, min_, max_):
    out = np.empty(image.shape, np.int16)
    lo, hi = image.min(), image.max()
    out[...] = min_ if lo == hi else (image - lo) * ((max_ - min_) / (hi - lo)) + min_
    return out


@pytest.mark.parametrize("bounds", [(0, 255), (-1000, 1000), (-12.5, 300.75)])
@pytest.mark.parametrize("shape", [(40, 33), (5, 6, 7)])
def test_normalise_formula(shape, bounds):
    a = np.random.default_rng(3).normal(size=shape) * 50
    got = op.image_normalize(a, *bounds)
    assert got.dtype == np.int16 and np.array_equal(got, _formula(a, *bounds))


def test_normalise_constant_and_empty():
    assert (op.image_normalize(np.full((3, 4), 2.5), -7, 9) == -7).all()
    with pytest.raises(ValueError):
        op.image_normalize(np.empty((0, 3)), 0, 255)
