"""The binary-morphology restatement (oracle/morphology.py) against SciPy, the footprints against their
formulas, and the host-side argument checks of invesalius3_b200.morphology (CPU only: every check here
raises before any device work).

The mask-morphology plugin erodes or dilates with skimage's disk(r) on every axial slice or ball(r) on the
volume; skimage's binary_erosion / binary_dilation are SciPy's with border_value 1 / 0."""
import numpy as np
import pytest
from scipy import ndimage as ndi

from invesalius3_b200 import morphology as mm
from oracle import morphology as om

RADII = [0, 1, 2, 3, 5, 10]
SHAPES = [(1, 1, 9), (1, 1, 1), (1, 7, 12), (1, 23, 5), (5, 9, 13), (7, 4, 11), (3, 3, 3), (12, 2, 17), (9, 15, 1)]


def scipy_morphology(a: np.ndarray, op: str, r: int, planar: bool) -> np.ndarray:
    """What the plugin computes, with SciPy as the callee: disk per z-slice, or ball on the volume."""
    if op == "erosion":
        f = lambda img, fp: ndi.binary_erosion(img, fp, border_value=1)    # noqa: E731
    else:
        f = lambda img, fp: ndi.binary_dilation(img, fp, border_value=0)   # noqa: E731
    if planar:
        return np.stack([f(s, mm.disk(r)) for s in a]).reshape(a.shape)
    return f(a, mm.ball(r))


def random_cases(seed: int):
    rng = np.random.default_rng(seed)
    for shape in SHAPES:
        for r in RADII:
            p = rng.choice([0.03, 0.3, 0.5, 0.9, 0.995])
            yield shape, r, rng.random(shape) < p


def test_disk_and_ball_formulas():
    for r in range(0, 16):
        ax = np.arange(-r, r + 1)
        d = mm.disk(r)
        assert d.dtype == np.uint8 and d.shape == (2 * r + 1,) * 2
        assert np.array_equal(d, (ax[:, None] ** 2 + ax[None, :] ** 2 <= r * r).astype(np.uint8))
        b = mm.ball(r)
        assert b.dtype == np.uint8 and b.shape == (2 * r + 1,) * 3
        assert np.array_equal(b, (ax[:, None, None] ** 2 + ax[None, :, None] ** 2 + ax[None, None, :] ** 2
                                  <= r * r).astype(np.uint8))
    assert mm.disk(2, dtype=bool).dtype == np.bool_
    assert np.array_equal(mm.disk(1), ndi.generate_binary_structure(2, 1))
    assert np.array_equal(mm.ball(1), ndi.generate_binary_structure(3, 1))
    assert [int(mm.disk(r).sum()) for r in (1, 2, 10)] == [5, 13, 317]
    assert [int(mm.ball(r).sum()) for r in (1, 2, 3, 10)] == [7, 33, 123, 4169]


@pytest.mark.parametrize("op", ["erosion", "dilation"])
@pytest.mark.parametrize("planar", [False, True])
def test_oracle_equals_scipy(op, planar):
    n = 0
    for shape, r, a in random_cases(1 + planar + 2 * (op == "dilation")):
        got = om.binary_morphology(a, op, r, planar)
        want = scipy_morphology(a, op, r, planar)
        assert got.dtype == np.bool_ and np.array_equal(got, want), (shape, r, op, planar)
        n += 1
    assert n == len(SHAPES) * len(RADII)


def test_oracle_edge_cases():
    """All set, none set, one voxel, and r beyond every dimension."""
    for shape in [(4, 5, 6), (1, 3, 3), (2, 1, 8)]:
        for a in (np.ones(shape, bool), np.zeros(shape, bool)):
            for r in (0, 2, 10):
                for op in ("erosion", "dilation"):
                    for planar in (False, True):
                        assert np.array_equal(om.binary_morphology(a, op, r, planar),
                                              scipy_morphology(a, op, r, planar))
    a = np.zeros((9, 9, 9), bool)
    a[4, 4, 4] = True
    assert np.array_equal(om.binary_morphology(a, "dilation", 3, False)[1:8, 1:8, 1:8], mm.ball(3).astype(bool))
    b = ~a
    assert int(om.binary_morphology(b, "erosion", 1, False).sum()) == b.sum() - 6


def test_argument_checks():
    img3 = np.zeros((3, 4, 5), bool)
    img2 = np.zeros((4, 5), np.uint8)
    with pytest.raises(NotImplementedError):
        mm.binary_erosion(img3.astype(np.int16))
    with pytest.raises(NotImplementedError):
        mm.binary_dilation(img2.astype(np.float32))
    with pytest.raises(NotImplementedError):
        mm.binary_erosion(np.zeros((2, 2, 2, 2), bool))
    with pytest.raises(RuntimeError, match="same dimensionality"):
        mm.binary_erosion(img3, mm.disk(1))
    with pytest.raises(RuntimeError, match="same dimensionality"):
        mm.binary_dilation(img2, mm.ball(2))
    with pytest.raises(NotImplementedError):
        mm.binary_erosion(img3, np.ones((3, 3, 3), np.uint8))     # a cube, not a ball
    with pytest.raises(NotImplementedError):
        mm.binary_dilation(img2, np.ones((2, 2), np.uint8))
    with pytest.raises(NotImplementedError):
        mm.binary_dilation(img2, np.ones((3, 5), np.uint8))
    with pytest.raises(NotImplementedError):
        mm.binary_erosion(img3, mm.ball(16))
    with pytest.raises(NotImplementedError):
        mm.binary_erosion(img3, out=np.zeros((3, 4, 5), np.uint8))
    with pytest.raises(NotImplementedError):
        mm.binary_erosion(img3, out=np.zeros((3, 4, 6), bool))
    with pytest.raises(ValueError):
        mm.disk(-1)
    with pytest.raises(ValueError):
        mm.ball(-2)
    with pytest.raises(TypeError):
        mm.disk(1.5)
    pad = np.zeros((4, 5, 6), np.uint8)
    with pytest.raises(ValueError):
        mm.mask_morphology(pad, 0, -1, 1)
    with pytest.raises(NotImplementedError):
        mm.mask_morphology(pad, 1, 16, 0)
    with pytest.raises(ValueError):
        mm.mask_morphology(pad, 2, 1, 0)
    with pytest.raises(ValueError):
        mm.mask_morphology(pad, 0, 1, 2)
    with pytest.raises(TypeError):
        mm.mask_morphology(pad.astype(np.int16), 0, 1, 0)


def test_footprint_recognition():
    """disk(r) / ball(r) in any dtype (SciPy reads non-zero as part of the element) give r; None gives 1."""
    assert mm._footprint_radius(None, 2) == 1 and mm._footprint_radius(None, 3) == 1
    for r in (0, 1, 4, 15):
        assert mm._footprint_radius(mm.disk(r), 2) == r
        assert mm._footprint_radius(mm.ball(r, dtype=bool), 3) == r
        assert mm._footprint_radius(mm.ball(r).astype(np.int64) * 3, 3) == r
    assert mm._footprint_radius(ndi.generate_binary_structure(3, 1), 3) == 1
