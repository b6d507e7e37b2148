"""Binary erosion and dilation on the device (invesalius3_b200.morphology) against SciPy, the callee behind
skimage's binary_erosion / binary_dilation, and against the restatement (oracle/morphology.py, pinned to
SciPy by tests/test_morphology_model.py) where SciPy takes tens of seconds. Every comparison is
np.array_equal."""
import numpy as np
import pytest
import torch
from scipy import ndimage as ndi

from oracle import morphology as om
from test_morphology_model import random_cases, scipy_morphology

pytestmark = pytest.mark.gpu


def _device(a: np.ndarray, op: str, r: int, planar: bool, threshold: int = 0) -> tuple[np.ndarray, int, int]:
    from invesalius3_b200 import morphology as mm
    t = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8) if a.dtype == np.bool_ else a).cuda()
    out, counts = mm.binary_morphology_device(t, op, r, planar, threshold=threshold, set_value=255)
    got = out.cpu().numpy()
    assert set(np.unique(got)) <= {0, 255}
    n_in, n_out = (int(v) for v in counts.cpu())
    return got == 255, n_in, n_out


@pytest.mark.parametrize("op", ["erosion", "dilation"])
@pytest.mark.parametrize("planar", [False, True])
def test_random_volumes_equal_scipy(op, planar):
    for shape, r, a in random_cases(11 + planar + 2 * (op == "dilation")):
        got, n_in, n_out = _device(a, op, r, planar)
        want = scipy_morphology(a, op, r, planar)
        assert np.array_equal(got, want), (shape, r, op, planar)
        assert (n_in, n_out) == (int(a.sum()), int(want.sum()))


@pytest.mark.parametrize("r", [1, 4, 7, 15])
def test_tiles_and_odd_rows(r):
    """Several 64 x 64 tiles per plane, rows that are not a multiple of four voxels, more than one z
    chunk, the largest radius, and a uint8 image where every non-zero value counts as set."""
    rng = np.random.default_rng(100 + r)
    for shape in [(70, 131, 129), (40, 64, 64), (3, 200, 67), (35, 66, 5)]:
        img = rng.choice(np.array([0, 1, 2, 127, 128, 254, 255], np.uint8), size=shape,
                         p=[0.55, 0.05, 0.05, 0.05, 0.1, 0.1, 0.1])
        a = img > 0
        for op in ("erosion", "dilation"):
            for planar in (False, True):
                got, n_in, n_out = _device(img, op, r, planar)
                want = om.binary_morphology(a, op, r, planar)
                assert np.array_equal(got, want), (shape, r, op, planar)
                assert (n_in, n_out) == (int(a.sum()), int(want.sum()))
    got, _, _ = _device(img, "dilation", r, False, threshold=127)
    assert np.array_equal(got, om.binary_morphology(img > 127, "dilation", r, False))
    if r <= 4:
        for op in ("erosion", "dilation"):
            assert np.array_equal(_device(img, op, r, False)[0], scipy_morphology(img > 0, op, r, False))


def test_more_planes_than_one_grid_dimension():
    """70000 z-slices: more than the 65535 blocks of one grid dimension."""
    rng = np.random.default_rng(5)
    a = rng.random((70000, 3, 6)) < 0.4
    for op in ("erosion", "dilation"):
        got, _, _ = _device(a, op, 2, False)
        assert np.array_equal(got, scipy_morphology(a, op, 2, False)), op
        got, _, _ = _device(a, op, 2, True)
        assert np.array_equal(got, om.binary_morphology(a, op, 2, True)), op


def test_drop_ins_equal_scipy():
    from invesalius3_b200 import morphology as mm
    rng = np.random.default_rng(7)
    for shape in [(17, 23, 30), (1, 40, 9), (6, 1, 33)]:
        for r in (0, 1, 3, 6):
            a = rng.random(shape) < 0.6
            for img in (a, a.astype(np.uint8) * np.uint8(200)):
                got = mm.binary_erosion(img, mm.ball(r))
                assert got.dtype == np.bool_ and np.array_equal(got, ndi.binary_erosion(img, mm.ball(r), border_value=1))
                got = mm.binary_dilation(img, mm.ball(r, dtype=bool))
                assert got.dtype == np.bool_ and np.array_equal(got, ndi.binary_dilation(img, mm.ball(r)))
            s = a[0]
            assert np.array_equal(mm.binary_erosion(s, mm.disk(r)), ndi.binary_erosion(s, mm.disk(r), border_value=1))
            assert np.array_equal(mm.binary_dilation(s, mm.disk(r)), ndi.binary_dilation(s, mm.disk(r)))
        a = rng.random(shape) < 0.5
        assert np.array_equal(mm.binary_erosion(a), ndi.binary_erosion(a, border_value=1))
        assert np.array_equal(mm.binary_dilation(a[0]), ndi.binary_dilation(a[0]))


def test_drop_ins_write_out():
    from invesalius3_b200 import morphology as mm
    rng = np.random.default_rng(8)
    a = rng.random((9, 31, 27)) < 0.5
    out = np.ones(a.shape, bool)
    res = mm.binary_dilation(a, mm.ball(2), out=out)
    assert res is out and np.array_equal(out, ndi.binary_dilation(a, mm.ball(2)))
    big = np.ones((9, 40, 40), bool)
    view = big[:, 3:34, 5:32]                      # a strided out
    res = mm.binary_erosion(a, mm.ball(3), out=view)
    assert res is view and np.array_equal(view, ndi.binary_erosion(a, mm.ball(3), border_value=1))
    assert big[:, :3].all() and big[:, 34:].all() and big[:, :, :5].all() and big[:, :, 32:].all()
    out2 = np.zeros(a.shape[1:], bool)
    res = mm.binary_erosion(a[4], mm.disk(4), out=out2)
    assert res is out2 and np.array_equal(out2, ndi.binary_erosion(a[4], mm.disk(4), border_value=1))


def _cranium(cranium) -> np.ndarray:
    shape = tuple(int(v) for v in cranium["full_shape"])
    return np.unpackbits(cranium["mask_0_bits_full"])[: int(np.prod(shape))].reshape(shape).astype(bool)


@pytest.mark.parametrize("r,planar", [(1, False), (3, False), (10, False), (10, True)])
def test_cranium_mask(cranium, r, planar):
    from invesalius3_b200 import morphology as mm
    a = _cranium(cranium)
    assert a.shape == (108, 256, 256)
    for op in ("erosion", "dilation"):
        if planar:
            got, n_in, n_out = _device(a, op, r, True)
        else:
            f = mm.binary_erosion if op == "erosion" else mm.binary_dilation
            got = f(a, mm.ball(r))
        quick = op == "erosion" or r <= 3
        want = scipy_morphology(a, op, r, planar) if quick else om.binary_morphology(a, op, r, planar)
        assert np.array_equal(got, want), (op, r, planar)
        assert want.sum() != a.sum()


def plugin_on_apply(matrix: np.ndarray, operation: int, radius: int, struct_type: int):
    """The plugin's OnApply restated with SciPy: foreground is > 0 in the body; disk per slice or ball;
    nothing when the mask or an erosion's result is empty; otherwise a fresh padded matrix whose first
    plane, row and column are 1 and whose body is 255 where the result is set."""
    body = matrix[1:, 1:, 1:] > 0
    if not body.any():
        return None
    result = scipy_morphology(body, "erosion" if operation == 0 else "dilation", radius, struct_type == 0)
    if operation == 0 and not result.any():
        return None
    new = np.zeros_like(matrix)
    new[0, :, :] = 1
    new[:, 0, :] = 1
    new[:, :, 0] = 1
    new[1:, 1:, 1:] = np.where(result, 255, 0)
    return new


def _marked_mask(shape, seed):
    """A padded mask whose body holds 0, the markers 1 / 2 / 253 / 254 and 255: a solid ellipsoid of
    mixed non-zero values (so that erosions up to r = 3 leave voxels) in sparse noise of all six."""
    rng = np.random.default_rng(seed)
    m = np.zeros(tuple(n + 1 for n in shape), np.uint8)
    values = np.array([0, 1, 2, 253, 254, 255], np.uint8)
    body = rng.choice(values, size=shape, p=[0.85, 0.03, 0.03, 0.03, 0.03, 0.03])
    z, y, x = np.indices(shape)
    inside = sum(((c - (n - 1) / 2) / (0.4 * n)) ** 2 for c, n in zip((z, y, x), shape)) <= 1
    body[inside] = rng.choice(values[1:], size=int(inside.sum()))
    m[1:, 1:, 1:] = body
    m[0, :, :] = rng.integers(0, 3, m.shape[1:])     # slice flags: the result overwrites them with 1
    m[:, 0, :] = 7
    m[:, :, 0] = 9
    return m


@pytest.mark.parametrize("struct_type", [0, 1])
@pytest.mark.parametrize("operation", [0, 1])
def test_mask_morphology_equals_plugin(operation, struct_type):
    from invesalius3_b200 import morphology as mm
    m = _marked_mask((21, 34, 29), 30 + 2 * operation + struct_type)
    before = int((m[1:, 1:, 1:] > 0).sum())
    for r in (1, 2, 3):
        want = plugin_on_apply(m, operation, r, struct_type)
        got, n_before, n_after = mm.mask_morphology(m, operation, r, struct_type)
        assert want is not None and got.dtype == np.uint8 and np.array_equal(got, want), (operation, r, struct_type)
        assert (n_before, n_after) == (before, int((want[1:, 1:, 1:] == 255).sum()))


def test_mask_morphology_unchanged_cases():
    from invesalius3_b200 import morphology as mm
    empty = np.zeros((6, 9, 11), np.uint8)
    empty[0] = 1
    empty[:, 0] = 1
    for op in (0, 1):
        for st in (0, 1):
            assert mm.mask_morphology(empty, op, 2, st) == (None, 0, 0)
    small = np.zeros((8, 10, 12), np.uint8)
    small[3:5, 4:7, 5:8] = 255                      # 2 x 3 x 3: ball(2) and disk(2) erode it away
    for st in (0, 1):
        assert plugin_on_apply(small, 0, 2, st) is None
        assert mm.mask_morphology(small, 0, 2, st) == (None, 18, 0)
        new, n0, n1 = mm.mask_morphology(small, 1, 2, st)
        assert np.array_equal(new, plugin_on_apply(small, 1, 2, st)) and (n0, n1) == (18, int((new[1:, 1:, 1:] == 255).sum()))
    new, n0, n1 = mm.mask_morphology(small, 0, 0, 1)   # r = 0 is the identity
    assert (n0, n1) == (18, 18) and np.array_equal(new[1:, 1:, 1:], small[1:, 1:, 1:])


def test_memmap_views(tmp_path):
    """The padded mask as an np.memmap, its [1:, 1:, 1:] view through the drop-ins, and mask_morphology."""
    from invesalius3_b200 import morphology as mm
    m = _marked_mask((19, 45, 38), 40)
    mm_arr = np.memmap(tmp_path / "mask.dat", np.uint8, "w+", shape=m.shape)
    mm_arr[...] = m
    view = mm_arr[1:, 1:, 1:]
    assert not view.flags.c_contiguous
    for r in (1, 3):
        assert np.array_equal(mm.binary_dilation(view, mm.ball(r)), ndi.binary_dilation(view, mm.ball(r)))
        assert np.array_equal(mm.binary_erosion(view[5], mm.disk(r)),
                              ndi.binary_erosion(view[5], mm.disk(r), border_value=1))
        for op in (0, 1):
            for st in (0, 1):
                got, _, _ = mm.mask_morphology(mm_arr, op, r, st)
                assert np.array_equal(got, plugin_on_apply(m, op, r, st)), (r, op, st)
    assert np.array_equal(mm_arr, m)               # the input is not written
