"""The slab projections (device.mip: MaxIP / MinIP / MeanIP, slice_.py:881-886) against NumPy on the
paths test_gpu_threshold_mip.py does not reach: float64 volumes with NaN and ±inf, the split
reduction (S > 1 partials folded by k_keepx_finish) for uint8 and int16, the scalar int16 paths, and
MeanIP on either side of the int32-accumulator guard."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KINDS = ("max", "min", "mean")


@pytest.fixture(scope="module")
def dev():
    from invesalius3_b200 import device
    device.require_cuda()
    return device


def numpy_mip(img, axis, kind):
    return {"max": img.max, "min": img.min, "mean": img.mean}[kind](axis)


def device_mip(dev, img, axis, kind):
    import torch
    return dev.mip(torch.from_numpy(np.ascontiguousarray(img)).cuda(), axis, kind).cpu().numpy()


def splits(shape, dt, axis, kind):
    """S of the keep-x reduction, from the workspace the C ABI asks for (S · plane · element size)."""
    from invesalius3_b200 import _lib
    dz, dy, dx = shape
    itemsize = np.dtype(dt).itemsize
    code = {np.dtype(np.int16): _lib.I16, np.dtype(np.uint8): _lib.U8}[np.dtype(dt)]
    ws = _lib.load().b2v_mip_workspace_bytes(code, dz, dy, dx, axis, {"max": 0, "min": 1, "mean": 2}[kind])
    plane = dy * dx if axis == 0 else dz * dx
    elem = 8 if kind == "mean" else itemsize
    return max(1, ws // (plane * elem))


def _rays(a, axis):
    """View of `a` as rays along `axis`: rays[i, j, t] is sample t of ray (i, j)."""
    return np.moveaxis(a, axis, -1)


@pytest.mark.parametrize("nx", [1, 5, 31, 33])
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_float64_nan_and_inf(dev, nx, axis):
    """NaN first, last and in the middle of a ray propagate as in NumPy; ±inf win their ray."""
    rng = np.random.default_rng(nx * 3 + axis)
    img = rng.normal(0.0, 500.0, (7, 6, nx))
    r = _rays(img, axis)
    n = r.shape[-1]
    rays = [(i, j) for i in range(r.shape[0]) for j in range(r.shape[1])]
    rng.shuffle(rays)
    plant = [(0, np.nan), (n - 1, np.nan), (n // 2, np.nan), (n - 1, np.inf), (0, -np.inf), (n // 2, np.inf),
             (n - 1, -np.inf)]
    for (i, j), (t, v) in zip(rays, plant):
        r[i, j, t] = v
    if len(rays) > len(plant) and n > 1:                      # +inf and -inf on one ray, NaN after an inf
        i, j = rays[len(plant)]
        r[i, j, 0], r[i, j, -1] = np.inf, -np.inf
    if len(rays) > len(plant) + 1 and n > 1:
        i, j = rays[len(plant) + 1]
        r[i, j, 0], r[i, j, -1] = np.inf, np.nan
    for kind in ("max", "min"):
        got = device_mip(dev, img, axis, kind)
        want = numpy_mip(img, axis, kind)
        assert got.dtype == want.dtype and got.shape == want.shape
        assert np.array_equal(got, want, equal_nan=True), (nx, axis, kind)
    assert np.isnan(want).any() and np.isinf(want).any()


def test_float64_mean_raises(dev):
    img = np.random.default_rng(0).normal(size=(4, 5, 6))
    for axis in (0, 1, 2):
        with pytest.raises(ValueError, match="MeanIP of a float64"):
            device_mip(dev, img, axis, "mean")


# shapes whose reduced axis forces S = 2, 4, 8, 16 (every output row fits in one block of x-vectors,
# so S doubles while the reduced axis keeps >= 32 rows per split: 64 / 128 / 256 / 512 rows)
SPLIT_SHAPES = [((100, 5, 7), 0, 2), ((200, 9, 13), 0, 4), ((300, 4, 16), 0, 8), ((600, 11, 17), 0, 16),
                ((2, 100, 40), 1, 2), ((3, 130, 24), 1, 4), ((2, 300, 13), 1, 8), ((1, 530, 64), 1, 16)]


def _planted(rng, shape, axis, dt):
    """Random values inside the type's range with the extremes planted on the first, a middle and
    the last row of the reduced axis, so that dropping any split changes the answer."""
    info = np.iinfo(dt)
    lo, hi = (20, 236) if dt == np.uint8 else (-20000, 20000)
    img = rng.integers(lo, hi, shape).astype(dt)
    r = _rays(img, axis)
    n = r.shape[-1]
    ii, jj = np.indices(r.shape[:2])
    group = (ii + jj) % 3
    for t, a in zip((0, n // 2, n - 1), (0, 1, 2)):
        r[group == a, t] = info.max
        r[group == (a + 1) % 3, t] = info.min
    return img


@pytest.mark.parametrize("shape, axis, S", SPLIT_SHAPES)
@pytest.mark.parametrize("dt", [np.uint8, np.int16])
def test_split_reduction(dev, shape, axis, S, dt):
    rng = np.random.default_rng(sum(shape) + S)
    img = _planted(rng, shape, axis, dt)
    for kind in KINDS:
        assert splits(shape, dt, axis, kind) == S, (shape, axis, kind)
        got = device_mip(dev, img, axis, kind)
        want = numpy_mip(img, axis, kind)
        assert got.dtype == want.dtype and np.array_equal(got, want), (shape, axis, kind, dt)
    # the last split alone decides some outputs: the last row's value is the unique extreme there
    last = np.zeros(shape, dt) + (np.iinfo(dt).max // 2)
    _rays(last, axis)[..., -1] = np.iinfo(dt).max
    assert np.array_equal(device_mip(dev, last, axis, "max"), numpy_mip(last, axis, "max"))


@pytest.mark.parametrize("shape", [(9, 10, 13), (70, 6, 13), (3, 150, 21), (5, 7, 8)])
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_int16_scalar_paths(dev, shape, axis):
    """int16 on a view one element past an aligned start, and on rows with nx % 8 != 0."""
    import torch
    rng = np.random.default_rng(shape[0] + axis)
    img = _planted(rng, shape, axis, np.int16)
    base = torch.zeros(img.size + 1, dtype=torch.int16, device="cuda")
    base[1:] = torch.from_numpy(img.ravel()).cuda()
    view = base[1:].view(shape)
    assert view.data_ptr() % 16 != 0 and view.is_contiguous()
    for kind in KINDS:
        want = numpy_mip(img, axis, kind)
        assert np.array_equal(dev.mip(view, axis, kind).cpu().numpy(), want), (shape, axis, kind)
        assert np.array_equal(device_mip(dev, img, axis, kind), want), (shape, axis, kind)


@pytest.mark.parametrize("dz", [262144, 262145])
@pytest.mark.parametrize("value", [-32768, 32767])
def test_mean_around_the_int32_guard(dev, dz, value):
    """nr <= 8 · 32768 rows take the packed int32 lane sums, one more row the int64 scalar path: the
    dispatch on either side of the guard, with every value at an end of the int16 range. With a
    single kept column block this shape splits the rows 16 ways (2048 rows per lane), so the lanes
    stay far from overflow here; test_mean_guard_without_splits checks the bound itself."""
    img = np.full((dz, 1, 8), value, np.int16)
    for axis in (0, 2):                     # axis 1 keeps dz > 65535 slices: refused by the kernel's grid
        got = device_mip(dev, img, axis, "mean")
        want = numpy_mip(img, axis, "mean")
        assert got.dtype == np.float64 and np.array_equal(got, want), (dz, value, axis)
    assert (device_mip(dev, img, 0, "mean") == value).all()


@pytest.mark.parametrize("nr", [262144, 262145, 3 * 262144])
@pytest.mark.parametrize("value", [-32768, 32767])
def test_mean_guard_without_splits(dev, nr, value):
    """Enough kept columns (4 · SMs rows of 8) that the reduction is not split (S = 1), so each int32
    lane sums nr / 8 values. At the guard, 32768 · 32768 = 2^30 still fits; at three times it an
    int32 lane would pass ±2^31, so the right mean there shows the guard sends it to the int64 path.
    The volume is made on the device (up to 6.6 GB) and released afterwards."""
    import torch
    dz = 4 * torch.cuda.get_device_properties(0).multi_processor_count
    shape = (dz, nr, 8)
    assert splits(shape, np.int16, 1, "mean") == 1
    t = torch.full(shape, value, dtype=torch.int16, device="cuda")
    try:
        got = dev.mip(t, 1, "mean").cpu().numpy()
    finally:
        del t
        torch.cuda.empty_cache()
    assert got.shape == (dz, 8) and (got == float(value)).all(), (nr, value, np.unique(got)[:4])
