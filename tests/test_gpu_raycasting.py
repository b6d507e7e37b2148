"""The volume rendering's data preparation on the device (invesalius3_b200.raycasting) against the C checker
(oracle/raycasting.c), bit for bit: the flip and shift, the preset convolutions, chains of them and the histogram,
on the checker tests' shapes, values and kernels, the Cranium crop, a 256x512x512 phantom, memmap and strided
inputs, RaycastingVolume across preset switches, and a volume of more than 2^31 voxels."""
import numpy as np
import pytest

from oracle import raycasting as orc
from test_oracle_raycasting import BAD_KERNELS, IDENTITY, KERNELS, SMOOTH, cases, image, random_kernel

pytestmark = pytest.mark.gpu


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _check(m, kernels=tuple(KERNELS.values()), chains=()):
    """Device against checker for one int16 volume: flip + shift, every kernel, the chains and the histogram."""
    import torch
    from invesalius3_b200 import raycasting as rc
    t = _t(m)
    u, rng = rc.flip_shift_device(t)
    want_u, want_rng = orc.flip_shift(m)
    assert rng == want_rng
    assert np.array_equal(u.cpu().numpy(), want_u)
    for w in kernels:
        assert np.array_equal(rc.convolve5x5_device(u, w).cpu().numpy(), orc.convolve(want_u, w))
    for chain in chains:
        got = u
        for w in chain:
            got = rc.convolve5x5_device(got, w)
        assert np.array_equal(got.cpu().numpy(), orc.convolve_chain(want_u, chain))
    counts, lo, hi = rc.accumulate_histogram_device(t)
    want, wlo, whi = orc.histogram(m)
    assert (lo, hi) == (wlo, whi) and counts.dtype == torch.int64
    assert np.array_equal(counts.cpu().numpy(), want)
    assert np.array_equal(t.cpu().numpy(), m)          # the input is not modified


@pytest.mark.parametrize("name,shape,kind", cases())
def test_small_volumes(name, shape, kind):
    _check(image(shape, kind))


@pytest.mark.parametrize("shape", [(1, 6, 40), (2, 4, 7), (3, 70, 37), (2, 131, 67), (1, 5, 300)])
def test_border_rule_and_tile_edges(shape):
    """Shapes around the device's 64 x 32 tiles and slices thinner than the kernel."""
    _check(image(shape, "full", seed=3), kernels=(IDENTITY, SMOOTH, random_kernel(9)))


@pytest.mark.parametrize("passes", [0, 1, 2, 3])
def test_chains(passes):
    chain = [SMOOTH, random_kernel(5), KERNELS["near_limit"]][:passes]
    _check(image((3, 33, 47), "full", seed=4), kernels=(), chains=(chain,))


def test_cranium(cranium):
    _check(cranium["matrix_crop"], chains=([SMOOTH, SMOOTH],))


def test_phantom_256x512x512():
    from invesalius3_b200 import phantom
    _check(phantom.ct((256, 512, 512), seed=1), kernels=(SMOOTH,), chains=([SMOOTH, SMOOTH],))


def _volume_against_checker(rv, m, spacing):
    u, rng = orc.flip_shift(m)
    dz, dy, dx = m.shape
    assert rv.scale == rng
    assert rv.extent == (0, dx - 1, 0, dy - 1, 0, dz - 1)
    assert rv.spacing == tuple(float(s) for s in spacing)
    assert rv.origin == (0.0, -(dy - 1) * spacing[1], 0.0)
    assert np.array_equal(rv.imagedata(), u)
    counts, init, end = rv.histogram()
    want, wlo, whi = orc.histogram(m)
    assert (init, end) == (wlo, whi) and np.array_equal(counts, want)
    return u


def test_raycasting_volume_preset_switches():
    from invesalius3_b200 import phantom, raycasting as rc
    m = phantom.ct((40, 150, 170), seed=3)
    spacing = (0.45, 0.5, 1.25)
    rv = rc.RaycastingVolume(m, spacing)
    u = _volume_against_checker(rv, m, spacing)
    for chain in ([SMOOTH], [], [SMOOTH, SMOOTH], [SMOOTH], [SMOOTH, random_kernel(1), SMOOTH]):
        got = rv.convolved(chain)
        assert np.array_equal(got, orc.convolve_chain(u, chain))
        assert np.array_equal(got, rc.RaycastingVolume(m, spacing).convolved(chain))
    assert np.array_equal(rv.imagedata(), u)                 # the chains leave the resident volume alone


def test_raycasting_volume_memmap_and_views(tmp_path):
    from invesalius3_b200 import phantom, raycasting as rc
    base = phantom.ct((20, 70, 90), seed=4)
    mm = np.memmap(tmp_path / "matrix.dat", dtype=np.int16, mode="w+", shape=base.shape)
    mm[:] = base
    mm.flush()
    ro = np.memmap(tmp_path / "matrix.dat", dtype=np.int16, mode="r", shape=base.shape)
    for m in (ro, ro[1:, 2:, 3:], base[:, ::2, :], base[::-1]):
        rv = rc.RaycastingVolume(m, (1.0, 0.8, 2.0))
        dense = np.ascontiguousarray(m)
        u = _volume_against_checker(rv, dense, (1.0, 0.8, 2.0))
        assert np.array_equal(rv.convolved([SMOOTH]), orc.convolve(u, SMOOTH))


@pytest.mark.parametrize("bad", sorted(BAD_KERNELS))
def test_rejected_kernels(bad):
    from invesalius3_b200 import raycasting as rc
    rv = rc.RaycastingVolume(image((2, 6, 7), "ct"), (1.0, 1.0, 1.0))
    with pytest.raises(ValueError):
        rv.convolved([BAD_KERNELS[bad]])
    with pytest.raises(ValueError):
        rv.convolved([SMOOTH, BAD_KERNELS[bad]])


def test_rejected_float32_image():
    from invesalius3_b200 import raycasting as rc
    m = image((2, 6, 7), "ct").astype(np.float32)
    with pytest.raises(NotImplementedError):
        rc.RaycastingVolume(m, (1.0, 1.0, 1.0))
    with pytest.raises(NotImplementedError):
        rc.flip_shift_device(_t(m))
    with pytest.raises(NotImplementedError):
        rc.accumulate_histogram_device(_t(m))


def test_past_2_31_voxels():
    """(1025, 1024, 2048): element 2^31 starts slice 1024. Slices are independent, so the slices around it are
    checked against the checker; the volume is generated on the device and freed before the test returns."""
    import torch
    from invesalius3_b200 import raycasting as rc
    shape = (1025, 1024, 2048)
    assert shape[0] * shape[1] * shape[2] > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(11)
    t = torch.randint(-1024, 3072, shape, dtype=torch.int16, device="cuda", generator=g)
    t[:, 0, 0] = -1024            # every slice holds the volume's min and max, so the checker's range on a
    t[:, 0, 1] = 3071             # few slices is the volume's range
    try:
        zs = slice(1021, 1025)
        m = t[zs].cpu().numpy()
        u, rng = rc.flip_shift_device(t)
        counts, lo, hi = rc.accumulate_histogram_device(t)
        n_max = int((t == 3071).sum())
        del t
        want_u, want_rng = orc.flip_shift(m)
        assert rng == want_rng == (-1024.0, 3071.0)
        got_u = u[zs].cpu().numpy()
        assert np.array_equal(got_u, want_u)
        out = rc.convolve5x5_device(u, SMOOTH)
        assert np.array_equal(out[zs].cpu().numpy(), orc.convolve(want_u, SMOOTH))
        assert (lo, hi) == (-1024.0, 3071.0)
        assert int(counts.sum()) == shape[0] * shape[1] * shape[2] - n_max
    finally:
        t = u = out = counts = None
        torch.cuda.empty_cache()
