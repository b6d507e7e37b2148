"""apply_view_matrix_transform on the device against the C checker (oracle/transforms.c) at its edges:
the random sweep and the closed-form cases of test_oracle_view_transform_model.py, quaternion
rotations composed like the viewer's, full-size slabs and the "Apply reorientation" action, a
misaligned input, and the Lanczos-4 rule on 2-voxel axes. Modes 0-2 bit for bit; Lanczos (its
kernel goes through sin, where libm and the device may differ in the last bit) within one unit on
fewer than 0.1 % of the voxels."""
import math
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import view_transform_model as vtm

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rs():
    from invesalius3_b200 import device, invesalius_rs
    device.require_cuda()
    return invesalius_rs


@pytest.fixture(scope="module")
def pool():
    # the checker is a ctypes call (the GIL is released): independent cases run side by side
    with ThreadPoolExecutor(max_workers=max(1, min(8, os.cpu_count() or 1))) as ex:
        yield ex


@pytest.fixture(scope="module")
def ct512():
    from invesalius3_b200 import phantom
    return phantom.ct((512, 512, 512))


class Tally:
    """Lanczos differences (in units) summed over many calls, judged once at the end."""

    def __init__(self):
        self.n = self.diff = 0
        self.max = 0.0

    def add(self, got, want):
        if got.dtype == np.float64:
            assert np.allclose(got, want, rtol=1e-12, atol=1e-9)
            return
        d = np.abs(got.astype(np.int64) - want.astype(np.int64))
        self.n += d.size
        self.diff += int((d != 0).sum())
        self.max = max(self.max, float(d.max()) if d.size else 0.0)

    def check(self):
        assert self.max <= 1 and self.diff < 1e-3 * max(self.n, 1), (self.max, self.diff, self.n)


def lanczos(minterpol):
    return minterpol not in (0, 1, 2)


def run_device(rs, vol, spacing, m, n, orient, minterpol, cval, oshape):
    got = np.zeros(oshape, vol.dtype)
    rs.apply_view_matrix_transform(vol, spacing, m, n, orient, minterpol, cval, got)
    return got


def compare(rs, orc, case, tally, want=None, rc=None):
    """Device against the checker on one case; a checker panic must be a ValueError on the device."""
    vol, spacing, m, n, orient, minterpol, cval, oshape = case
    if want is None:
        want = np.zeros(oshape, vol.dtype)
        rc = orc.apply_view_matrix_transform_rc(vol, spacing, m, n, orient, minterpol, cval, want)
    if rc:
        match = "index out of bounds" if rc == vtm.INDEX else "not representable"
        with pytest.raises(ValueError, match=match):
            run_device(rs, *case)
        return rc
    got = run_device(rs, *case)
    if lanczos(minterpol):
        tally.add(got, want)
    else:
        assert got.tobytes() == want.tobytes(), (vol.shape, vol.dtype, orient, n, minterpol, oshape)
    return rc


def compare_all(rs, orc, pool, cases):
    def chk(case):
        vol, spacing, m, n, orient, minterpol, cval, oshape = case
        want = np.zeros(oshape, vol.dtype)
        return want, orc.apply_view_matrix_transform_rc(vol, spacing, m, n, orient, minterpol, cval, want)
    tally = Tally()
    codes = [compare(rs, orc, case, tally, *res) for case, res in zip(cases, pool.map(chk, cases))]
    tally.check()
    return codes


def test_random_sweep(rs, orc, pool):
    """The CPU model test's sweep: every axis length in {1, 2, 3, 4, 5, 17}, int16 / uint8 /
    float64, four orientations, n at 0 / middle / last / past the end, minterpol -1, 0, 1, 2, 3, 7."""
    cases = [c for s in range(4) for c in vtm.random_cases(100 + s, 150)]
    codes = compare_all(rs, orc, pool, cases)
    assert set(codes) == {vtm.OK, vtm.CAST, vtm.INDEX}


def _closed_form_cases():
    cases = []
    rng = np.random.default_rng(3)
    for dt in (np.int16, np.uint8, np.float64):
        info = np.iinfo(dt) if dt != np.float64 else None
        vol = (rng.integers(-3000, 3000, (5, 6, 7)) * 0.25 if dt == np.float64
               else rng.integers(max(info.min, -3000), min(info.max, 3000), (5, 6, 7)).astype(dt))
        for perm, flips in (((0, 1, 2), (True, False, True)), ((2, 1, 0), (False, False, False)),
                            ((1, 2, 0), (False, True, False)), ((2, 0, 1), (True, True, True))):
            m = vtm.permutation_flip_matrix(vol.shape, vtm.EXACT_SPACING, perm, flips)
            oshape = tuple(vol.shape[k] for k in perm)
            for minterpol in (0, 1, 2, 3):
                cases.append((vol, vtm.EXACT_SPACING, m, 0, "VOLUME", minterpol, vol.min(), oshape))
                if perm[0] == 0:
                    cases.append((vol, vtm.EXACT_SPACING, m, 2, "AXIAL", minterpol, vol.min(), (2,) + oshape[1:]))
        w2 = np.eye(4); w2[3, 3] = 2.0
        w0 = np.eye(4); w0[3, 3] = 0.0
        for minterpol in (0, 1, 2, 3):
            cases.append((vol, vtm.EXACT_SPACING, w2, 0, "VOLUME", minterpol, vol.min(), (9, 11, 13)))
            cases.append((vol, vtm.EXACT_SPACING, w0, 1, "AXIAL", minterpol, vol.min(), (2, 6, 7)))
            for axis in range(3):
                d = vol.shape[axis]
                for t in (float(d - 1), math.nextafter(d - 1.0, 0.0), float(d - 2)):
                    m = np.eye(4); m[axis, 3] = t
                    cases.append((vol, (1.0, 1.0, 1.0), m, 0, "VOLUME", minterpol, vol.min(), (2, 2, 2)))
    prof = np.broadcast_to(np.array([1000, -1000, -1000, -1000, -1000], np.int16), (4, 4, 5)).copy()
    half = np.eye(4); half[2, 3] = 0.5
    for cval in (-1200, -1100):
        cases.append((prof, (1.0, 1.0, 1.0), half, 0, "VOLUME", 2, cval, (3, 3, 3)))
    u8 = np.broadcast_to(np.array([0, 255, 255, 255, 255], np.uint8), (4, 4, 5)).copy()
    cases.append((u8, (1.0, 1.0, 1.0), half, 0, "VOLUME", 2, 0, (3, 3, 3)))
    return cases


def test_closed_form_cases(rs, orc, pool):
    """Permutation / flip matrices, w = 2 and w = 0, coordinates on d - 1, just below it and on d - 2,
    the clamped tricubic undershoot and the uint8 overshoot."""
    codes = compare_all(rs, orc, pool, _closed_form_cases())
    assert vtm.CAST in codes and vtm.INDEX not in codes


@pytest.mark.parametrize("angle, axis", [(1e-9, (0.3, -0.5, 0.8)), (math.pi / 2, (0, 0, 1)), (math.pi / 2, (1, 0, 0)),
                                         (math.pi, (0, 1, 0)), (math.pi, (1, 1, 0)), (0.7, "random")])
def test_quaternion_rotations(rs, orc, pool, angle, axis):
    """Rotations composed as the viewer composes them, T1 · Rᵀ · T0 about the centre, on a smooth
    volume, every interpolator and orientation."""
    from scipy import ndimage
    rng = np.random.default_rng(11)
    shape = (21, 34, 29)
    vol = (ndimage.gaussian_filter(rng.normal(size=shape), 1.2) * 6000).astype(np.int16)
    sp = (0.78125, 0.78125, 1.25)
    if axis == "random":
        axis = tuple(rng.normal(size=3))
    m = vtm.view_matrix(shape, sp, vtm.quaternion_about_axis(angle, axis))
    cases = []
    for minterpol in (0, 1, 2, 3):
        for orient, n, oshape in (("AXIAL", 9, (3, 34, 29)), ("CORONAL", 0, (21, 2, 29)), ("SAGITAL", 27, (21, 34, 2)),
                                  ("VOLUME", 0, shape)):
            cases.append((vol, sp, m, n, orient, minterpol, int(vol.min()), oshape))
    assert set(compare_all(rs, orc, pool, cases)) == {vtm.OK}


def test_phantom_slabs_512(rs, orc, pool, ct512):
    """A 4-slice slab per orientation of the 512³ phantom at spacing (0.5, 0.5, 1.0), rotated about a
    random axis, cval = matrix.min(), for all four interpolators."""
    vol = ct512
    sp = (0.5, 0.5, 1.0)
    m = vtm.view_matrix(vol.shape, sp, vtm.quaternion_about_axis(0.35, (0.4, -0.7, 0.6)))
    cval = int(vol.min())
    cases = [(vol, sp, m, n, orient, minterpol, cval, oshape)
             for minterpol in (0, 1, 2, 3)
             for orient, n, oshape in (("AXIAL", 254, (4, 512, 512)), ("CORONAL", 100, (512, 4, 512)),
                                       ("SAGITAL", 400, (512, 512, 4)))]
    assert set(compare_all(rs, orc, pool, cases)) == {vtm.OK}
    got = run_device(rs, *cases[0])
    assert (got != cval).mean() > 0.5


def test_apply_reorientation_full_size(rs, orc, pool, ct512, tmp_path):
    """"Apply reorientation": a whole 256×512×512 int16 volume resampled with tricubic from one memmap
    into another, then an edited mask's padded (dz+1, dy+1, dx+1) uint8 matrix with nearest and cval 0."""
    shape = (256, 512, 512)
    sp = (0.5, 0.5, 1.0)
    src = np.memmap(tmp_path / "mcopy.dat", dtype=np.int16, mode="w+", shape=shape)
    src[:] = ct512[128:384]
    m = vtm.view_matrix(shape, sp, vtm.quaternion_about_axis(0.4, (0.2, 0.9, -0.3)))
    cval = int(src.min())
    mshape = tuple(s + 1 for s in shape)
    mask = np.zeros(mshape, np.uint8)
    mask[1:, 1:, 1:] = np.where(ct512[128:384] > 300, 255, 0)
    mask[1:40, 0, 0] = 1

    def checker(vol, interp, c, osh):
        want = np.zeros(osh, vol.dtype)
        return want, orc.apply_view_matrix_transform_rc(vol, sp, m, 0, "AXIAL", interp, c, want)
    fut_img = pool.submit(checker, src, 2, cval, shape)
    fut_mask = pool.submit(checker, mask, 0, 0, mshape)
    out = np.memmap(tmp_path / "matrix.dat", dtype=np.int16, mode="w+", shape=shape)
    rs.apply_view_matrix_transform(src, sp, m, 0, "AXIAL", 2, cval, out)
    mout = np.memmap(tmp_path / "mask.dat", dtype=np.uint8, mode="w+", shape=mshape)
    rs.apply_view_matrix_transform(mask, sp, m, 0, "AXIAL", 0, 0, mout)
    want, rc = fut_img.result()
    assert rc == 0 and np.array_equal(out, want)
    assert (want != cval).mean() > 0.5
    want, rc = fut_mask.result()
    assert rc == 0 and np.array_equal(mout, want)
    assert (want == 255).sum() > 0.5 * (mask == 255).sum()


@pytest.mark.parametrize("minterpol", [0, 1, 2, 3])
def test_misaligned_input(rs, orc, minterpol):
    """A contiguous device tensor one element past an aligned start, handed to the C ABI: the kernel
    reads it as it is. The same misaligned array on the host goes through invesalius_rs, which copies
    it into a fresh aligned tensor first, so that half is the control case."""
    import ctypes as C
    import torch
    from invesalius3_b200 import _lib, device
    rng = np.random.default_rng(5)
    shape = (9, 14, 11)
    base = np.empty(np.prod(shape) + 1, np.int16)
    vol = base[1:].reshape(shape)
    vol[:] = rng.integers(-1000, 2000, shape)
    assert vol.flags.c_contiguous and vol.ctypes.data % 16 != 0
    sp = (0.9, 1.1, 1.3)
    m = vtm.view_matrix(shape, sp, vtm.quaternion_about_axis(0.5, (1, 2, 3)))
    want = np.zeros((3, 14, 11), np.int16)
    assert orc.apply_view_matrix_transform_rc(vol, sp, m, 4, "AXIAL", minterpol, -1000, want) == 0
    tally = Tally()
    got = run_device(rs, vol, sp, m, 4, "AXIAL", minterpol, -1000, (3, 14, 11))
    tbase = torch.from_numpy(base).cuda()
    tvol = tbase[1:].view(shape)
    assert tvol.data_ptr() % 16 != 0 and tvol.is_contiguous()
    tout = torch.empty((3, 14, 11), dtype=torch.int16, device="cuda")
    ws = device._workspace(256, tvol.device)
    spa = np.ascontiguousarray(sp, np.float64)
    ma = np.ascontiguousarray(m, np.float64)
    _lib.call("b2v_apply_view_matrix_transform", device._p(tvol), _lib.I16, *shape, C.c_void_p(spa.ctypes.data),
              C.c_void_p(ma.ctypes.data), 4, 0, minterpol, -1000.0, device._p(tout), 3, 14, 11, device._p(ws),
              device._stream())
    for g in (got, tout.cpu().numpy()):
        if lanczos(minterpol):
            tally.add(g, want)
        else:
            assert np.array_equal(g, want)
    tally.check()
    assert (want != -1000).mean() > 0.3


@pytest.mark.parametrize("shape, orient, oshape", [((2, 5, 6), "AXIAL", (1, 5, 6)), ((5, 2, 6), "CORONAL", (5, 1, 6)),
                                                   ((5, 6, 2), "SAGITAL", (5, 6, 1)), ((2, 2, 2), "VOLUME", (2, 2, 2))])
@pytest.mark.parametrize("minterpol", [-1, 3, 7])
def test_lanczos_two_voxel_axis(rs, orc, shape, orient, oshape, minterpol):
    """An in-range sample on a 2-voxel axis raises on the device and in the checker (the crate's
    index panics); a slab whose samples all fall outside [0, d - 1) returns cval, as the crate does."""
    vol = np.random.default_rng(2).integers(-900, 900, shape).astype(np.int16)
    for dt, cval in ((np.int16, -5), (np.uint8, 5), (np.float64, -5.5)):
        v = vol.astype(dt) if dt != np.uint8 else (vol % 200).astype(np.uint8)
        with pytest.raises(ValueError, match="index out of bounds"):
            orc.apply_view_matrix_transform(v, (1.0, 1.0, 1.0), np.eye(4), 0, orient, minterpol, cval, np.zeros(oshape, dt))
        with pytest.raises(ValueError, match="index out of bounds"):
            run_device(rs, v, (1.0, 1.0, 1.0), np.eye(4), 0, orient, minterpol, cval, oshape)
        away = np.eye(4)
        away[:3, 3] = 1.0                    # every sample lands on index 1 = d - 1 of the short axis, or beyond
        want = np.zeros(oshape, dt)
        assert orc.apply_view_matrix_transform_rc(v, (1.0, 1.0, 1.0), away, 0, orient, minterpol, cval, want) == 0
        got = run_device(rs, v, (1.0, 1.0, 1.0), away, 0, orient, minterpol, cval, oshape)
        assert (want == np.asarray(cval, dt)).all() and got.tobytes() == want.tobytes()
