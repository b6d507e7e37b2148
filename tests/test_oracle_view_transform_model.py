"""The C checker of apply_view_matrix_transform (oracle/transforms.c) against an independent NumPy
restatement of the crate (tests/view_transform_model.py), bit for bit, and both against closed forms
that need neither of them."""
import math

import numpy as np
import pytest

import view_transform_model as vtm


def checker(orc, vol, spacing, m, n, orientation, minterpol, cval, oshape):
    out = np.zeros(oshape, vol.dtype)
    rc = orc.apply_view_matrix_transform_rc(vol, spacing, m, n, orientation, minterpol, cval, out)
    return out, rc


def same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes()


def both(orc, *case):
    """Checker and model on one case; they must agree on every bit and on the code."""
    got, rc = checker(orc, *case)
    want, code = vtm.transform(*case)
    assert rc == code and same_bits(got, want), (case[0].shape, case[0].dtype, case[4], case[3], case[5], rc, code)
    return got, rc


@pytest.mark.parametrize("seed", range(4))
def test_random_cases_checker_equals_model(orc, seed):
    codes = set()
    inside = 0
    for case in vtm.random_cases(100 + seed, 150):
        out, rc = both(orc, *case)
        codes.add(rc)
        inside += int((out != case[6]).sum())
    assert vtm.OK in codes and vtm.INDEX in codes
    assert inside > 500                    # the sweep really samples the volumes


def test_sweep_covers_its_axes():
    """Every axis length, dtype, orientation, n position and mode occurs in the sweep."""
    cases = [c for s in range(4) for c in vtm.random_cases(100 + s, 150)]
    assert {d for c in cases for d in c[0].shape} == set(vtm.AXES)
    assert {c[0].dtype for c in cases} == {np.dtype(t) for t in vtm.DTYPES}
    assert {c[4] for c in cases} == set(vtm.ORIENTATIONS)
    assert {c[5] for c in cases} == set(vtm.INTERPS)
    slab = [(c[3], c[0].shape[vtm.ORIENT[c[4]]]) for c in cases if c[4] in vtm.ORIENT]
    assert any(n == 0 for n, d in slab) and any(0 < n < d - 1 for n, d in slab)
    assert any(n == d - 1 for n, d in slab) and any(n >= d for n, d in slab)


def _perm_vol(dt, shape=(5, 6, 7), seed=3):
    rng = np.random.default_rng(seed)
    if dt == np.float64:
        return rng.integers(-3000, 3000, shape) * 0.25       # exact in binary, no -0.0
    info = np.iinfo(dt)
    return rng.integers(max(info.min, -3000), min(info.max, 3000), shape).astype(dt)


PERMS = [((0, 1, 2), (False, False, False)), ((0, 1, 2), (True, False, True)), ((2, 1, 0), (False, False, False)),
         ((1, 2, 0), (False, True, False)), ((2, 0, 1), (True, True, True)), ((1, 0, 2), (False, False, True))]


@pytest.mark.parametrize("dt", [np.int16, np.uint8, np.float64])
@pytest.mark.parametrize("minterpol", [0, 1, 2, 3])
def test_permutation_and_flip_matrices(orc, dt, minterpol):
    """0/1 permutation and flip matrices with spacings exact in binary: every sample lands on a voxel
    centre, so the output is np.transpose / np.flip of the volume wherever the voxel sampled is in
    range, exactly for modes 0-2 and within one unit for Lanczos (its kernel is only ~1e-16 at the
    non-zero integers)."""
    vol = _perm_vol(dt)
    cval = vol.min()
    for perm, flips in PERMS:
        oshape = tuple(vol.shape[k] for k in perm)
        m = vtm.permutation_flip_matrix(vol.shape, vtm.EXACT_SPACING, perm, flips)
        want = vtm.permutation_flip_expected(vol, perm, flips, cval)
        got, rc = both(orc, vol, vtm.EXACT_SPACING, m, 0, "VOLUME", minterpol, cval, oshape)
        assert rc == 0
        if minterpol < 3:
            assert same_bits(got, want), (perm, flips)
        else:
            assert np.abs(got.astype(np.float64) - want).max() <= 1, (perm, flips)
        if perm[0] == 0:                   # an AXIAL slab: output slice k is volume slice n + k
            n = 2
            got, rc = both(orc, vol, vtm.EXACT_SPACING, m, n, "AXIAL", minterpol, cval, (2,) + oshape[1:])
            want = vtm.permutation_flip_expected(vol, perm, flips, cval, n, 2)
            assert rc == 0 and (same_bits(got, want) if minterpol < 3 else np.abs(got.astype(float) - want).max() <= 1)


@pytest.mark.parametrize("dt", [np.int16, np.uint8, np.float64])
def test_projective_bottom_row(orc, dt):
    """Bottom row (0, 0, 0, 2): every index is halved. Trilinear gives the voxel at even indices and,
    at odd ones, the mean of the 2^k neighbours (k odd indices), truncated for integer types."""
    vol = _perm_vol(dt, (4, 5, 6), 8)
    m = np.eye(4)
    m[3, 3] = 2.0
    oshape = tuple(2 * d - 1 for d in vol.shape)
    got, rc = both(orc, vol, vtm.EXACT_SPACING, m, 0, "VOLUME", 1, 0, oshape)
    assert rc == 0
    want = np.zeros(oshape, np.float64)
    for z, y, x in np.ndindex(*oshape):
        if z >= 2 * vol.shape[0] - 2 or y >= 2 * vol.shape[1] - 2 or x >= 2 * vol.shape[2] - 2:
            continue
        nb = vol[z // 2:(z + 1) // 2 + 1, y // 2:(y + 1) // 2 + 1, x // 2:(x + 1) // 2 + 1].astype(np.float64)
        want[z, y, x] = nb.mean()
    want = want if dt == np.float64 else np.trunc(want).astype(dt)
    assert same_bits(got, want)
    assert same_bits(got[::2, ::2, ::2][:-1, :-1, :-1], vol[:-1, :-1, :-1])


@pytest.mark.parametrize("minterpol", [-1, 0, 1, 2, 3, 7])
def test_zero_w_gives_cval(orc, minterpol):
    """w = 0 divides every coordinate by zero: ±inf or NaN, never in range, cval everywhere."""
    m = np.eye(4)
    m[3, 3] = 0.0
    for dt, cval in ((np.int16, -7), (np.uint8, 9), (np.float64, -0.5)):
        vol = _perm_vol(dt, (4, 5, 6), 1)
        got, rc = both(orc, vol, (0.7, 1.1, 1.3), m, 1, "AXIAL", minterpol, cval, (2, 5, 6))
        assert rc == 0 and (got == np.asarray(cval, dt)).all()


@pytest.mark.parametrize("minterpol", [0, 1, 2, 3])
def test_bound_is_strict_at_d_minus_one(orc, minterpol):
    """A coordinate exactly on d - 1 is outside [0, d - 1) and gives cval; nextafter(d - 1, 0) is
    inside and interpolates (nearest: the voxel d - 2, the others: within one unit of d - 1)."""
    vol = _perm_vol(np.int16, (6, 7, 8), 5)
    cval = -32768
    for axis in range(3):
        d = vol.shape[axis]
        for t, inside in ((float(d - 1), False), (math.nextafter(d - 1.0, 0.0), True)):
            m = np.eye(4)
            m[axis, 3] = t                  # spacing 1: output index 0 samples t along `axis`
            got, rc = both(orc, vol, (1.0, 1.0, 1.0), m, 0, "VOLUME", minterpol, cval, (1, 1, 1))
            assert rc == 0
            v = int(got[0, 0, 0])
            if not inside:
                assert v == cval
                continue
            idx = [0, 0, 0]
            idx[axis] = d - 2 if minterpol == 0 else d - 1
            assert v != cval and abs(v - int(vol[tuple(idx)])) <= (0 if minterpol == 0 else 1)


def test_tricubic_undershoot_clamps_and_uint8_overshoot_raises(orc):
    """Along x the profile [1000, -1000, -1000, -1000] is constant in y and z, so the tricubic is the
    1-D cubic: -1125 at x = 1.5, clamped up to cval when cval is higher. [0, 255, 255, 255] gives
    270.9375 there, which uint8 cannot hold: the reference panics."""
    prof = np.array([1000, -1000, -1000, -1000, -1000], np.int16)
    vol = np.broadcast_to(prof, (4, 4, 5)).copy()
    m = np.eye(4)
    m[2, 3] = 0.5                           # x + 0.5
    for cval, want in ((-1200, -1125), (-1125, -1125), (-1100, -1100)):
        got, rc = both(orc, vol, (1.0, 1.0, 1.0), m, 0, "VOLUME", 2, cval, (3, 3, 3))
        assert rc == 0 and (got[:, :, 1] == want).all()
    u8 = np.broadcast_to(np.array([0, 255, 255, 255, 255], np.uint8), (4, 4, 5)).copy()
    got, rc = both(orc, u8, (1.0, 1.0, 1.0), m, 0, "VOLUME", 2, 0, (3, 3, 3))
    assert rc == vtm.CAST and got[0, 0, 1] == 0
    with pytest.raises(ValueError, match="not representable"):
        orc.apply_view_matrix_transform(u8, (1.0, 1.0, 1.0), m, 0, "VOLUME", 2, 0, np.zeros((3, 3, 3), np.uint8))
    assert vtm.cubic(0.0, 255.0, 255.0, 255.0, 0.5) == 270.9375


LANCZOS_2 = [((2, 5, 6), "AXIAL", 0, (1, 5, 6)), ((5, 2, 6), "CORONAL", 0, (5, 1, 6)), ((5, 6, 2), "SAGITAL", 0, (5, 6, 1))]


@pytest.mark.parametrize("shape, orient, n, oshape", LANCZOS_2)
@pytest.mark.parametrize("minterpol", [-1, 3, 7])
def test_lanczos_on_a_two_voxel_axis(orc, shape, orient, n, oshape, minterpol):
    """Lanczos-4 on an axis of 2 voxels: the tap floor(f) - 3 = -3 is -1 after the wrap. The crate's
    index panics as soon as one sample is in range; when none is, every output is cval."""
    vol = _perm_vol(np.int16, shape, 2)
    got, rc = both(orc, vol, (1.0, 1.0, 1.0), np.eye(4), n, orient, minterpol, -5, oshape)
    assert rc == vtm.INDEX
    with pytest.raises(ValueError, match="index out of bounds"):
        orc.apply_view_matrix_transform(vol, (1.0, 1.0, 1.0), np.eye(4), n, orient, minterpol, -5, np.zeros(oshape, np.int16))
    # the slab's only slice is the volume's last (index 1 along the 2-voxel axis): out of range
    got, rc = both(orc, vol, (1.0, 1.0, 1.0), np.eye(4), 1, orient, minterpol, -5, oshape)
    assert rc == 0 and (got == -5).all()
    # tricubic's taps stay inside on the same axis
    got, rc = both(orc, vol, (1.0, 1.0, 1.0), np.eye(4), n, orient, 2, -32768, oshape)
    assert rc == 0


def test_quaternion_matrix_closed_forms():
    """The formula the tests compose rotations with: 90° about z maps x to y, 180° about x negates y
    and z, a tiny angle is the identity to within the angle; any rotation is orthonormal with
    determinant 1 and keeps its axis, and a quaternion's scale does not matter."""
    r = vtm.quaternion_matrix(vtm.quaternion_about_axis(math.pi / 2, (0, 0, 1)))
    assert np.allclose(r @ [1, 0, 0, 1], [0, 1, 0, 1], atol=1e-15)
    r = vtm.quaternion_matrix(vtm.quaternion_about_axis(math.pi, (1, 0, 0)))
    assert np.allclose(r, np.diag([1.0, -1.0, -1.0, 1.0]), atol=1e-15)
    r = vtm.quaternion_matrix(vtm.quaternion_about_axis(1e-9, (1, 2, 3)))
    assert np.abs(r - np.eye(4)).max() < 2e-9
    axis = np.array([0.3, -1.2, 0.7])
    q = vtm.quaternion_about_axis(2.1, axis)
    r = vtm.quaternion_matrix(q)
    assert np.allclose(r[:3, :3] @ r[:3, :3].T, np.eye(3), atol=1e-15) and np.isclose(np.linalg.det(r[:3, :3]), 1.0)
    assert np.allclose(r[:3, :3] @ axis, axis, atol=1e-15)
    assert np.allclose(vtm.quaternion_matrix(3.5 * q), r, atol=1e-15)
