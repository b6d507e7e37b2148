"""A vectorised NumPy float64 restatement of invesalius_rs.apply_view_matrix_transform
(transforms_py.rs:12-49 -> transforms.rs:9-55 -> interpolation.rs:6-188), written independently of
the C checker (oracle/transforms.c) so that each can be checked against the other, and the cases
both are run on.

Every float64 step is one IEEE operation in the reference's order (NumPy does not fuse
multiply-adds): the matrix rows as ((m0 c0 + m1 c1) + m2 c2) + m3 c3, then / w / spacing; the
strict bounds test 0 <= f < d - 1; get_value's one-step wrap; the cubic and Lanczos sums in the
crate's loop order; NumCast's range test and truncation. The Lanczos kernel calls math.sin, the
libm sin the checker calls, so even Lanczos results can be compared bit for bit.

`transform` returns (out, code) with the checker's codes: 0, CAST when a cast to the output type
panics in the reference, INDEX when a tap is still outside the volume after the wrap (ndarray's
index panics). A panicking sample is written as 0, as the checker writes it.
"""
from __future__ import annotations

import math

import numpy as np

ORIENT = {"AXIAL": 0, "CORONAL": 1, "SAGITAL": 2}
OK, CAST, INDEX = 0, 3, 4
_CAST_OPEN = {np.dtype(np.int16): (-32769.0, 32768.0), np.dtype(np.uint8): (-1.0, 256.0)}


def sample_coords(spacing, m, n, orientation, oshape):
    """(fz, fy, fx) of every output voxel: the volume index it samples, as float64."""
    sx, sy, sz = (float(v) for v in spacing)
    m = np.asarray(m, np.float64).reshape(4, 4)
    cz, cy, cx = np.indices(oshape, dtype=np.int64)
    o = ORIENT.get(orientation, 3)
    z = cz + n if o == 0 else cz
    y = cy + n if o == 1 else cy
    x = cx + n if o == 2 else cx
    c = (z.astype(np.float64) * sz, y.astype(np.float64) * sy, x.astype(np.float64) * sx, 1.0)
    nc = [((m[k, 0] * c[0] + m[k, 1] * c[1]) + m[k, 2] * c[2]) + m[k, 3] * c[3] for k in range(4)]
    with np.errstate(divide="ignore", invalid="ignore"):
        return (nc[0] / nc[3]) / sz, (nc[1] / nc[3]) / sy, (nc[2] / nc[3]) / sx


class _Gather:
    """get_value on flat arrays of taps: one wrap per axis; taps still outside are recorded."""

    def __init__(self, vol):
        self.v = np.asarray(vol).astype(np.float64)
        self.d = vol.shape
        self.bad = None

    def __call__(self, x, y, z):
        idx = []
        for i, n in zip((z, y, x), self.d):
            i = np.where(i < 0, i + n, np.where(i >= n, i - n, i))
            out = (i < 0) | (i >= n)
            self.bad = out if self.bad is None else self.bad | out
            idx.append(np.clip(i, 0, n - 1))
        return self.v[idx[0], idx[1], idx[2]]


def cubic(p0, p1, p2, p3, x):
    return p1 + 0.5 * x * (p2 - p0 + x * (2.0 * p0 - 5.0 * p1 + 4.0 * p2 - p3 + x * (3.0 * (p1 - p2) + p3 - p0)))


_msin = np.frompyfunc(math.sin, 1, 1)


def lanczos_kernel(x):
    """interpolation.rs:55-64 with a = 4, sin from libm (math.sin)."""
    x = np.asarray(x, np.float64)
    s1 = _msin(math.pi * x).astype(np.float64)
    s2 = _msin(math.pi * (x / 4.0)).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        k = (4.0 * s1 * s2) / (math.pi * math.pi * x * x)
    return np.where(x == 0.0, 1.0, np.where((-4.0 <= x) & (x < 4.0), k, 0.0))


def _interpolate(vol, fz, fy, fx, minterpol):
    """Unclamped float64 result of modes 1, 2 and Lanczos at in-range samples, and the samples
    whose taps leave the volume."""
    get = _Gather(vol)
    fl = [np.floor(f).astype(np.int64) for f in (fx, fy, fz)]
    x0, y0, z0 = fl
    if minterpol == 1:
        xd, yd, zd = fx - x0.astype(np.float64), fy - y0.astype(np.float64), fz - z0.astype(np.float64)
        x1, y1, z1 = x0 + 1, y0 + 1, z0 + 1
        v000, v100, v010, v001 = get(x0, y0, z0), get(x1, y0, z0), get(x0, y1, z0), get(x0, y0, z1)
        v110, v101, v011, v111 = get(x1, y1, z0), get(x1, y0, z1), get(x0, y1, z1), get(x1, y1, z1)
        c00 = v000 * (1.0 - xd) + v100 * xd
        c10 = v010 * (1.0 - xd) + v110 * xd
        c01 = v001 * (1.0 - xd) + v101 * xd
        c11 = v011 * (1.0 - xd) + v111 * xd
        c0 = c00 * (1.0 - yd) + c10 * yd
        c1 = c01 * (1.0 - yd) + c11 * yd
        res = c0 * (1.0 - zd) + c1 * zd
    elif minterpol == 2:
        ty, tz = fy - y0.astype(np.float64), fz - z0.astype(np.float64)
        r = []
        for a in range(4):          # p[a][b][c] = value at (x0 + a - 1, y0 + b - 1, z0 + c - 1)
            arr = [cubic(*[get(x0 + a - 1, y0 + b - 1, z0 + c - 1) for c in range(4)], tz) for b in range(4)]
            r.append(cubic(*arr, ty))
        res = cubic(*r, fx - x0.astype(np.float64))
    else:
        xi, yi, zi = x0 - 3, y0 - 3, z0 - 3
        kx = [lanczos_kernel(fx - (xi + k).astype(np.float64)) for k in range(7)]
        ky = [lanczos_kernel(fy - (yi + k).astype(np.float64)) for k in range(7)]
        kz = [lanczos_kernel(fz - (zi + k).astype(np.float64)) for k in range(7)]
        res = 0.0
        for kk in range(7):
            ly = 0.0
            for jj in range(7):
                lx = 0.0
                for ii in range(7):
                    lx = lx + get(xi + ii, yi + jj, zi + kk) * kx[ii]
                ly = ly + lx * ky[jj]
            res = res + ly * kz[kk]
    bad = get.bad if get.bad is not None else np.zeros(fx.shape, bool)
    return np.where(bad, 0.0, res), bad


def transform(vol, spacing, m, n, orientation, minterpol, cval, oshape):
    """out[oshape] and the checker's code for apply_view_matrix_transform(vol, ...)."""
    vol = np.asarray(vol)
    dt = vol.dtype
    out = np.full(oshape, cval, dt)
    fz, fy, fx = sample_coords(spacing, m, n, orientation, oshape)
    dz, dy, dx = vol.shape
    inside = (fz >= 0.0) & (fz < dz - 1.0) & (fy >= 0.0) & (fy < dy - 1.0) & (fx >= 0.0) & (fx < dx - 1.0)
    fz, fy, fx = fz[inside], fy[inside], fx[inside]
    if minterpol == 0:
        out[inside] = vol[fz.astype(np.int64), fy.astype(np.int64), fx.astype(np.int64)]
        return out, OK
    res, bad = _interpolate(vol, fz, fy, fx, minterpol)
    if dt == np.float64:
        ok = np.ones(res.shape, bool)
        val = res.copy()
    else:
        lo, hi = _CAST_OPEN[dt]
        ok = (res > lo) & (res < hi)
        val = np.trunc(np.where(ok, res, 0.0)).astype(dt)
    if minterpol != 1:
        val = np.where(ok & (val < cval), np.asarray(cval, dt), val)
    val = np.where(bad, np.zeros((), dt), val)
    out[inside] = val
    code = INDEX if bad.any() else (CAST if not ok[~bad].all() else OK)
    return out, code


# ------------------------------------------------------------------------------------- cases
AXES = (1, 2, 3, 4, 5, 17)
DTYPES = (np.int16, np.uint8, np.float64)
ORIENTATIONS = ("AXIAL", "CORONAL", "SAGITAL", "VOLUME")
INTERPS = (-1, 0, 1, 2, 3, 7)


def quaternion_matrix(q):
    """4x4 homogeneous rotation of the quaternion q = (w, x, y, z), normalised first: the rotation
    v -> q v q* written out for a unit quaternion (a non-zero q is required)."""
    w, x, y, z = np.asarray(q, np.float64) / np.linalg.norm(q)
    r = np.eye(4)
    r[:3, :3] = [[1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - w * z), 2.0 * (x * z + w * y)],
                 [2.0 * (x * y + w * z), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - w * x)],
                 [2.0 * (x * z - w * y), 2.0 * (y * z + w * x), 1.0 - 2.0 * (x * x + y * y)]]
    return r


def quaternion_about_axis(angle, axis):
    axis = np.asarray(axis, np.float64)
    axis = axis / np.linalg.norm(axis)
    return np.concatenate([[math.cos(angle / 2.0)], axis * math.sin(angle / 2.0)])


def view_matrix(shape, spacing, q):
    """T1 · Rᵀ · T0 about the volume centre (x, y, z) = shape[::-1] * spacing / 2, in the (z, y, x)
    millimetres of the view matrix: how the viewer composes its rotation (slice_.py:857-859)."""
    cx, cy, cz = (s * d / 2.0 for d, s in zip(shape[::-1], spacing))
    T0 = np.eye(4); T0[:3, 3] = (-cz, -cy, -cx)
    T1 = np.eye(4); T1[:3, 3] = (cz, cy, cx)
    return T1 @ quaternion_matrix(q).T @ T0


def _volume(rng, shape, dt):
    if dt == np.float64:
        return rng.normal(0.0, 300.0, shape)
    if dt == np.uint8:
        lo, hi = (0, 256) if rng.random() < 0.3 else (40, 216)
        return rng.integers(lo, hi, shape).astype(np.uint8)
    lo, hi = (-32768, 32768) if rng.random() < 0.15 else (-1500, 3000)
    return rng.integers(lo, hi, shape).astype(np.int16)


def random_case(rng):
    """(vol, spacing, m, n, orientation, minterpol, cval, oshape) drawn over every axis length in
    AXES, the three dtypes, four orientations, n at 0 / middle / last / past the end, every mode."""
    shape = tuple(int(v) for v in rng.choice(AXES, 3))
    dt = DTYPES[rng.integers(len(DTYPES))]
    orient = ORIENTATIONS[rng.integers(len(ORIENTATIONS))]
    minterpol = int(rng.choice(INTERPS))
    oshape = list(shape)
    ax = ORIENT.get(orient)
    d = shape[ax] if ax is not None else shape[0]
    n = int((0, d // 2, d - 1, d + int(rng.integers(0, 3)))[rng.integers(4)])
    if ax is not None:
        oshape[ax] = int(rng.integers(1, 4))
    spacing = tuple(float(v) for v in (rng.uniform(0.3, 2.0, 3) if rng.random() < 0.7 else rng.choice([0.5, 1.0, 2.0], 3)))
    axis = rng.normal(size=3)
    q = quaternion_about_axis(rng.uniform(-math.pi, math.pi) * (rng.random() < 0.85), axis)
    m = view_matrix(shape, spacing, q)
    m[:3, 3] += rng.normal(0.0, 0.5, 3) * np.array(spacing[::-1])
    if rng.random() < 0.25:             # projective bottom row
        m[3, :3] = rng.normal(0.0, 0.02, 3)
        m[3, 3] = rng.uniform(0.8, 1.25)
    vol = _volume(rng, shape, dt)
    if dt == np.float64:
        cval = float(rng.choice([0.0, vol.min(), -1e3]))
    else:
        info = np.iinfo(dt)
        cval = int(rng.choice([int(vol.min()), int(info.min), int(rng.integers(info.min, info.max + 1))]))
    return vol, spacing, m, n, orient, minterpol, cval, tuple(oshape)


def random_cases(seed, count):
    rng = np.random.default_rng(seed)
    return [random_case(rng) for _ in range(count)]


# ---- closed forms: cases whose answer is known without either restatement ----------------------
EXACT_SPACING = (2.0, 0.5, 1.0)           # (sx, sy, sz), exact in binary


def permutation_flip_matrix(shape, spacing, perm, flips):
    """The view matrix whose output is np.flip(np.transpose(vol, perm), flipped axes): output axis
    j samples volume axis perm[j], mirrored about the centre (d - 1) / 2 where flips[j]."""
    s = np.array(spacing[::-1], np.float64)          # (sz, sy, sx)
    m = np.zeros((4, 4))
    m[3, 3] = 1.0
    for j, k in enumerate(perm):
        sign = -1.0 if flips[j] else 1.0
        m[k, j] = sign * s[k] / s[j]
        if flips[j]:
            m[k, 3] = (shape[k] - 1) * s[k]
    return m


def permutation_flip_expected(vol, perm, flips, cval, n=0, nslices=None):
    """np.transpose / np.flip of the volume, cval where the sampled voxel lies on a last plane
    (outside [0, d - 1)); an AXIAL slab of it from slice n when nslices is given."""
    t = np.transpose(vol, perm)
    inside = np.ones(vol.shape, bool)
    for k in range(3):
        sl = [slice(None)] * 3
        sl[k] = -1
        inside[tuple(sl)] = False
    ti = np.transpose(inside, perm)
    ax = [j for j in range(3) if flips[j]]
    want = np.where(np.flip(ti, ax), np.flip(t, ax), np.asarray(cval, vol.dtype))
    if nslices is not None:
        want = want[n:n + nslices]
    return want
