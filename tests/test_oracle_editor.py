"""The 3-D mask editor's C restatement (oracle/editor.c) against an independent vectorised NumPy
float64 restatement of polygon_mask.rs, mask_cut.rs and brush_mask.rs, closed-form cases, and the
argument checks of invesalius3_b200.mask_editor (all raised before any device work)."""
import math

import numpy as np
import pytest


@pytest.fixture(scope="session")
def ed():
    """The editor's C checker (oracle/editor.py over oracle/editor.c)."""
    from oracle import editor
    editor.lib()
    return editor


# ----------------------------------------------------------------------------- NumPy restatement
def np_polygon2mask(shape, pts):
    w, h = shape
    out = np.zeros((w, h), bool)
    n = len(pts)
    if n == 0 or w == 0 or h == 0:
        return out
    xs, ys = pts[:, 0], pts[:, 1]
    x0 = min(max(math.floor(xs.min()) - 1, 0), w); x1 = min(max(math.ceil(xs.max()) + 1, 0), w)
    y0 = min(max(math.floor(ys.min()) - 1, 0), h); y1 = min(max(math.ceil(ys.max()) + 1, 0), h)
    px = np.arange(x0, min(x1, w - 1) + 1, dtype=np.float64)[:, None]
    py = np.arange(y0, min(y1, h - 1) + 1, dtype=np.float64)[None, :]
    inside = np.zeros((px.shape[0], py.shape[1]), bool)
    j = n - 1
    with np.errstate(all="ignore"):
        for i in range(n):
            xi, yi, xj, yj = xs[i], ys[i], xs[j], ys[j]
            cross = (yi > py) != (yj > py)
            inside ^= cross & (px < (xj - xi) * (py - yi) / (yj - yi) + xi)
            j = i
    out[x0:x0 + inside.shape[0], y0:y0 + inside.shape[1]] = inside
    return out


def np_mask_cut(sx, sy, sz, max_depth, mask, M, MV, out, edit_mode):
    h, w = mask.shape
    zz, yy, xx = np.nonzero(out > 127)
    p = (xx * sx, yy * sy, zz * sz)

    def row(m, i):
        return ((m[i, 0] * p[0] + m[i, 1] * p[1]) + m[i, 2] * p[2]) + m[i, 3] * 1.0

    with np.errstate(all="ignore"):
        q3 = row(M, 3)
        front = q3 > 0
        q0, q1 = row(M, 0) / q3, row(M, 1) / q3
        c3 = row(MV, 3)
        c0, c1, c2 = row(MV, 0) / c3, row(MV, 1) / c3, row(MV, 2) / c3
        dist = np.sqrt((c0 * c0 + c1 * c1) + c2 * c2)
        px = (q0 / 2.0 + 0.5) * float((w - 1) % 2 ** 64)    # `(w - 1) as f64` on a usize
        py = (q1 / 2.0 + 0.5) * float((h - 1) % 2 ** 64)
        on = (px >= 0.0) & (px < w) & (py >= 0.0) & (py < h)
        hit = np.zeros(len(zz), bool)
        hit[on] = mask[py[on].astype(np.int64), px[on].astype(np.int64)]
    zero = front & (dist <= max_depth) & (hit | (~on & (edit_mode == 0)))
    out[zz[zero], yy[zero], xx[zero]] = 0


def np_brush_box(shape, spacing, center, radius):
    box = []
    for n, s, c in zip(shape[::-1], spacing, center):                # x, y, z
        lo = np.fmax(np.floor((c - radius) / s), 0.0)
        hi = np.fmin(np.fmax(np.ceil((c + radius) / s), 0.0), float((n - 1) % 2 ** 64))
        box.append((lo, hi))
    return box[::-1]                                                 # z, y, x


def np_brush(out, orig, spacing, center, radius, edit_mode):
    d, h, w = out.shape
    (z0, z1), (y0, y1), (x0, x1) = np_brush_box(out.shape, spacing, center, radius)
    z, y, x = np.meshgrid(np.arange(d), np.arange(h), np.arange(w), indexing="ij")
    inbox = (z >= z0) & (z <= z1) & (y >= y0) & (y <= y1) & (x >= x0) & (x <= x1)
    ddx, ddy, ddz = x * spacing[0] - center[0], y * spacing[1] - center[1], z * spacing[2] - center[2]
    inside = inbox & (((ddx * ddx + ddy * ddy) + ddz * ddz) <= radius * radius)
    if edit_mode == 1:
        out[inside & (out > 0)] = 0
    elif edit_mode == 0:
        if orig is None:
            out[inside] = 255
        else:
            sel = inside & (orig > 0)
            out[sel] = orig[sel]


# ----------------------------------------------------------------------------- cameras and polygons
def look_at(eye, target, up):
    f = target - eye; f = f / np.linalg.norm(f)
    s = np.cross(f, up); s = s / np.linalg.norm(s)
    u = np.cross(s, f)
    V = np.eye(4)
    V[0, :3], V[1, :3], V[2, :3] = s, u, -f
    V[:3, 3] = -V[:3, :3] @ eye
    return V


def perspective(fovy_deg, aspect, near, far):
    f = 1.0 / np.tan(np.radians(fovy_deg) / 2)
    P = np.zeros((4, 4))
    P[0, 0], P[1, 1] = f / aspect, f
    P[2, 2], P[2, 3] = (far + near) / (near - far), 2 * far * near / (near - far)
    P[3, 2] = -1.0
    return P


def random_camera(rng, shape, spacing, w, h):
    """World -> screen and world -> camera matrices as the editor builds them
    (mask3d_editor_state.py:135-148): VTK-style projection times look-at, then the inv_Y flip.
    Returns (M, MV, near, far)."""
    dz, dy, dx = shape
    centre = np.array([dx * spacing[0], -dy * spacing[1], dz * spacing[2]]) / 2   # y flipped by inv_Y
    radius = np.linalg.norm(centre)
    d = rng.normal(size=3); d /= np.linalg.norm(d)
    eye = centre + d * radius * rng.uniform(1.8, 3.0)
    up = rng.normal(size=3)
    V = look_at(eye, centre, up)
    dist = np.linalg.norm(eye - centre)
    near, far = dist - radius, dist + radius
    P = perspective(rng.uniform(25, 50), w / float(h), near, far)
    inv_y = np.eye(4); inv_y[1, 1] = -1
    return np.ascontiguousarray(P @ V @ inv_y), np.ascontiguousarray(V @ inv_y), near, far


def star_polygon(rng, w, h, n):
    c = np.array([rng.uniform(0.3, 0.7) * w, rng.uniform(0.3, 0.7) * h])
    ang = np.sort(rng.uniform(0, 2 * np.pi, n))
    r = rng.uniform(0.1, 0.45, n) * min(w, h)
    return np.stack([c[0] + r * np.cos(ang), c[1] + r * np.sin(ang)], axis=1)


def tangled_polygon(rng, w, h, n):
    """Random vertices in random order: self-intersecting, some off-screen."""
    return np.stack([rng.uniform(-0.2, 1.2, n) * w, rng.uniform(-0.2, 1.2, n) * h], axis=1)


def editor_filter(polys, w, h, edit_mode, p2m):
    """get_filters + CutMaskFromPolygons (mask3d_editor_state.py:158-200): OR, transpose, NOT for include."""
    filt = np.logical_or.reduce([p2m((w, h), p) for p in polys]).T
    if edit_mode == 0:
        np.logical_not(filt, out=filt)
    return filt


def random_mask(rng, shape, frac=0.4):
    m = np.where(rng.random(shape) < frac, 255, 0).astype(np.uint8)
    m[rng.random(shape) < 0.05] = 100             # never selected (<= 127)
    return m


# ----------------------------------------------------------------------------- oracle == NumPy
def test_polygon2mask_matches_numpy(ed):
    rng = np.random.default_rng(11)
    for k in range(40):
        w, h = int(rng.integers(1, 90)), int(rng.integers(1, 90))
        n = int(rng.integers(3, 60))
        pts = star_polygon(rng, w, h, n) if k % 2 else tangled_polygon(rng, w, h, n)
        if k % 5 == 0:
            pts = np.round(pts)                    # vertices on cell centres: ties in every comparison
        got = ed.polygon2mask_rs((w, h), pts)
        assert got.dtype == np.bool_ and got.shape == (w, h)
        assert np.array_equal(got, np_polygon2mask((w, h), pts)), k


@pytest.mark.parametrize("edit_mode", [0, 1, 2])
def test_mask_cut_matches_numpy(ed, edit_mode):
    rng = np.random.default_rng(20 + edit_mode)
    cut = 0
    for k in range(6):
        shape = tuple(int(s) for s in rng.integers(5, 28, 3))
        sp = tuple(rng.uniform(0.4, 2.0, 3))
        w, h = int(rng.integers(20, 80)), int(rng.integers(20, 80))
        M, MV, near, far = random_camera(rng, shape, sp, w, h)
        polys = [star_polygon(rng, w, h, 12), tangled_polygon(rng, w, h, 7)][: 1 + k % 2]
        filt = editor_filter(polys, w, h, edit_mode, ed.polygon2mask_rs)
        depth = near + (far - near) * rng.uniform(0.3, 1.0)
        base = random_mask(rng, shape)
        want, got = base.copy(), base.copy()
        np_mask_cut(*sp, depth, filt, M, MV, want, edit_mode)
        ed.mask_cut(base, *sp, depth, filt, M, MV, got, edit_mode)
        assert np.array_equal(got, want), k
        cut += bool((got != base).any() and ((got == base) & (base > 127)).any())
    assert cut >= 4                                # most cameras cut part of the mask and keep part


def test_brushes_match_numpy(ed):
    rng = np.random.default_rng(5)
    for k in range(30):
        shape = tuple(int(s) for s in rng.integers(4, 30, 3))
        sp = tuple(rng.uniform(0.3, 1.7, 3))
        ext = np.array(shape[::-1]) * sp
        centre = tuple(rng.uniform(-0.3, 1.3, 3) * ext)
        radius = float(rng.uniform(0.5, 0.6 * ext.max()))
        mode = k % 3
        base = random_mask(rng, shape)
        orig = random_mask(rng, shape, 0.7) if k % 2 else None
        want, got = base.copy(), base.copy()
        np_brush(want, orig, sp, centre, radius, mode)
        ed.brush_mask_rs(got, orig, sp, centre, radius, mode)
        assert np.array_equal(got, want), k


def test_library_brush_box_matches_numpy():
    """The one place the brush box is computed (b2v_brush_mask_box, host code) against brush_mask.rs."""
    from invesalius3_b200.mask_editor import brush_mask_box
    rng = np.random.default_rng(8)
    for k in range(200):
        shape = tuple(int(s) for s in rng.integers(1, 60, 3))
        sp = tuple(rng.uniform(0.2, 2.0, 3))
        centre = tuple(rng.uniform(-20, 80, 3))
        radius = float(rng.uniform(-5, 40))
        want = np_brush_box(shape, sp, centre, radius)
        got = brush_mask_box(shape, sp, centre, radius)
        if any(lo > hi for lo, hi in want):
            assert got is None, k
        else:
            assert got == tuple((int(lo), int(hi)) for lo, hi in want), k


# ----------------------------------------------------------------------------- closed forms
def _ortho(w, h):
    """px = x + 0.5 and py = y + 0.5 on a (w, h) viewport, unit spacing, camera at the origin."""
    M = np.zeros((4, 4))
    M[0, 0], M[0, 3] = 2.0 / (w - 1), 1.0 / (w - 1) - 1.0
    M[1, 1], M[1, 3] = 2.0 / (h - 1), 1.0 / (h - 1) - 1.0
    M[3, 3] = 1.0
    return M, np.eye(4)


@pytest.mark.parametrize("edit_mode", [0, 1])
def test_orthographic_rectangle_cuts_a_known_box(ed, edit_mode):
    w, h = 13, 11
    shape = (4, 10, 14)                        # x = 13 projects to px = 13.5: off-screen
    M, MV = _ortho(w, h)
    rect = np.array([[2.5, 3.5], [7.5, 3.5], [7.5, 6.5], [2.5, 6.5]])
    filt = editor_filter([rect], w, h, edit_mode, ed.polygon2mask_rs)
    base = random_mask(np.random.default_rng(1), shape, 0.8)
    got = base.copy()
    ed.mask_cut(base, 1.0, 1.0, 1.0, 1e9, filt, M, MV, got, edit_mode)
    in_rect = np.zeros(shape, bool)
    in_rect[:, 4:7, 3:8] = True                # px 3..7, py 4..6
    sel = base > 127
    want = base.copy()
    if edit_mode == 1:
        want[sel & in_rect] = 0
    else:
        want[sel & ~in_rect] = 0
    assert np.array_equal(got, want)
    edge = base[:, :, 13]                      # off-screen: cut in include mode only
    assert np.array_equal(got[:, :, 13], np.where(edge > 127, 0, edge) if edit_mode == 0 else edge)


@pytest.mark.parametrize("radius", [3.0, 2.5, 4.2])
def test_unit_brush_changes_exactly_the_lattice_points(ed, radius):
    shape, c = (12, 13, 14), (5, 6, 7)
    out = np.zeros(shape, np.uint8)
    ed.brush_mask_rs(out, None, (1.0, 1.0, 1.0), c, radius, 0)
    r100 = int(round(radius * 10)) ** 2         # 100 r^2, exactly
    z, y, x = np.meshgrid(*(np.arange(n) for n in shape), indexing="ij")
    d2 = (x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2
    assert np.array_equal(out == 255, 100 * d2 <= r100)
    count = sum(1 for i in range(-5, 6) for j in range(-5, 6) for k in range(-5, 6) if 100 * (i * i + j * j + k * k) <= r100)
    assert int((out == 255).sum()) == count
    ed.brush_mask_rs(out, None, (1.0, 1.0, 1.0), c, radius, 1)
    assert not out.any()


@pytest.mark.parametrize("pts", [np.zeros((0, 2)), np.array([[3.0, 4.0]]), np.array([[1.0, 1.0], [6.0, 5.0]])])
def test_degenerate_polygons_are_empty(ed, pts):
    assert not ed.polygon2mask_rs((9, 8), pts).any()
    assert not np_polygon2mask((9, 8), pts).any()


def test_horizontal_edges_never_divide(ed):
    rect = np.array([[2.0, 3.0], [6.0, 3.0], [6.0, 7.0], [2.0, 7.0]])
    want = np.zeros((10, 10), bool)
    want[2:6, 3:7] = True
    assert np.array_equal(ed.polygon2mask_rs((10, 10), rect), want)


def test_behind_the_camera_or_beyond_depth_is_kept(ed):
    w, h = 13, 11
    M, MV = _ortho(w, h)
    base = random_mask(np.random.default_rng(2), (4, 10, 14), 0.8)
    everything = np.ones((h, w), bool)
    behind = M.copy(); behind[3, 3] = -1.0     # q_w < 0
    on_plane = M.copy(); on_plane[3, 3] = 0.0   # q_w == 0
    for m, depth in ((behind, 1e9), (on_plane, 1e9), (M, -1.0), (M, float("nan"))):
        for mode in (0, 1):
            got = base.copy()
            ed.mask_cut(base, 1.0, 1.0, 1.0, depth, everything, m, MV, got, mode)
            assert np.array_equal(got, base)


@pytest.mark.parametrize("vp", [(0, 5), (5, 0), (0, 0)])
def test_empty_viewport_puts_everything_off_screen(ed, vp):
    w, h = vp
    M, MV = _ortho(7, 7)
    base = random_mask(np.random.default_rng(3), (3, 6, 6), 0.8)
    empty = np.zeros((h, w), bool)
    for mode, want in ((0, np.where(base > 127, 0, base).astype(np.uint8)), (1, base)):
        got = base.copy()
        ed.mask_cut(base, 1.0, 1.0, 1.0, 1e9, empty, M, MV, got, mode)
        assert np.array_equal(got, want), mode
        ref = base.copy()
        np_mask_cut(1.0, 1.0, 1.0, 1e9, empty, M, MV, ref, mode)
        assert np.array_equal(ref, want), mode


# ----------------------------------------------------------------------------- argument checks
def _cut_args(**kw):
    a = dict(image=np.zeros((2, 3, 4), np.int16), sx=1.0, sy=1.0, sz=1.0, max_depth=5.0,
             mask=np.zeros((4, 5), bool), m=np.eye(4), mv=np.eye(4), out=np.zeros((3, 4, 5), np.uint8), edit_mode=0)
    a.update(kw)
    return a


@pytest.mark.parametrize("kw, exc", [
    (dict(image=np.zeros((2, 3, 4), np.float32)), TypeError),
    (dict(image=np.zeros((3, 4), np.int16)), TypeError),
    (dict(out=np.zeros((3, 4, 5), np.int16)), TypeError),
    (dict(out=np.zeros((4, 5), np.uint8)), TypeError),
    (dict(out=np.broadcast_to(np.zeros(1, np.uint8), (3, 4, 5))), TypeError),     # read-only
    (dict(mask=np.zeros((4, 5), np.uint8)), TypeError),
    (dict(mask=np.zeros((2, 4, 5), bool)), TypeError),
    (dict(m=np.eye(4, dtype=np.float32)), TypeError),
    (dict(mv=np.eye(4).reshape(1, 4, 4)), TypeError),
    (dict(m=np.asfortranarray(np.arange(16.0).reshape(4, 4))), ValueError),      # not C-contiguous
    (dict(mv=np.eye(3)), ValueError),                                             # 9 elements
    (dict(edit_mode=2 ** 31), OverflowError),
    (dict(edit_mode=1.0), TypeError),
])
def test_mask_cut_argument_errors(kw, exc):
    from invesalius3_b200.mask_editor import mask_cut
    with pytest.raises(exc):
        mask_cut(**_cut_args(**kw))


def test_brush_argument_errors():
    from invesalius3_b200.mask_editor import brush_mask_rs
    out = np.zeros((5, 6, 7), np.uint8)
    with pytest.raises(ValueError):
        brush_mask_rs(out, np.zeros((5, 6, 6), np.uint8), (1.0, 1.0, 1.0), (2.0, 2.0, 2.0), 2.0, 0)
    with pytest.raises(TypeError):
        brush_mask_rs(out, np.zeros((5, 6, 7), np.int16), (1.0, 1.0, 1.0), (2.0, 2.0, 2.0), 2.0, 0)
    with pytest.raises(TypeError):
        brush_mask_rs(out.astype(np.float64), None, (1.0, 1.0, 1.0), (2.0, 2.0, 2.0), 2.0, 0)
    with pytest.raises(TypeError):
        brush_mask_rs(out[0], None, (1.0, 1.0, 1.0), (2.0, 2.0, 2.0), 2.0, 0)
    with pytest.raises(OverflowError):
        brush_mask_rs(out, None, (1.0, 1.0, 1.0), (2.0, 2.0, 2.0), 2.0, -(2 ** 31) - 1)


@pytest.mark.parametrize("poly, exc", [
    (np.array([[1.0, 2.0], [np.nan, 3.0], [4.0, 4.0]]), ValueError),
    (np.array([[1.0, 2.0], [np.inf, 3.0], [4.0, 4.0]]), ValueError),
    (np.array([[1.0, -np.inf], [2.0, 3.0], [4.0, 4.0]]), ValueError),
    (np.array([[1, 2], [2, 3], [4, 4]], np.float32), TypeError),
    (np.array([1.0, 2.0, 3.0]), TypeError),
])
def test_polygon_argument_errors(poly, exc):
    from invesalius3_b200.mask_editor import polygon2mask_rs
    with pytest.raises(exc):
        polygon2mask_rs((10, 10), poly)
