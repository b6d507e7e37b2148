"""The 3-D mask editor on the device (invesalius3_b200.mask_editor) against the C restatement of
polygon_mask.rs, mask_cut.rs and brush_mask.rs (oracle/editor.c): equal on every case."""
import numpy as np
import pytest

from test_oracle_editor import ed, editor_filter, random_camera, star_polygon, tangled_polygon  # noqa: F401 (ed: fixture)

pytestmark = pytest.mark.gpu


def _bone(shape, seed):
    from invesalius3_b200 import phantom
    vol = phantom.ct(shape, seed=seed)
    m = np.where((vol >= 226) & (vol <= 3071), 255, 0).astype(np.uint8)
    m[(vol > 100) & (vol < 150)] = 254          # selected too (> 127)
    m[(vol > 0) & (vol < 20)] = 2               # never selected
    return vol, m


def _padded(m):
    """The mask as the editor holds it: the [1:, 1:, 1:] view of a (dz+1, dy+1, dx+1) array."""
    p = np.full(tuple(s + 1 for s in m.shape), 7, np.uint8)
    p[1:, 1:, 1:] = m
    return p, p[1:, 1:, 1:]


@pytest.mark.parametrize("edit_mode", [0, 1, 2])
def test_mask_cut_matches_oracle(ed, edit_mode):
    from invesalius3_b200 import mask_editor as me
    rng = np.random.default_rng(100 + edit_mode)
    sp = (0.83, 0.91, 1.4)
    for k, shape in enumerate([(37, 61, 83), (50, 45, 29), (1, 33, 70), (23, 1, 17)]):
        vol, mask = _bone(shape, seed=k)
        images = [vol[:-1], mask[:, :3], vol.astype(np.float64)[::2]]        # dtype only; shapes differ from out
        for c in range(3):
            w, h = [(96, 64), (61, 97), (128, 80)][c]
            M, MV, near, far = random_camera(rng, shape, sp, w, h)
            polys = [star_polygon(rng, w, h, 15), tangled_polygon(rng, w, h, 9)][: 1 + c % 2]
            filt = editor_filter(polys, w, h, edit_mode, me.polygon2mask_rs)
            assert np.array_equal(filt, editor_filter(polys, w, h, edit_mode, ed.polygon2mask_rs))
            depth = near + (far - near) * [1.0, 0.5, 0.25][c]
            want = mask.copy()
            ed.mask_cut(vol, *sp, depth, filt, M, MV, want, edit_mode)
            padded, got = _padded(mask)
            me.mask_cut(images[c], *sp, depth, filt, M, MV, got, edit_mode)
            assert np.array_equal(got, want), (shape, c)
            assert (padded[0] == 7).all() and (padded[:, 0] == 7).all() and (padded[:, :, 0] == 7).all()
            dense = mask.copy()
            me.mask_cut(images[c], *sp, depth, filt, M, MV, dense, edit_mode)
            assert np.array_equal(dense, want), (shape, c)


def test_mask_cut_full_size(ed):
    """256 x 512 x 512 bone mask, include and exclude, as the editor calls it."""
    from invesalius3_b200 import mask_editor as me
    rng = np.random.default_rng(7)
    shape, sp = (256, 512, 512), (0.5, 0.5, 0.8)
    vol, mask = _bone(shape, seed=2)
    w, h = 1280, 800
    M, MV, near, far = random_camera(rng, shape, sp, w, h)
    for mode in (0, 1):
        filt = editor_filter([star_polygon(rng, w, h, 40)], w, h, mode, me.polygon2mask_rs)
        depth = near + (far - near) * 0.7
        want = mask.copy()
        ed.mask_cut(vol, *sp, depth, filt, M, MV, want, mode)
        padded, got = _padded(mask)
        me.mask_cut(vol, *sp, depth, filt, M, MV, got, mode)
        assert np.array_equal(got, want), mode
        assert (want != mask).sum() > 10000 and ((want == mask) & (mask > 127)).sum() > 10000


def test_mask_cut_device_keeps_the_mask_resident(ed):
    import torch
    from invesalius3_b200 import mask_editor as me
    rng = np.random.default_rng(9)
    shape, sp = (40, 70, 90), (0.7, 0.7, 1.1)
    vol, mask = _bone(shape, seed=4)
    t = torch.from_numpy(mask.copy()).cuda()
    want = mask.copy()
    for mode in (1, 0, 1):
        w, h = 100, 90
        M, MV, near, far = random_camera(rng, shape, sp, w, h)
        poly = star_polygon(rng, w, h, 20)
        f = me.polygon2mask_device((w, h), poly).T.contiguous()
        filt = ed.polygon2mask_rs((w, h), poly).T.copy()
        if mode == 0:
            f = 1 - f
            np.logical_not(filt, out=filt)
        me.mask_cut_device(t, sp, far, f, M, MV, mode)
        ed.mask_cut(vol, *sp, far, filt, M, MV, want, mode)
    assert np.array_equal(t.cpu().numpy(), want)


@pytest.mark.parametrize("vp", [(1280, 800), (1, 7), (7, 1), (33, 517), (0, 9)])
def test_polygon2mask_matches_oracle(ed, vp):
    from invesalius3_b200 import mask_editor as me
    w, h = vp
    rng = np.random.default_rng(w * 1000 + h)
    polys = [np.zeros((0, 2)), np.array([[0.2, 3.0]]), np.array([[0.0, 0.0], [5.0, 4.0]]),
             np.array([[0.0, 0.0], [w, 0.0], [w, h], [0.0, h]], np.float64)]
    for n in (3, 40, 511, 512, 513, 3000):             # 512 vertices per shared-memory chunk
        polys.append(star_polygon(rng, max(w, 1), max(h, 1), n))
        if n <= 513:
            polys.append(tangled_polygon(rng, max(w, 1), max(h, 1), n))
    polys.append(np.round(star_polygon(rng, max(w, 1), max(h, 1), 64)))
    polys.append(np.array([[-1e6, -1e6], [2e6, -5.0], [3.0, 4e6]]))       # far off-screen, clamped box
    for p in polys:
        got = me.polygon2mask_rs((w, h), p)
        want = ed.polygon2mask_rs((w, h), p)
        assert got.dtype == np.bool_ and got.shape == (w, h)
        assert np.array_equal(got, want), len(p)


def _brush_cases(shape, sp):
    ext = np.array(shape[::-1]) * np.array(sp)              # x, y, z extent in mm
    mid = ext / 2
    cases = [(tuple(mid), 6.0)]
    for axis in range(3):                                    # clipped at every face
        for at in (0.0, ext[axis]):
            c = mid.copy(); c[axis] = at + (-1.3 if at else 1.1)
            cases.append((tuple(c), 7.5))
    cases.append(((-4.0, mid[1], mid[2]), 6.0))             # centre outside, sphere reaches in
    cases.append(((-40.0, -40.0, -40.0), 5.0))              # centre far outside: no-op
    cases.append((tuple(ext + 2.0), 4.0))                     # beyond the last corner
    cases.append((tuple(mid), 1000.0))                       # the whole volume
    cases.append((tuple(mid), 0.0))                          # one voxel or none
    cases.append((tuple(mid), -3.0))                         # negative radius
    return cases


@pytest.mark.parametrize("edit_mode", [0, 1, 2])
def test_brush_matches_oracle(ed, edit_mode):
    from invesalius3_b200 import mask_editor as me
    sp = (0.45, 0.6, 1.25)
    for k, shape in enumerate([(29, 41, 53), (12, 1, 30)]):
        _, mask = _bone(shape, seed=10 + k)
        _, orig = _bone(shape, seed=20 + k)
        orig[orig == 2] = 0
        orig_padded, orig_view = _padded(orig)
        for centre, radius in _brush_cases(shape, sp):
            for o in (None, orig_view, orig):
                want = mask.copy()
                ed.brush_mask_rs(want, None if o is None else np.ascontiguousarray(o), sp, centre, radius, edit_mode)
                padded, got = _padded(mask)
                me.brush_mask_rs(got, o, sp, centre, radius, edit_mode)
                assert np.array_equal(got, want), (shape, centre, radius, o is None)
                assert (padded[0] == 7).all() and (padded[:, 0] == 7).all() and (padded[:, :, 0] == 7).all()
                dense = mask.copy()
                me.brush_mask_rs(dense, o, sp, centre, radius, edit_mode)
                assert np.array_equal(dense, want)


def test_brush_device_on_a_resident_volume(ed):
    import torch
    from invesalius3_b200 import mask_editor as me
    shape, sp = (31, 47, 59), (0.5, 0.7, 1.3)
    _, mask = _bone(shape, seed=3)
    _, orig = _bone(shape, seed=5)
    t, to = torch.from_numpy(mask.copy()).cuda(), torch.from_numpy(orig).cuda()
    want = mask.copy()
    for i, (centre, radius) in enumerate(_brush_cases(shape, sp)):
        mode, o = i % 2, (to if i % 3 else None)
        me.brush_mask_device(t, o, sp, centre, radius, mode)
        ed.brush_mask_rs(want, orig if i % 3 else None, sp, centre, radius, mode)
    assert np.array_equal(t.cpu().numpy(), want)


def test_a_brush_stroke_moves_only_its_box(monkeypatch):
    from invesalius3_b200 import device as dev
    from invesalius3_b200 import mask_editor as me
    moved = []
    to_device, to_host = dev.to_device, dev.to_host

    def rec_to_device(a, device=None):
        moved.append(("h2d", a.shape))
        return to_device(a, device)

    def rec_to_host(t, out):
        moved.append(("d2h", out.shape))
        return to_host(t, out)

    monkeypatch.setattr(dev, "to_device", rec_to_device)
    monkeypatch.setattr(dev, "to_host", rec_to_host)
    shape, sp = (120, 160, 200), (0.5, 0.5, 1.0)
    padded = np.zeros(tuple(s + 1 for s in shape), np.uint8)
    orig = np.full_like(padded, 200)
    centre, radius = (40.0, 35.0, 60.0), 5.0
    box = me.brush_mask_box(shape, sp, centre, radius)
    bshape = tuple(hi - lo + 1 for lo, hi in box)
    me.brush_mask_rs(padded[1:, 1:, 1:], orig[1:, 1:, 1:], sp, centre, radius, 0)
    assert moved == [("h2d", bshape), ("h2d", bshape), ("d2h", bshape)]
    assert np.prod(bshape) < 25 * 25 * 15
    assert (padded == 200).sum() > 0 and np.isin(padded, (0, 200)).all()
