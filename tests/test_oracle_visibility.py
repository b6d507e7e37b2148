"""The C checker of "Remove non-visible faces" (oracle/visibility.c) and the host-side argument checks of
invesalius3_b200.visible_faces, on the CPU: the camera restatement, occlusion by a nested shell, the
remove_visible branch, the merge and first-use numbering of vtkCleanPolyData, and the empty result."""
import math

import numpy as np
import pytest

from oracle import visibility as ov
from visibility_meshes import cube, icosphere, nested_shells, select_and_clean

ANGLE = 30.0 * 0.017453292519943295


def test_camera_distance_is_radius_over_sin_15():
    b = np.array([-3.0, 5.0, 1.0, 2.0, -7.0, 0.5])
    cams = ov.cameras(b)
    r = math.sqrt(8.0 ** 2 + 1.0 ** 2 + 7.5 ** 2) / 2
    assert np.all(cams[:, 28] == r)
    assert np.all(cams[:, 27] == r / math.sin(ANGLE * 0.5))
    centre = np.array([1.0, 1.5, -3.25])
    assert np.array_equal(cams[:, 19:22], np.tile(centre, (6, 1)))
    dist = np.linalg.norm(cams[:, 16:19] - centre, axis=1)
    np.testing.assert_allclose(dist, r / math.sin(math.radians(15)), rtol=1e-14)
    # the camera sits along each axis direction
    np.testing.assert_allclose((cams[:, 16:19] - centre) / dist[:, None], np.array(ov.DEFAULT_POSITIONS), atol=1e-15)


def test_single_point_bounds_use_unit_squared_diagonal():
    cams = ov.cameras(np.array([2.0, 2.0, -1.0, -1.0, 0.0, 0.0]))
    assert np.all(cams[:, 28] == 0.5)        # sqrt(1) * 0.5


def test_view_up_sequence_for_the_six_axes():
    cams = ov.cameras(np.array([0.0, 1.0, 0.0, 1.0, 0.0, 1.0]))
    want = [(0, 1, 0), (0, 1, 0), (0, 0, 1), (0, 0, 1), (-1, 0, 0), (-1, 0, 0)]
    assert np.array_equal(cams[:, 22:25], np.array(want, np.float64))


def test_clipping_range_on_a_known_box():
    cams = ov.cameras(np.array([0.0, 2.0, 0.0, 2.0, 0.0, 2.0]))
    D = (math.sqrt(12.0) * 0.5) / math.sin(ANGLE * 0.5)
    near0, far0 = D - 1.0, D + 1.0            # nearest and farthest corners along each axis
    near = 0.99 * near0 - (far0 - near0) * 0.5
    far = 1.01 * far0 + (far0 - near) * 0.5
    np.testing.assert_allclose(cams[:, 25], near, rtol=1e-13)
    np.testing.assert_allclose(cams[:, 26], far, rtol=1e-13)
    assert np.all(cams[:, 25] >= 0.001 * cams[:, 26])


def test_composite_matrix_maps_the_clipping_planes_to_depth_0_and_1():
    cams = ov.cameras(np.array([0.0, 2.0, 0.0, 2.0, 0.0, 2.0]))
    for c in cams:
        M = c[:16].reshape(4, 4)
        pos, fp = c[16:19], c[19:22]
        d = (fp - pos) / np.linalg.norm(fp - pos)
        for depth, want in ((c[25], 0.0), (c[26], 1.0)):
            p = M @ np.append(pos + depth * d, 1.0)
            assert abs(p[2] / p[3] - want) < 1e-12
            assert abs(p[0] / p[3]) < 1e-12 and abs(p[1] / p[3]) < 1e-12


def test_nested_shells_inner_removed_outer_kept():
    v, f, n_outer = nested_shells(1.0, 4)
    vo, fo, dbg = ov.remove_non_visible_faces(v, f, debug=True)
    vis = dbg["visible"]
    assert vis[:len(v) // 2].all() and not vis[len(v) // 2:].any()
    assert len(fo) == n_outer
    assert np.array_equal(vo[fo], v[f[:n_outer]])   # the outer shell's faces, in order, same geometry
    assert dbg["zbuf"].shape == (6, 800, 800)
    assert (dbg["zbuf"] < 1.0).any(axis=(1, 2)).all() and (dbg["zbuf"] >= 0).all()


def test_remove_visible_keeps_exactly_the_faces_with_an_invisible_vertex():
    v, f, n_outer = nested_shells(1.0, 3)
    vo, fo, dbg = ov.remove_non_visible_faces(v, f, remove_visible=True, debug=True)
    assert len(fo) == len(f) - n_outer
    assert np.array_equal(vo[fo], v[f[n_outer:]])
    wv, wf = select_and_clean(v, f, dbg["visible"], True)
    assert np.array_equal(vo, wv) and np.array_equal(fo, wf)


def test_first_use_numbering_and_partial_selection():
    # a sphere seen from +x only: the far side is invisible, faces come back renumbered by first use
    v, f = icosphere(2.0, 3)
    perm = np.random.default_rng(3).permutation(len(v))
    inv = np.argsort(perm)
    v2, f2 = v[perm], inv[f].astype(np.int32)
    vo, fo, dbg = ov.remove_non_visible_faces(v2, f2, positions=[(1, 0, 0)], debug=True)
    assert 0 < len(fo) < len(f2)
    wv, wf = select_and_clean(v2, f2, dbg["visible"], False)
    assert np.array_equal(vo, wv) and np.array_equal(fo, wf)
    first = [int(x) for x in dict.fromkeys(fo.reshape(-1).tolist())]
    assert first == list(range(len(vo)))


def test_merge_of_coincident_points_on_a_hand_built_mesh():
    # two triangles of a square in z = 0, as a soup: 6 vertices, two coincident pairs, one pair as -0 / +0;
    # a third face collapses after the merge (a line in VTK) but its points stay numbered
    v = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0],      # face 0
                  [-0.0, 0, 0], [1, 1, 0], [0, 1, 0],   # face 1: vertex 3 == vertex 0, vertex 4 == vertex 2
                  [2, 2, 0], [2, 2, 0], [0, 1, 0]],     # face 2: 6 == 7 -> degenerate
                 np.float32)
    f = np.arange(9, dtype=np.int64).reshape(3, 3)
    vo, fo = ov.remove_non_visible_faces(v, f)
    assert np.array_equal(fo, np.array([[0, 1, 2], [0, 2, 3]], np.int32))
    assert np.array_equal(vo, np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [2, 2, 0]], np.float32))
    assert np.signbit(vo[0, 0]) == np.signbit(v[0, 0])          # the first use's bits win
    vo2, fo2 = ov.remove_non_visible_faces(v[[3, 1, 2, 0, 4, 5, 6, 7, 8]], f)
    assert np.signbit(vo2[0, 0]) and np.array_equal(fo2, fo)


def test_leading_three_form_and_int32():
    v, f = cube(1.0)
    f4 = np.concatenate([np.full((len(f), 1), 3, np.int32), f], 1)
    a = ov.remove_non_visible_faces(v, f)
    b = ov.remove_non_visible_faces(v, f4.astype(np.int64))
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert len(a[1]) == 12 and len(a[0]) == 8


def test_empty_result():
    v, f = icosphere(1.0, 2)
    vo, fo = ov.remove_non_visible_faces(v, f, remove_visible=True)   # a lone convex shell: all visible
    assert vo.shape == (0, 3) and fo.shape == (0, 3)
    vo, fo = ov.remove_non_visible_faces(v, f[:0])
    assert vo.shape == (0, 3) and fo.shape == (0, 3)


def test_oracle_argument_errors():
    v, f = cube(1.0)
    with pytest.raises(TypeError):
        ov.remove_non_visible_faces(v.astype(np.float64), f)
    with pytest.raises(TypeError):
        ov.remove_non_visible_faces(v, f.astype(np.float32))
    with pytest.raises(ValueError):
        ov.remove_non_visible_faces(v, f + 8)
    with pytest.raises(ValueError):
        ov.remove_non_visible_faces(v, np.concatenate([np.full((12, 1), 4, np.int32), f], 1))
    with pytest.raises(ValueError):
        ov.remove_non_visible_faces(v, f, positions=[(1, 0, 0), (0, 0, 0)])
    bad = v.copy()
    bad[3, 1] = np.nan
    with pytest.raises(ValueError):
        ov.remove_non_visible_faces(bad, f)


def test_product_argument_errors_before_any_device_work():
    from invesalius3_b200 import visible_faces as vf
    v, f = cube(1.0)
    with pytest.raises(TypeError):
        vf.remove_non_visible_faces(v.astype(np.float64), f)
    with pytest.raises(TypeError):
        vf.remove_non_visible_faces(v, f.astype(np.uint8))
    with pytest.raises(TypeError):
        vf.remove_non_visible_faces(list(v), f)
    with pytest.raises(ValueError):
        vf.remove_non_visible_faces(v[:, :2].copy(), f)
    with pytest.raises(ValueError):
        vf.remove_non_visible_faces(v, f[:, :2].copy())
    with pytest.raises(ValueError):
        vf.remove_non_visible_faces(v, f, positions=[(0, 0, 0)])
    with pytest.raises(ValueError):
        vf.remove_non_visible_faces(v, f, positions=[(1, 0, np.inf)])
    with pytest.raises(ValueError):
        vf.remove_non_visible_faces(v, f, positions=[])
    bad = v.copy()
    bad[0, 0] = np.inf
    with pytest.raises(ValueError):
        vf.remove_non_visible_faces(bad, f)
    vo, fo = vf.remove_non_visible_faces(v, f[:0])
    assert vo.shape == (0, 3) and fo.shape == (0, 3) and fo.dtype == np.int32
