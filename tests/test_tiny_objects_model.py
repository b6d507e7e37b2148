"""The NumPy / SciPy model of the "Remove tiny objects" plugin (tests/tiny_objects_model.py) against hand-counted
cases. The GPU tests compare the device with this model."""
import numpy as np

import tiny_objects_model as M


def _hand_case():
    # body [1][3][5]; 6-connected regions in raster order of their first voxel:
    #   1: (0,0) (0,1)          size 2
    #   2: (0,4)                size 1   (marker 254)
    #   3: (1,3) (2,3) (2,4)    size 3   (marker 1 and 1)
    #   4: (2,0)                size 1   (marker 2)
    #   background: 15 - 7 = 8
    body = np.array([[[255, 255, 0, 0, 254],
                      [0, 0, 0, 1, 0],
                      [2, 0, 0, 1, 1]]], np.uint8)
    m = np.full((2, 4, 6), 7, np.uint8)
    m[1:, 1:, 1:] = body
    return m


def test_find_regions_hand_counted():
    m = _hand_case()
    labels, n, counts = M.find_regions(m)
    assert n == 4 and labels.dtype == np.int32
    assert np.array_equal(labels[0], [[1, 1, 0, 0, 2], [0, 0, 0, 3, 0], [4, 0, 0, 3, 3]])
    assert counts.dtype == np.uint32
    assert np.array_equal(counts[0], [[2, 2, 8, 8, 1], [8, 8, 8, 3, 8], [1, 8, 8, 3, 3]])


def test_preview_and_remove_hand_counted():
    m = _hand_case()
    _, _, counts = M.find_regions(m)
    p1 = M.preview(counts, 1)
    assert p1.dtype == np.uint8
    assert np.array_equal(p1[0] // 255, [[0, 0, 0, 0, 1], [0, 0, 0, 0, 0], [1, 0, 0, 0, 0]])
    p2 = M.preview(counts, 2)
    assert np.array_equal(p2[0] // 255, [[1, 1, 0, 0, 1], [0, 0, 0, 0, 0], [1, 0, 0, 0, 0]])
    out = M.remove(m, p2)
    want = m.copy()
    want[1, 1, 1] = want[1, 1, 2] = want[1, 1, 5] = want[1, 3, 1] = 1
    assert np.array_equal(out, want)
    assert np.array_equal(m, _hand_case())           # the input is not changed
    # min_size compares exactly with the uint32 sizes, as NumPy 2 does with a Python int
    assert not M.preview(counts, -1).any()
    assert (M.preview(counts, 2 ** 40) == 255).all()
    assert (M.preview(counts, 8) == 255).all()       # 8: the background too


def test_background_quirk():
    """The background is a region like any other: where it is no larger than min_size it is previewed and
    its voxels are "removed", i.e. set to 1."""
    body = np.full((2, 3, 4), 255, np.uint8)
    body[1, 2, 3] = 0
    m = np.zeros((3, 4, 5), np.uint8)
    m[1:, 1:, 1:] = body
    labels, n, counts = M.find_regions(m)
    assert n == 1 and counts[1, 2, 3] == 1 and (np.delete(counts.ravel(), -1) == 23).all()
    p = M.preview(counts, 1)
    assert p[1, 2, 3] == 255 and int(p.sum()) == 255
    out = M.remove(m, p)
    assert out[2, 3, 4] == 1 and int((out != m).sum()) == 1
    # after the removal the voxel is a feature (1 is non-zero): the one region now fills the body
    _, n2, counts2 = M.find_regions(out)
    assert n2 == 1 and (counts2 == 24).all()


def test_empty_body():
    m = np.zeros((4, 5, 6), np.uint8)
    m[0] = 1
    labels, n, counts = M.find_regions(m)
    assert n == 0 and not labels.any()
    assert (counts == 3 * 4 * 5).all()
    assert not M.preview(counts, 59).any() and (M.preview(counts, 60) == 255).all()
    out = M.remove(m, M.preview(counts, 60))
    assert (out[1:, 1:, 1:] == 1).all() and np.array_equal(out[0], m[0])
