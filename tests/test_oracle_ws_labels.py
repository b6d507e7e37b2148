"""The O(N) labelling checker of the device flood (oracle/watershed.c::orc_ws_labels), pinned on the
CPU.

  * 6-connected, both cost models: equal, labels AND ambiguous mask, bit for bit, to the
    whole-array NumPy restatement tests/ws_model.py on hundreds of random volumes: plateaus (2 to
    65536 grey levels), negative labels and the int16 extremes, marker blobs, the flat-array
    neighbourhood of mode 0 that wraps rows and planes, 2-D volumes (nz = 1 and 2-D arrays);
  * 18/26-connected: where the order-independence model (orc_ws_model) gives a voxel one label,
    that is the checker's label; the checker's mask is that model's "several labels" set;
  * hop counts on corridors whose length is known in closed form.
"""
import numpy as np
import pytest
from scipy.ndimage import generate_binary_structure

import ws_model
from oracle import watershed as W

EXTREMES = np.array([-32768, -32767, -1, 1, 32766, 32767], np.int16)


def _case(rng, maxdim=9, two_d=False):
    if two_d:
        shape = (1, int(rng.integers(1, 14)), int(rng.integers(1, 14)))
    else:
        shape = tuple(int(rng.integers(1, maxdim)) for _ in range(3))
    levels = int(rng.choice([2, 3, 8, 40, 300, 65536]))
    img = rng.integers(0, levels, shape).astype(np.uint16)
    mk = np.zeros(shape, np.int16)
    for _ in range(int(rng.integers(1, 6))):
        r = rng.random()
        if r < 0.4:
            lab = int(rng.choice(EXTREMES))
        elif r < 0.7:
            lab = int(rng.integers(1, 6)) * (1 if rng.random() < 0.6 else -1)
        else:
            lab = int(rng.integers(-32768, 32768)) or 7
        z, y, x = (int(rng.integers(s)) for s in shape)
        if rng.random() < 0.3:        # a small blob: markers next to markers of the same label
            mk[z: z + 2, y: y + 2, x: x + 2] = lab
        else:
            mk[z, y, x] = lab
    return img, mk


@pytest.mark.parametrize("mode", [0, 1])
def test_equals_numpy_model_six_connected(mode):
    rng = np.random.default_rng(7 + mode)
    st = generate_binary_structure(3, 1)
    amb_seen = neg_seen = 0
    for i in range(320):
        img, mk = _case(rng, two_d=(i % 5 == 4))
        lab, amb = W.ws_labels(img, mk, st, mode)
        want_lab, want_amb = ws_model.flood(img, mk, mode)
        assert np.array_equal(lab, want_lab), (i, img.shape)
        assert np.array_equal(amb, want_amb), (i, img.shape)
        amb_seen += int(amb.any())
        neg_seen += int((mk == -32768).any() and (lab == -32768).sum() > (mk == -32768).sum())
    # the family exercises what it claims to: ambiguous voxels, and -32768 spreading past its markers
    assert amb_seen > 50 and neg_seen > 10, (amb_seen, neg_seen)


@pytest.mark.parametrize("mode", [0, 1])
def test_two_d_arrays_equal_a_single_plane(mode):
    rng = np.random.default_rng(30 + mode)
    for _ in range(40):
        img, mk = _case(rng, two_d=True)
        lab2, amb2 = W.ws_labels(img[0], mk[0], generate_binary_structure(2, 1), mode)
        want_lab, want_amb = ws_model.flood(img, mk, mode)
        assert np.array_equal(lab2, want_lab[0]) and np.array_equal(amb2, want_amb[0])


def test_minus_32768_alone_is_not_ambiguous():
    """One marker of label -32768 on a plateau: every voxel it reaches has one label, so nothing is
    ambiguous (a set encoding that gives -32768 the code of "several labels" says otherwise)."""
    img = np.zeros((3, 4, 5), np.uint16)
    mk = np.zeros(img.shape, np.int16)
    mk[1, 2, 3] = -32768
    for mode in (0, 1):
        lab, amb = W.ws_labels(img, mk, generate_binary_structure(3, 1), mode)
        assert (lab == -32768).all() and not amb.any()
        want_lab, want_amb = ws_model.flood(img, mk, mode)
        assert np.array_equal(lab, want_lab) and np.array_equal(amb, want_amb)


@pytest.mark.parametrize("conn", [2, 3])
@pytest.mark.parametrize("mode", [0, 1])
def test_single_label_sets_decide_18_26(conn, mode):
    rng = np.random.default_rng(50 + 10 * conn + mode)
    st = generate_binary_structure(3, conn)
    for i in range(150):
        img, mk = _case(rng, two_d=(i % 6 == 5))
        lab, amb = W.ws_labels(img, mk, st, mode)
        _, sets = W.order_independence_model(img, mk, st, mode)
        assert np.array_equal(amb.astype(bool), sets == W.MULTI), i
        one = (sets != W.MULTI) & (sets != 0)
        assert np.array_equal(lab[one], sets[one].astype(np.int16)), i
        assert np.array_equal(lab == 0, sets == 0), i


@pytest.mark.parametrize("mode", [0, 1])
def test_hops_along_a_serpentine(mode):
    """A one-voxel corridor of known length: hop counts 0 .. L-1 along it, the two markers at its
    ends split it in the middle, the smaller label taking the voxel at equal hops."""
    ny, nx = 9, 14           # walls in columns 0 and nx - 1: mode 0's row wrap joins walls only
    img = np.full((1, ny, nx), 1000, np.uint16)
    path = []
    for y in range(0, ny, 2):
        xs = range(1, nx - 1) if (y // 2) % 2 == 0 else range(nx - 2, 0, -1)
        path += [(0, y, x) for x in xs]
        if y + 2 < ny:
            path.append((0, y + 1, nx - 2 if (y // 2) % 2 == 0 else 1))
    for p in path:
        img[p] = 10
    L = len(path)
    mk = np.zeros(img.shape, np.int16)
    mk[path[0]] = 5
    mk[path[-1]] = -2
    lab, amb, hops = W.ws_labels(img, mk, generate_binary_structure(3, 1), mode, return_hops=True)
    got = np.array([hops[p] for p in path])
    want = np.minimum(np.arange(L), np.arange(L)[::-1])
    assert np.array_equal(got, want)
    labels_on_path = np.array([lab[p] for p in path])
    k = np.arange(L)
    assert np.array_equal(labels_on_path, np.where(k < L - 1 - k, 5, -2))
    want_lab, want_amb = ws_model.flood(img, mk, mode)
    assert np.array_equal(lab, want_lab) and np.array_equal(amb, want_amb)
