"""The "Remove tiny objects" plugin on the device (invesalius3_b200.tiny_objects) against the NumPy / SciPy model
of tests/tiny_objects_model.py, bit for bit: labels, their number, the region-size image, the preview bytes and the
whole padded mask after removal, flag planes included. Also count_regions for every label dtype, and the size
table, preview and removal kernels on a volume of more than 2^31 voxels."""
import numpy as np
import pytest
import torch

import tiny_objects_model as M

pytestmark = pytest.mark.gpu

MARKERS = np.array([0, 1, 2, 253, 254, 255], np.uint8)


def _sweep(counts):
    """The min_size values every case runs: 0, 1, 10, 10^3, the largest region and -1."""
    return [0, 1, 10, 1000, int(counts.max()), -1]


def _check(mask, min_sizes=None, t=None):
    """TinyObjects(mask) (or the given state) against the model at each min_size; returns the model's counts."""
    from invesalius3_b200.tiny_objects import TinyObjects
    labels, n, counts = M.find_regions(mask)
    t = t or TinyObjects(mask)
    assert t.num_labels == n
    assert np.array_equal(t.labels.cpu().numpy(), labels)
    assert np.array_equal(t.counts(), counts)
    for ms in (_sweep(counts) if min_sizes is None else min_sizes):
        want_p = M.preview(counts, ms)
        got_p = t.preview(ms)
        assert np.array_equal(got_p, want_p), ms
        want_m = M.remove(mask, want_p)
        got_m = mask.copy()
        t.remove(got_m, ms)
        assert np.array_equal(got_m, want_m), ms
        got_a = mask.copy()
        t.apply_preview(got_a, want_p)
        assert np.array_equal(got_a, want_m), ms
    return counts


@pytest.mark.parametrize("density", [0.05, 0.2, 0.35, 0.6])
def test_random_masks(density):
    rng = np.random.default_rng(int(density * 100))
    for shape in ((7, 33, 45), (40, 96, 128)):       # odd sizes: the preview's scalar tail
        body = np.where(rng.random(shape) < density, 255, 0).astype(np.uint8)
        _check(M.padded(body, rng))


def test_more_than_65535_labels():
    rng = np.random.default_rng(11)
    body = np.where(rng.random((64, 256, 256)) < 0.1, 255, 0).astype(np.uint8)
    mask = M.padded(body, rng)
    _check(mask, [0, 1, 2, 10])
    assert M.find_regions(mask)[1] > 65535


def test_every_marker_value():
    """1, 2, 253 and 254 are features like 255; so is any other non-zero byte."""
    rng = np.random.default_rng(5)
    for p0 in (0.3, 0.7):
        p = np.full(len(MARKERS), (1 - p0) / (len(MARKERS) - 1))
        p[0] = p0
        body = rng.choice(MARKERS, size=(24, 50, 70), p=p)
        _check(M.padded(body, rng))
    body = rng.integers(0, 256, size=(16, 40, 52), dtype=np.uint8)
    body[rng.random(body.shape) < 0.6] = 0
    _check(M.padded(body, rng))


def test_empty_and_full_masks():
    rng = np.random.default_rng(3)
    shape = (9, 20, 31)
    n = 9 * 20 * 31
    for fill in (0, 255, 1):
        body = np.full(shape, fill, np.uint8)
        counts = _check(M.padded(body, rng), [0, 1, n - 1, n, n + 1, 2 ** 32 - 1, 2 ** 32, 2 ** 40, -1, -(2 ** 40)])
        assert (counts == n).all()
    from invesalius3_b200.tiny_objects import TinyObjects
    assert TinyObjects(M.padded(np.zeros(shape, np.uint8), rng)).num_labels == 0


def test_resident_state_through_a_sweep():
    """One state driven like the open dialog: preview, remove, then refresh on the modified mask; at each step it
    equals a fresh state and the model."""
    from invesalius3_b200.tiny_objects import TinyObjects
    rng = np.random.default_rng(8)
    body = np.where(rng.random((30, 64, 80)) < 0.3, 255, 0).astype(np.uint8)
    body[rng.random(body.shape) < 0.05] = 254
    mask = M.padded(body, rng)
    t = TinyObjects(mask)
    _, _, counts = M.find_regions(mask)
    for ms in _sweep(counts):
        fresh = TinyObjects(mask)
        assert t.num_labels == fresh.num_labels
        assert torch.equal(t.labels, fresh.labels) and torch.equal(t.sizes, fresh.sizes)
        _, _, counts = M.find_regions(mask)
        want_p = M.preview(counts, ms)
        out = np.full(want_p.shape, 17, np.uint8)
        assert t.preview(ms, out=out) is out
        assert np.array_equal(out, want_p) and np.array_equal(fresh.preview(ms), want_p)
        want_m = M.remove(mask, want_p)
        t.remove(mask, ms)
        assert np.array_equal(mask, want_m), ms
        t.refresh(mask)


def test_preview_into_a_memmap(tmp_path):
    """The plugin's preview matrix is a uint8 memmap of the body's shape."""
    from invesalius3_b200.tiny_objects import TinyObjects
    rng = np.random.default_rng(2)
    body = np.where(rng.random((12, 30, 40)) < 0.25, 255, 0).astype(np.uint8)
    mask = M.padded(body, rng)
    mm = np.memmap(tmp_path / "mask.dat", mode="w+", dtype=np.uint8, shape=mask.shape)
    mm[:] = mask
    pv = np.memmap(tmp_path / "preview.dat", mode="w+", dtype=np.uint8, shape=body.shape)
    t = TinyObjects(mm)
    t.preview(10, out=pv)
    _, _, counts = M.find_regions(mask)
    assert np.array_equal(pv, M.preview(counts, 10))
    t.apply_preview(mm, pv)
    assert np.array_equal(mm, M.remove(mask, M.preview(counts, 10)))


def test_bad_arguments():
    from invesalius3_b200.tiny_objects import TinyObjects
    mask = M.padded(np.full((4, 5, 6), 255, np.uint8))
    t = TinyObjects(mask)
    with pytest.raises(TypeError):
        t.preview(1.5)
    with pytest.raises(ValueError):
        t.preview(1, out=np.empty((4, 5, 7), np.uint8))
    with pytest.raises(ValueError):
        t.remove(np.zeros((5, 6, 8), np.uint8), 1)
    with pytest.raises(ValueError):
        t.apply_preview(mask.copy(), np.zeros((4, 5, 6), np.int16))
    with pytest.raises(TypeError):
        TinyObjects(mask.astype(np.int16))
    with pytest.raises(ValueError):
        TinyObjects(np.zeros((1, 5, 6), np.uint8))


def _cranium_masks(cranium):
    shape = tuple(int(s) for s in cranium["full_shape"])
    n = int(np.prod(shape))
    for i in (0, 1):
        bits = np.unpackbits(cranium[f"mask_{i}_bits_full"])[:n].reshape(shape)
        m = np.zeros(tuple(s + 1 for s in shape), np.uint8)
        m[1:, 1:, 1:] = bits * np.uint8(255)
        m[0, :, :] = 1
        yield m


def test_cranium_masks(cranium):
    for mask in _cranium_masks(cranium):
        _check(mask)


def test_thresholded_phantom_256x512x512():
    from invesalius3_b200 import phantom
    vol = phantom.ct((256, 512, 512), seed=2)
    body = np.where((vol >= 226) & (vol <= 3071), 255, 0).astype(np.uint8)
    del vol
    mask = np.zeros(tuple(s + 1 for s in body.shape), np.uint8)
    mask[1:, 1:, 1:] = body
    mask[1:, 0, 0] = 1
    del body
    counts = _check(mask, [10, 1000])
    assert counts.max() > 10 ** 6


@pytest.mark.parametrize("dtype", [np.int16, np.int32, np.int64, np.uint8])
def test_count_regions_every_label_dtype(dtype):
    from invesalius3_b200 import labeling
    from invesalius3_b200.invesalius_rs import count_regions
    rng = np.random.default_rng(4)
    shape = (20, 48, 60)
    lab, n = M.find_regions(M.padded(np.where(rng.random(shape) < 0.3, 255, 0).astype(np.uint8)))[:2]
    if dtype == np.uint8:
        lab, n = lab % 200, 199
    img = lab.astype(dtype)
    want = np.bincount(img.ravel(), minlength=n + 1)[img].astype(np.uint32)
    for fn in (count_regions, labeling.count_regions):
        got = fn(img, n)
        assert got.dtype == np.uint32 and np.array_equal(got, want)
    assert np.array_equal(count_regions(img, n + 5), want)         # a larger table changes nothing
    high = img.copy()
    high[3, 4, 5] = n + 1
    with pytest.raises(ValueError):
        count_regions(high, n)          # the reference indexes out of bounds and panics
    if dtype != np.uint8:
        neg = img.copy()
        neg[-1, -1, -1] = -1
        with pytest.raises(ValueError):
            count_regions(neg, n)
    if dtype == np.int64:
        big = img.copy()
        big[0, 0, 0] = 2 ** 33
        with pytest.raises(ValueError):
            count_regions(big, n)
    with pytest.raises(TypeError):
        count_regions(img.astype(np.uint32), n)


def test_count_regions_one_dominant_label():
    """A single label over the whole volume, and the background with a few scattered voxels."""
    from invesalius3_b200 import labeling
    for dtype in (torch.int16, torch.int32, torch.int64, torch.uint8):
        t = torch.zeros((64, 128, 129), dtype=dtype, device="cuda")
        assert labeling.region_sizes_device(t, 0).cpu().tolist() == [t.numel()]
        t.view(-1)[::997] = 3
        n3 = (t.numel() + 996) // 997
        assert labeling.region_sizes_device(t, 3).cpu().tolist() == [t.numel() - n3, 0, 0, n3]


def test_kernels_past_2_31_voxels():
    """The size table, the preview and the removal on a label image of 2^31 + 2^21 voxels, with labels placed
    past flat index 2^31 (and one before it)."""
    from invesalius3_b200 import _lib, labeling
    from invesalius3_b200.device import _p, _stream
    dz, dy, dx = 1025, 1024, 2048
    n = dz * dy * dx
    assert n > 2 ** 31
    pts = {1: [(1024, 1023, 2047), (1024, 0, 5)], 2: [(1000, 7, 9)]}
    labels = torch.zeros((dz, dy, dx), dtype=torch.int32, device="cuda")
    for lab, ps in pts.items():
        for p in ps:
            labels[p] = lab
    sizes = labeling.region_sizes_device(labels, 2)           # uint32 values in int32 tensors
    assert sizes.cpu().numpy().view(np.uint32).tolist() == [n - 3, 2, 1]
    out = labeling.count_regions_device(labels, 2)
    got = [out[p].item() & 0xFFFFFFFF for p in ((1024, 1023, 2047), (1000, 7, 9), (1024, 1023, 2046))]
    assert got == [2, 1, n - 3]
    del out
    prev = torch.empty(n, dtype=torch.uint8, device="cuda")
    _lib.call("b2v_tiny_objects_preview", _p(labels), n, _p(sizes), 3, 2, _p(prev), _stream())
    prev = prev.view(dz, dy, dx)
    assert int(prev.sum(dtype=torch.int64)) == 3 * 255
    assert all(prev[p].item() == 255 for ps in pts.values() for p in ps)
    del prev
    mask = torch.zeros((dz + 1, dy + 1, dx + 1), dtype=torch.uint8, device="cuda")
    mask[0] = 7
    mask[:, 0] = 7
    mask[:, :, 0] = 7
    _lib.call("b2v_tiny_objects_remove", _p(labels), dz, dy, dx, _p(sizes), 3, 1, _p(mask), _stream())
    z, y, x = pts[2][0]
    assert mask[z + 1, y + 1, x + 1].item() == 1
    assert int(mask[1:, 1:, 1:].sum(dtype=torch.int64)) == 1
    assert bool((mask[0] == 7).all()) and bool((mask[:, 0] == 7).all()) and bool((mask[:, :, 0] == 7).all())
