"""GPU parity for the flood-fill family, called through the invesalius_rs-shaped shim
(numpy in/out -> C ABI). Known answers are the reference's own
(tests/test_segmentation_tools.py:17-134); everything else is checked bit-exact against
the oracle on seeded inputs."""
import numpy as np
import pytest
from scipy import ndimage
from scipy.ndimage import generate_binary_structure

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rs():
    from invesalius3_b200 import device, invesalius_rs
    device.require_cuda()
    return invesalius_rs


@pytest.fixture(autouse=True, params=["persistent", "host-rounds"])
def engine(request):
    """Every test runs on both convergence engines (one cooperative launch / a launch per round)."""
    from invesalius3_b200 import _lib
    lib = _lib.load()
    lib.b2v_floodfill_set_engine(1 if request.param == "persistent" else 0)
    yield request.param
    lib.b2v_floodfill_set_engine(1)


def test_region_growing_threshold(rs):
    image = np.array([[[1, 1, 1, 5, 5], [1, 2, 2, 5, 5], [1, 2, 3, 5, 5], [1, 2, 2, 5, 5], [1, 1, 1, 5, 5]]],
                     dtype=np.int16)
    out_mask = np.zeros((1, 5, 5), dtype=np.uint8)
    rs.floodfill_threshold(image, [[2, 2, 0]], 2, 3, 1, generate_binary_structure(3, 1), out_mask)
    expected = np.array([[0, 0, 0, 0, 0], [0, 1, 1, 0, 0], [0, 1, 1, 0, 0], [0, 1, 1, 0, 0], [0, 0, 0, 0, 0]],
                        dtype=np.uint8)
    assert np.array_equal(out_mask[0], expected)


def test_region_growing_strct_disconnected(rs):
    image = np.array([[[2, 2, 0], [0, 2, 0], [0, 0, 2]]], dtype=np.int16)
    out8 = np.zeros((1, 3, 3), dtype=np.uint8)
    rs.floodfill_threshold(image, [[0, 0, 0]], 2, 2, 1, generate_binary_structure(3, 2), out8)
    assert np.array_equal(out8, np.array([[[1, 1, 0], [0, 1, 0], [0, 0, 1]]], dtype=np.uint8))
    out4 = np.zeros((1, 3, 3), dtype=np.uint8)
    rs.floodfill_threshold(image, [[0, 0, 0]], 2, 2, 1, generate_binary_structure(3, 1), out4)
    assert np.array_equal(out4, np.array([[[1, 1, 0], [0, 1, 0], [0, 0, 0]]], dtype=np.uint8))


def test_fill_holes_automatically(rs):
    mask_2d = np.ones((7, 7), dtype=np.uint8)
    mask_2d[3, 3] = 0
    mask = mask_2d[np.newaxis, ...]
    labels_2d, nlabels = ndimage.label(mask_2d == 0, structure=np.ones((3, 3), np.uint8), output=np.uint32)
    border = set(labels_2d[:, 0]) | set(labels_2d[:, -1]) | set(labels_2d[0, :]) | set(labels_2d[-1, :])
    for bl in border:
        labels_2d[labels_2d == bl] = 0
    labels = labels_2d[np.newaxis, ...]
    ret = rs.fill_holes_automatically(mask, labels, int(labels.max()), 1)
    expected = np.ones((1, 7, 7), dtype=np.uint8)
    expected[0, 3, 3] = 254
    assert ret and np.array_equal(mask, expected)


STRUCTS = {
    "6": generate_binary_structure(3, 1), "18": generate_binary_structure(3, 2), "26": generate_binary_structure(3, 3),
    "133": np.ones((1, 3, 3), bool), "313": np.ones((3, 1, 3), bool), "331": np.ones((3, 3, 1), bool),
    "2d4": generate_binary_structure(2, 1)[None], "even": np.ones((2, 2, 2), np.uint8),
}


def _blobs(shape, seed, lo=-1000, hi=2000, smooth=2.0):
    rng = np.random.default_rng(seed)
    f = ndimage.gaussian_filter(rng.normal(size=shape), smooth)
    f = (f - f.min()) / (f.max() - f.min() + 1e-9)
    return (lo + f * (hi - lo)).astype(np.int16)


@pytest.mark.parametrize("shape", [(1, 5, 5), (7, 9, 11), (33, 65, 129), (40, 70, 300), (70, 50, 600)])
@pytest.mark.parametrize("sname", list(STRUCTS))
def test_floodfill_threshold_matches_oracle(rs, orc, shape, sname):
    st = STRUCTS[sname]
    data = _blobs(shape, 3)
    rng = np.random.default_rng(5)
    t0, t1 = 300, 2000
    seeds = [(int(rng.integers(shape[2])), int(rng.integers(shape[1])), int(rng.integers(shape[0]))) for _ in range(6)]
    zz, yy, xx = np.nonzero(data >= 900)
    if len(zz):
        seeds.append((int(xx[0]), int(yy[0]), int(zz[0])))
    out0 = np.zeros(shape, np.uint8)
    out0[rng.random(shape) < 0.02] = 1        # pre-filled walls
    out0[rng.random(shape) < 0.02] = 200      # unrelated values stay untouched
    want, got = out0.copy(), out0.copy()
    orc.floodfill_threshold(data, seeds, t0, t1, 1, st, want)
    rs.floodfill_threshold(data, seeds, t0, t1, 1, st, got)
    assert np.array_equal(got, want), (shape, sname, int((got != want).sum()))


def test_floodfill_asymmetric_structuring_element(rs, orc):
    """The walk is directed (p -> p + offset); a one-sided element must not be symmetrised."""
    rng = np.random.default_rng(11)
    for trial in range(6):
        st = (rng.random((3, 3, 3)) < 0.25).astype(np.uint8)
        data = (rng.random((12, 14, 70)) < 0.8).astype(np.int16)
        seeds = [(35, 7, 6), (0, 0, 0), (69, 13, 11)]
        want = np.zeros(data.shape, np.uint8); got = want.copy()
        orc.floodfill_threshold(data, seeds, 1, 1, 7, st, want)
        rs.floodfill_threshold(data, seeds, 1, 1, 7, st, got)
        assert np.array_equal(got, want), trial


@pytest.mark.parametrize("dtype", [np.int16, np.uint8, np.float64])
def test_floodfill_dtypes_inplace_and_equal(rs, orc, dtype):
    rng = np.random.default_rng(2)
    shape = (9, 20, 45)
    base = rng.integers(0, 4, shape)
    data = (base * (1 if dtype != np.float64 else 1.5)).astype(dtype)
    st = generate_binary_structure(3, 1)
    seeds = [(3, 3, 3), (44, 19, 8), (10, 0, 0)]
    t0, t1 = (1, 2) if dtype != np.float64 else (1.5, 3.0)
    want = np.zeros(shape, np.uint8); got = want.copy()
    if dtype == np.float64:
        # reference quirk: the wrapper floats `fill` for f64 data and PyO3's `fill: u8` rejects
        # it (invesalius_rs/__init__.py:36-40, floodfill_py.rs:143) -> always TypeError
        with pytest.raises(TypeError):
            orc.floodfill_threshold(data, seeds, t0, t1, 9, st, want)
        with pytest.raises(TypeError):
            rs.floodfill_threshold(data, seeds, t0, t1, 9, st, got)
        # the f64 kernel itself is reachable from the device API: check it against the core
        import torch
        from invesalius3_b200 import device as dev
        orc._floodfill_threshold_core(data, seeds, t0, t1, 9, np.ascontiguousarray(st, np.uint8), want)
        o = torch.zeros(shape, dtype=torch.uint8, device="cuda")
        dev.floodfill_threshold(torch.from_numpy(data).cuda(), seeds, t0, t1, 9, st, o)
        got = o.cpu().numpy()
    else:
        orc.floodfill_threshold(data, seeds, t0, t1, 9, st, want)
        rs.floodfill_threshold(data, seeds, t0, t1, 9, st, got)
    assert np.array_equal(got, want) and want.any()
    a, b = data.copy(), data.copy()
    fill = 3 if dtype != np.float64 else 4.5
    orc.floodfill_threshold_inplace(a, seeds, t0, t1, fill, generate_binary_structure(3, 3))
    rs.floodfill_threshold_inplace(b, seeds, t0, t1, fill, generate_binary_structure(3, 3))
    assert np.array_equal(a, b)
    v = data[4, 4, 4]
    want = np.zeros(shape, np.uint8); got = want.copy()
    orc.floodfill(data, 4, 4, 4, v, 5, want)
    rs.floodfill(data, 4, 4, 4, v, 5, got)
    assert np.array_equal(got, want) and got[4, 4, 4] == 5


def test_floodfill_mask_edit_usage_on_memmap_view(rs, orc, tmp_path):
    """styles.py:2450-2458 / 2493: the callers pass mask.matrix[1:,1:,1:] (strided memmap)."""
    shape = (12, 30, 41)
    mm = np.memmap(tmp_path / "mask.dat", dtype=np.uint8, mode="w+", shape=tuple(s + 1 for s in shape))
    rng = np.random.default_rng(8)
    body = (ndimage.gaussian_filter(rng.normal(size=shape), 1.5) > 0).astype(np.uint8) * 255
    mm[1:, 1:, 1:] = body
    mm[1:, 0, 0] = 1
    ref = np.array(mm)
    view, rview = mm[1:, 1:, 1:], ref[1:, 1:, 1:]
    zz, yy, xx = np.nonzero(body == 0)
    seed = [(int(xx[0]), int(yy[0]), int(zz[0]))]
    st = generate_binary_structure(3, 1)
    rs.floodfill_threshold_inplace(view, seed, 0, 2, 254, st)    # "fill holes" tool
    orc.floodfill_threshold_inplace(rview, seed, 0, 2, 254, st)
    assert np.array_equal(np.array(mm), ref)
    zz, yy, xx = np.nonzero(body == 255)
    seed = [(int(xx[-1]), int(yy[-1]), int(zz[-1]))]
    rs.floodfill_threshold_inplace(view, seed, 253, 255, 1, st)  # "remove parts" tool
    orc.floodfill_threshold_inplace(rview, seed, 253, 255, 1, st)
    assert np.array_equal(np.array(mm), ref)
    # select parts: floodfill_threshold(mask -> select_mask) (styles.py:2932-2953)
    sel = np.zeros(shape, np.uint8); rsel = sel.copy()
    rs.floodfill_threshold(view, seed, 1, 1, 254, st, sel)
    orc.floodfill_threshold(rview, seed, 1, 1, 254, st, rsel)
    assert np.array_equal(sel, rsel)
    # 2-D usage: reshaped (1, dy, dx) slices (styles.py:3121-3134)
    sl = np.ascontiguousarray(body[5]).reshape(1, *body[5].shape)
    o1 = np.zeros(sl.shape, np.uint8); o2 = o1.copy()
    rs.floodfill_threshold(sl, [(0, 0, 0)], 0, 255, 1, np.ones((1, 3, 3), np.uint8), o1)
    orc.floodfill_threshold(sl, [(0, 0, 0)], 0, 255, 1, np.ones((1, 3, 3), np.uint8), o2)
    assert np.array_equal(o1, o2) and o1.all()


def test_floodfill_aliased_data_out(rs, orc):
    m = (np.random.default_rng(0).random((6, 9, 40)) < 0.6).astype(np.uint8) * 255
    want = m.copy()
    orc.floodfill_threshold_inplace(want, [(0, 0, 0)], int(m[0, 0, 0]), int(m[0, 0, 0]), 254,
                                    generate_binary_structure(3, 1))
    rs.floodfill_threshold(m, [(0, 0, 0)], int(m[0, 0, 0]), int(m[0, 0, 0]), 254, generate_binary_structure(3, 1), m)
    assert np.array_equal(m, want)


def test_floodfill_errors_and_edges(rs):
    data = np.zeros((4, 5, 6), np.int16)
    out = np.zeros(data.shape, np.uint8)
    st = generate_binary_structure(3, 1)
    rs.floodfill_threshold(data, [], 0, 0, 1, st, out)            # no seeds: nothing happens
    assert not out.any()
    rs.floodfill_threshold(data, [(1, 1, 1)], 5, 9, 1, st, out)   # seed fails the threshold: ignored
    assert not out.any()
    rs.floodfill_threshold(data, [(1, 1, 1)], 0, 0, 1, st, out)
    assert out.all()
    with pytest.raises(OverflowError):
        rs.floodfill_threshold(data, [(1, 1, 1)], 0, 40000, 1, st, out)
    with pytest.raises(IndexError):
        rs.floodfill_threshold(data, [(6, 1, 1)], 0, 0, 1, st, out)
    with pytest.raises(TypeError):
        rs.floodfill_threshold(data.astype(np.float32), [(1, 1, 1)], 0, 0, 1, st, out)
    with pytest.raises(TypeError):
        rs.floodfill_threshold(data, [(1, 1, 1)], 0, 0, 1, st, out.astype(np.int16))
    with pytest.raises(TypeError):
        rs.floodfill_threshold_inplace(data, [(1, 1, 1)], 0.5, 1, 1, st)
    with pytest.raises(ValueError):
        rs.floodfill_threshold(data, [(1, 1, 1)], 0, 0, 1, np.ones((5, 5, 5), np.uint8), out)


def test_fill_holes_matches_oracle(rs, orc):
    rng = np.random.default_rng(4)
    shape = (20, 40, 70)
    mask = (ndimage.gaussian_filter(rng.normal(size=shape), 1.2) > -0.1).astype(np.uint8) * 255
    st = generate_binary_structure(3, 1)
    labels, n = ndimage.label(~(mask > 127), st, output=np.uint32)
    for max_size in (0, 1, 5, 50, 10 ** 6):
        a, b = mask.copy(), mask.copy()
        ra = orc.fill_holes_automatically(a, labels, n, max_size)
        rb = rs.fill_holes_automatically(b, labels, n, max_size)
        assert ra == rb and np.array_equal(a, b), max_size
    with pytest.raises(ValueError):
        rs.fill_holes_automatically(mask.copy(), labels, n - 1, 5)  # label > nlabels panics in the reference


def test_floodfill_512_properties(rs):
    """Full-size (BASELINE config 2) checks that do not need the oracle: idempotence,
    containment in the threshold set, agreement with torch-side connected set growth."""
    import torch
    from invesalius3_b200 import device as dev, phantom
    vol = phantom.ct((256, 512, 512), seed=2)
    seed = phantom.first_seed_in_range(vol, 128, 226, 3071)
    t = torch.from_numpy(vol).cuda()
    out = torch.zeros(vol.shape, dtype=torch.uint8, device="cuda")
    st = generate_binary_structure(3, 1)
    rounds = dev.floodfill_threshold(t, [seed], 226, 3071, 1, st, out)
    assert rounds > 0
    n1 = int(out.sum())
    assert n1 > 1000
    inrange = (t >= 226) & (t <= 3071)
    assert not bool((out.bool() & ~inrange).any())
    # closed under one more dilation step restricted to the threshold set
    o = out.bool()
    grown = o.clone()
    grown[1:] |= o[:-1]; grown[:-1] |= o[1:]
    grown[:, 1:] |= o[:, :-1]; grown[:, :-1] |= o[:, 1:]
    grown[:, :, 1:] |= o[:, :, :-1]; grown[:, :, :-1] |= o[:, :, 1:]
    assert torch.equal(grown & inrange, o)
    # idempotent: running again from the same seed changes nothing
    out2 = out.clone()
    dev.floodfill_threshold(t, [seed], 226, 3071, 1, st, out2)
    assert torch.equal(out, out2)


def test_floodfill_and_surface_full_size_exact(rs, orc):
    """Full-size volume (a 256 x 512 x 512 half of BASELINE config 2) against the serial CPU checker,
    exactly: the grown mask for 6- and 26-connectivity, and the mesh contoured from it (triangle
    indices bit for bit, vertices equal)."""
    import torch
    from invesalius3_b200 import device as dev, phantom
    from invesalius3_b200.mesh import marching_cubes
    vol = phantom.ct((256, 512, 512), seed=2)
    seed = phantom.first_seed_in_range(vol, 128, 226, 3071)
    t = torch.from_numpy(vol).cuda()
    for conn in (1, 3):
        st = generate_binary_structure(3, conn)
        out = torch.zeros(vol.shape, dtype=torch.uint8, device="cuda")
        dev.floodfill_threshold(t, [seed], 226, 3071, 254, st, out)
        want = np.zeros(vol.shape, np.uint8)
        orc.floodfill_threshold(vol, [seed], 226, 3071, 254, st, want)
        assert np.array_equal(out.cpu().numpy(), want), conn
        if conn == 1:
            v, f = marching_cubes(out, 127, (1.0, 1.0, 1.0), (0, 0, 0), True)
            vo, fo = orc.marching_cubes(want, 127, (1.0, 1.0, 1.0), (0, 0, 0), True)
            assert np.array_equal(f.cpu().numpy(), fo) and np.array_equal(v.cpu().numpy(), vo)


def test_floodfill_wide_rows_many_x_tiles(rs, orc):
    """2048-wide rows (BASELINE config 5 geometry): 64 words per row = 4 tiles along x."""
    rng = np.random.default_rng(12)
    shape = (5, 37, 2048)
    data = (ndimage.gaussian_filter(rng.normal(size=shape), (1, 2, 6)) > -0.05).astype(np.int16) * 1000
    seeds = [(3, 3, 0), (2040, 30, 4), (1024, 18, 2)]
    for conn in (1, 3):
        st = generate_binary_structure(3, conn)
        want = np.zeros(shape, np.uint8); got = want.copy()
        orc.floodfill_threshold(data, seeds, 500, 1500, 200, st, want)
        rs.floodfill_threshold(data, seeds, 500, 1500, 200, st, got)
        assert np.array_equal(got, want), conn
        assert (want == 200).sum() > 1000


@pytest.mark.parametrize("shape", [(37, 45, 1100), (16, 16, 544), (33, 17, 2048), (8, 8, 1100)])
def test_floodfill_canonical_tiles_across_x(rs, orc, shape):
    """The 6-connected fast path on 16 x 16 x 16-word tiles with several tiles along x (rows
    wider than 512 voxels), partial tiles on every side: the run fill has to cross word and
    tile boundaries through the halo words. Also in place. (8 x 8 x 1100 has 8 x 8-row tiles,
    which the generic 6-connected tile processor takes.)"""
    rng = np.random.default_rng(31)
    # long thin structures along x so that the flood travels through many x tiles
    data = (ndimage.gaussian_filter(rng.normal(size=shape), (1.5, 1.5, 12)) > 0.0).astype(np.int16) * 1000
    dz, dy, dx = shape
    seeds = [(1, 1, 0), (dx - 2, dy - 2, dz - 1), (dx // 2, dy // 2, dz // 2), (515, 3, 5)]
    st = generate_binary_structure(3, 1)
    want = np.zeros(shape, np.uint8)
    orc.floodfill_threshold(data, seeds, 500, 1500, 200, st, want)
    assert (want == 200).sum() > 5000
    got = np.zeros(shape, np.uint8)
    rs.floodfill_threshold(data, seeds, 500, 1500, 200, st, got)
    assert np.array_equal(got, want)
    mask = (data > 0).astype(np.uint8) * 255
    want_ip = mask.copy(); got_ip = mask.copy()
    orc.floodfill_threshold_inplace(want_ip, seeds, 255, 255, 7, st)
    rs.floodfill_threshold_inplace(got_ip, seeds, 255, 255, 7, st)
    assert np.array_equal(got_ip, want_ip)
