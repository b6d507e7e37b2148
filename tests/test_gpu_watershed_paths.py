"""The persistent watershed engine (watershed_fast.cu) and the generic kernels (watershed.cu) on the
paths that smooth-noise volumes never reach, checked on EVERY voxel — labels and ambiguous mask —
against the O(N) checker oracle/watershed.c::orc_ws_labels (pinned against tests/ws_model.py in
tests/test_oracle_ws_labels.py):

  * mazes: one-voxel corridors in high walls, so that a tile stays unsettled after kMaxSets sweep
    sets and re-queues itself (counted in b2v_ws_stats slot 3), in one 16^3 tile, over many tiles,
    on full aligned tiles, partial tiles and a 2-D slice;
  * the 24-bit hop limit of the 32-bit phase-2 keys: two corridors longer than 0xff0000 voxels that
    meet, so the labels where they meet are decided by hop counts above 2^24; exactly one fallback
    to 64-bit keys (slot 7), labels equal to the 64-bit-only run; and a case just under the limit;
  * unaligned images (the vector loads of full tiles switched off) and full / partial tiles mixed;
  * the int16 label extremes, exactly 256 and 257 distinct labels (32- / 64-bit keys), through the
    persistent engine, the generic kernels and 18 / 26-connected structures;
  * a 192 x 512 x 512 CT phantom through watershed_device, both algorithms.
"""
import ctypes as C
import time

import numpy as np
import pytest
from scipy import ndimage
from scipy.ndimage import generate_binary_structure

pytestmark = pytest.mark.gpu

SIX = generate_binary_structure(3, 1)
ALG = {0: "Watershed IFT", 1: "Watershed"}
WALL, FLOOR = 1000, 10
KEY_FULL_HOPS = 0xFF0000      # kKeyFull32 >> 8: a 32-bit key at or above it stops the 32-bit phase


@pytest.fixture(scope="module")
def wp():
    from invesalius3_b200 import device, watershed_process
    device.require_cuda()
    return watershed_process


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _stats(reset=True):
    from invesalius3_b200 import _lib
    out = (C.c_int * 8)()
    _lib.load().b2v_ws_stats(out, 1 if reset else 0)
    return list(out)


def _device(wp, img, mk, mode, st=SIX, img_t=None):
    lab, amb = wp.flood(_t(img.view(np.int16)) if img_t is None else img_t, _t(mk), st, ALG[mode], True)
    return lab.cpu().numpy(), amb.cpu().numpy()


def _assert_checker(got, img, mk, mode, st=SIX, what=""):
    from oracle import watershed as W
    lab, amb = got
    want_lab, want_amb = W.ws_labels(img, mk, st, mode)
    bad = np.flatnonzero((lab != want_lab).ravel())
    assert bad.size == 0, f"{what}: {bad.size} labels differ, first at {np.unravel_index(bad[0], img.shape)}"
    bad = np.flatnonzero((amb != want_amb).ravel())
    assert bad.size == 0, f"{what}: {bad.size} ambiguous flags differ, first at {np.unravel_index(bad[0], img.shape)}"


# ---- corridors --------------------------------------------------------------------------------------
def snake(shape, x_lo, x_hi):
    """Flat indices, in path order, of a one-voxel corridor that fills the volume: rows along x over
    [x_lo, x_hi] at even y of even z planes, each row joined to the next at its end through the odd
    row between them, the last row of a plane joined to the next plane through the odd plane."""
    nz, ny, nx = shape
    zs, ys = np.arange(0, nz, 2), np.arange(0, ny, 2)
    P, Y = len(zs), len(ys)
    up = (np.arange(P) % 2 == 0)[:, None]
    yy = np.where(up, ys[None, :], ys[::-1][None, :])
    zz = np.broadcast_to(zs[:, None], (P, Y))
    fwd = (np.arange(P * Y).reshape(P, Y) % 2) == 0
    xs = np.arange(x_lo, x_hi + 1)
    row = (zz[..., None] * ny + yy[..., None]) * nx + np.where(fwd[..., None], xs, xs[::-1])
    last = np.zeros((P, Y), bool)
    last[:, -1] = True
    cy = np.where(last, yy, yy + np.where(up, 1, -1))
    cz = np.where(last, zz + 1, zz)
    con = (cz * ny + cy) * nx + np.where(fwd, x_hi, x_lo)
    return np.concatenate([row, con[..., None]], axis=2).reshape(-1)[:-1]


def _check_path(path, shape):
    nz, ny, nx = shape
    d = np.abs(np.diff(path))
    assert np.isin(d, [1, nx, ny * nx]).all() and np.unique(path).size == path.size


def maze(shape, x_lo, x_hi, rng=None):
    path = snake(shape, x_lo, x_hi)
    img = np.full(shape, WALL, np.uint16)
    img.ravel()[path] = FLOOR if rng is None else rng.integers(FLOOR, FLOOR + 4, path.size)
    return img, path


# ---- mazes: tiles that re-queue themselves ----------------------------------------------------------
# rows stay inside the first tile column, so a tile holds 8 rows of a plane (and 8 planes): more
# than kMaxSets sweep sets' worth of turns
MAZES = [
    ("one_tile", (16, 16, 16), 1, 14),          # one full aligned tile
    ("tiles", (48, 64, 64), 1, 14),             # 12 full aligned tiles along the corridor
    ("partial", (17, 23, 29), 1, 14),           # partial tiles (nx % 16 != 0: no full tile at all)
    ("slice", (1, 64, 64), 1, 14),              # a 2-D slice
]


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("name,shape,x_lo,x_hi", MAZES, ids=[m[0] for m in MAZES])
def test_maze(wp, name, shape, x_lo, x_hi, mode):
    rng = np.random.default_rng(len(name) + mode)
    for flat in (True, False):
        img, path = maze(shape, x_lo, x_hi, None if flat else rng)
        _check_path(path, shape)
        mk = np.zeros(shape, np.int16)
        mk.ravel()[path[0]] = 3
        mk.ravel()[path[-1]] = -7
        mk.ravel()[path[path.size // 3]] = 12
        _stats()
        got = _device(wp, img, mk, mode)
        s = _stats()
        print(f"{name} mode {mode} {'flat' if flat else 'noisy'}: path {path.size}, rounds {wp.LAST_ROUNDS}, "
              f"re-queued visits {s[3]}, phase-1 visits {s[0]}, phase-2 visits {s[4]}")
        _assert_checker(got, img, mk, mode, what=f"{name} mode {mode}")
        assert s[3] > 0, "no tile re-queued itself"
        assert s[7] == 0


# ---- the 24-bit hop limit of the 32-bit keys ----------------------------------------------------------
def _hop_maze(half_len_min):
    """nx = 16 (one tile column, walls at x = 0 and 15 so that mode 0's row wrap joins walls only),
    ny = 2048: the fewest even planes whose snake is at least 2 * half_len_min + 1 voxels long."""
    ny, per_plane = 2048, 1024 * 15
    planes = -(-(2 * half_len_min + 2) // per_plane)
    return (2 * planes - 1, ny, 16)


def _hop_case(length):
    """A corridor of `length` voxels (a prefix of the snake), markers 1 and 2 at its two ends."""
    shape = _hop_maze(length // 2)
    path = snake(shape, 1, 14)
    assert path.size >= length
    path = path[:length]
    img = np.full(shape, WALL, np.uint16)
    img.ravel()[path] = FLOOR
    mk = np.zeros(shape, np.int16)
    mk.ravel()[path[0]] = 1
    mk.ravel()[path[-1]] = 2
    return img, mk, path


def _hop_case_one_marker(far):
    """The whole snake as corridor, one marker placed so that the farther end is `far` hops away.
    One marker: no two fronts meet, so no key ever exceeds its final value on the corridor (where
    two fronts meet, the faster one overshoots the middle before the other arrives)."""
    shape = _hop_maze(far - 1024 * 15)
    path = snake(shape, 1, 14)
    at = path.size - 1 - far
    assert 0 <= at <= far
    img = np.full(shape, WALL, np.uint16)
    img.ravel()[path] = FLOOR
    mk = np.zeros(shape, np.int16)
    mk.ravel()[path[at]] = 1
    return img, mk, path


@pytest.mark.parametrize("mode", [0, 1])
def test_hop_limit_falls_back_to_64_bit_keys(wp, mode, monkeypatch):
    """Two corridors of more than 0xff0000 voxels each (the two halves of one corridor, a marker
    at each far end) meet in the middle: the labels there are decided by hop counts above 2^24."""
    from oracle import watershed as W
    length = 2 * (KEY_FULL_HOPS + 4096) + 1
    img, mk, path = _hop_case(length)
    want_lab, want_amb, hops = W.ws_labels(img, mk, SIX, mode, return_hops=True)
    k = np.arange(path.size)
    assert np.array_equal(hops.ravel()[path], np.minimum(k, path.size - 1 - k)), "the corridor has a shortcut"
    mid = path.size // 2
    assert hops.ravel()[path[mid]] > KEY_FULL_HOPS and (path.size - 1) // 2 > KEY_FULL_HOPS
    _stats()
    t0 = time.perf_counter()
    lab, amb = _device(wp, img, mk, mode)
    wall = time.perf_counter() - t0
    s = _stats()
    print(f"hop limit mode {mode}: shape {img.shape}, corridor {path.size} voxels, {hops.max()} hops at most, "
          f"rounds {wp.LAST_ROUNDS}, {wall:.2f} s, 32->64-bit fallbacks {s[7]}, re-queued visits {s[3]}")
    assert s[7] == 1, "expected exactly one fallback to 64-bit keys"
    assert np.array_equal(lab, want_lab) and np.array_equal(amb, want_amb)
    assert lab.ravel()[path[mid - 1]] == 1 and lab.ravel()[path[mid + 1]] == 2
    monkeypatch.setenv("B2V_WS_KEY64", "1")
    t0 = time.perf_counter()
    lab64, amb64 = _device(wp, img, mk, mode)
    wall64 = time.perf_counter() - t0
    s = _stats()
    print(f"  64-bit keys only: rounds {wp.LAST_ROUNDS}, {wall64:.2f} s, fallbacks {s[7]}")
    assert s[7] == 0
    assert np.array_equal(lab64, lab) and np.array_equal(amb64, amb)


def test_hop_limit_just_under(wp):
    """The same maze with its farthest voxel a few hops under 0xff0000: no fallback."""
    from oracle import watershed as W
    img, mk, path = _hop_case_one_marker(KEY_FULL_HOPS - 64)
    want_lab, want_amb, hops = W.ws_labels(img, mk, SIX, 0, return_hops=True)
    reached = hops[hops != 0xFFFFFFFF]
    assert reached.size == img.size and hops.ravel()[path[-1]] == KEY_FULL_HOPS - 64
    assert KEY_FULL_HOPS - 64 <= reached.max() < KEY_FULL_HOPS, reached.max()
    _stats()
    t0 = time.perf_counter()
    lab, amb = _device(wp, img, mk, 0)
    wall = time.perf_counter() - t0
    s = _stats()
    print(f"just under the hop limit: {reached.max()} hops at most, rounds {wp.LAST_ROUNDS}, {wall:.2f} s, "
          f"fallbacks {s[7]}")
    assert s[7] == 0
    assert np.array_equal(lab, want_lab) and np.array_equal(amb, want_amb)


# ---- alignment, full and partial tiles mixed ------------------------------------------------------------
def _noise_case(shape, seed, levels=300):
    rng = np.random.default_rng(seed)
    img = ndimage.gaussian_filter(rng.normal(size=shape), 1.2)
    img = ((img - img.min()) / (np.ptp(img) + 1e-9) * levels).astype(np.uint16)
    mk = np.zeros(shape, np.int16)
    for lab in (1, 2, -3, 2, 5):
        z, y, x = (int(rng.integers(0, s)) for s in shape)
        mk[z, max(0, y - 1): y + 2, max(0, x - 1): x + 2] = lab
    return img, mk


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("shape", [(33, 47, 64), (16, 16, 16), (1, 64, 64), (20, 16, 48)])
def test_unaligned_image_and_tile_mix(wp, shape, mode):
    """The same input from a 16-byte-aligned tensor and from a view 2 bytes off: the unaligned one
    takes the scalar tile loads (g.vec = 0) where nx % 16 == 0 would allow vectors."""
    import torch
    for seed, maze_too in ((sum(shape), False), (sum(shape) + 1, True)):
        img, mk = _noise_case(shape, seed)
        if maze_too and shape[0] > 1:
            m, path = maze(shape, 1, shape[2] - 2)
            img = np.where(m == WALL, img + 200, img).astype(np.uint16)
        n = img.size
        buf = torch.zeros(n + 8, dtype=torch.int16, device="cuda")
        aligned = buf[:n].view(shape)
        shifted = buf[1:n + 1].view(shape)
        assert aligned.data_ptr() % 16 == 0 and shifted.data_ptr() % 16 == 2
        res = []
        for view in (aligned, shifted):
            view.copy_(_t(img.view(np.int16)))
            res.append(_device(wp, img, mk, mode, img_t=view))
        assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1])
        _assert_checker(res[1], img, mk, mode, what=f"{shape} mode {mode}")


# ---- labels: int16 extremes, 256 / 257 distinct labels, every kernel family -----------------------------
def _many_labels(shape, nlab, seed):
    rng = np.random.default_rng(seed)
    img, _ = _noise_case(shape, seed, levels=120)
    extremes = np.array([-32768, -1, 1, 32767], np.int16)
    others = np.setdiff1d(np.arange(-32768, 32768), np.concatenate([extremes, [0]]))
    labs = np.concatenate([extremes, rng.choice(others, nlab - 4, replace=False)]).astype(np.int16)
    assert np.unique(labs).size == nlab
    mk = np.zeros(shape, np.int16)
    pos = rng.choice(img.size, nlab, replace=False)
    mk.ravel()[pos] = labs
    return img, mk


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("engine", ["persistent", "generic", "conn18", "conn26"])
@pytest.mark.parametrize("nlab", [4, 256, 257])
def test_labels(wp, nlab, engine, mode, monkeypatch):
    """Markers from {-32768, -1, 1, 32767} (nlab = 4), or exactly 256 / 257 distinct labels that
    include them (the largest set of the 32-bit ranked keys, and the first that needs 64 bits)."""
    st = {"persistent": SIX, "generic": SIX, "conn18": generate_binary_structure(3, 2),
          "conn26": generate_binary_structure(3, 3)}[engine]
    if engine == "generic":
        monkeypatch.setenv("B2V_WS_GENERIC", "1")
    for shape in ((24, 40, 64), (13, 21, 35)):
        img, mk = _many_labels(shape, nlab, seed=nlab + len(engine) + sum(shape))
        if nlab == 4:
            # a plateau region only -32768 reaches: none of it is ambiguous
            img[: shape[0] // 2] = 0
            mk[: shape[0] // 2] = 0
            mk[1, 1, 1] = -32768
        got = _device(wp, img, mk, mode, st)
        _assert_checker(got, img, mk, mode, st, what=f"{nlab} labels, {engine}, {shape}, mode {mode}")
        if nlab > 4:
            assert np.unique(got[0][mk == 0]).size > 50


def test_minus_32768_region_is_not_ambiguous(wp):
    """All voxels reached only by label -32768 are unambiguous, in both engines and both modes."""
    shape = (20, 32, 48)
    img = np.zeros(shape, np.uint16)
    img[:, :, 24:] = 500
    mk = np.zeros(shape, np.int16)
    mk[3, 4, 5] = -32768
    mk[10, 20, 40] = 32767
    for mode in (0, 1):
        for st in (SIX, generate_binary_structure(3, 3)):
            lab, amb = _device(wp, img, mk, mode, st)
            assert (lab[:, :, :24] == -32768).all()
            assert not amb[:, :, :24].any()
            _assert_checker((lab, amb), img, mk, mode, st, what=f"mode {mode}")


# ---- full size -------------------------------------------------------------------------------------------
def test_full_size_ct_phantom(wp):
    """192 x 512 x 512 CT phantom, Cranium window, 6-connected, both algorithms: every voxel,
    ambiguous ones included, equals the checker on the same pre-processed image."""
    from invesalius3_b200 import phantom
    from oracle import watershed as W
    shape = (192, 512, 512)
    vol = phantom.ct(shape, seed=4)
    rng = np.random.default_rng(4)
    markers = np.zeros(shape, np.int16)
    inside, outside = np.argwhere(vol > 600), np.argwhere(vol < -900)
    for _ in range(4):
        z, y, x = inside[rng.integers(len(inside))]; markers[z, y, x] = 1
        z, y, x = outside[rng.integers(len(outside))]; markers[z, y, x] = 2
    pre = W.preprocess(vol, True, -18, 406)
    t_vol, t_mk = _t(vol), _t(markers)
    for algorithm, mode in (("Watershed", 1), ("Watershed IFT", 0)):
        cost = ndimage.morphological_gradient(pre, 3) if mode == 1 else pre
        lab, amb = wp.watershed_device(t_vol, t_mk, SIX, algorithm, 3, True, -18, 406, return_ambiguous=True)
        _assert_checker((lab.cpu().numpy(), amb.cpu().numpy()), cost, markers, mode, what=algorithm)
        print(f"{algorithm} {shape}: rounds {wp.LAST_ROUNDS}, ambiguous {float(amb.float().mean()):.4f}")
