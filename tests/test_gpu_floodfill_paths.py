"""Flood-fill paths that the parity tests of test_gpu_floodfill.py do not reach: the tuning knob
B2V_FF_GRID (each setting in a process of its own), more than 1024 tiles, floods of thousands of
rounds and the round cap, and int16 and uint8 data and thresholds at their limits through every
build of the bit volumes.

Every device result is compared bit for bit with the serial C checker; where the element is
symmetric and the volume large, also with the seeded components of the passable set that
scipy.ndimage.label finds."""
import ctypes as C
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
from scipy import ndimage
from scipy.ndimage import generate_binary_structure

import bitpack_model
import ff_knob_child as knob

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
_MEMO = {}


def _memo(key, fn):
    if key not in _MEMO:
        _MEMO[key] = fn()
    return _MEMO[key]


@pytest.fixture(scope="module")
def rs():
    from invesalius3_b200 import device, invesalius_rs
    device.require_cuda()
    return invesalius_rs


@pytest.fixture(params=["persistent", "host-rounds"])
def engine(request):
    """The convergence engine: one cooperative launch, or a launch per round."""
    from invesalius3_b200 import _lib
    lib = _lib.load()
    lib.b2v_floodfill_set_engine(1 if request.param == "persistent" else 0)
    yield request.param
    lib.b2v_floodfill_set_engine(1)


def _checker(orc, data, seeds, t0, t1, fill, st, out0):
    want = out0.copy()
    orc.floodfill_threshold(data, seeds, t0, t1, fill, st, want)
    return want


def _label_answer(data, seeds, t0, t1, fill, st, out0):
    """The union of the components of the passable set (in range, out != fill, plus the valid seeds)
    that hold a valid seed, written with `fill` into out0. For symmetric elements only."""
    inr = (data >= t0) & (data <= t1)
    passable = inr & (out0 != fill)
    valid = [(x, y, z) for x, y, z in seeds if inr[z, y, x]]
    for x, y, z in valid:
        passable[z, y, x] = True
    lab, _ = ndimage.label(passable, structure=st)
    ids = sorted({int(lab[z, y, x]) for x, y, z in valid})
    res = out0.copy()
    res[np.isin(lab, ids)] = fill
    return res


def _layout_tiles(shape):
    from invesalius3_b200 import _lib
    lay = (C.c_int64 * 8)()
    _lib.call("b2v_floodfill_layout", *shape, 1, lay)
    return int(lay[4])


# ---------------------------------------------------------------------------------- A. tuning knobs
@pytest.mark.parametrize("setting", list(knob.SETTINGS))
def test_floodfill_knob_setting(orc, tmp_path, setting):
    """One process per knob setting (the knob is read once per process): every case of the
    setting on both engines against the checker, and proof that the setting took effect: the
    fallback signature (the host-driven rounds ran: the persistent kernel's round counter stayed 0,
    the returned count did not)."""
    knobs, shapes = knob.SETTINGS[setting]
    env = {k: v for k, v in os.environ.items() if not k.startswith("B2V_FF_")}
    env.update(knobs)
    env["PYTHONPATH"] = os.pathsep.join([str(ROOT), *filter(None, [os.environ.get("PYTHONPATH")])])
    cmd = [sys.executable, *(["-s"] if sys.flags.no_user_site else []), str(ROOT / "tests" / "ff_knob_child.py"),
           setting, str(tmp_path)]
    r = subprocess.run(cmd, env=env, timeout=900, capture_output=True, text=True)
    assert r.returncode == 0, f"child failed ({r.returncode}):\n{r.stdout[-4000:]}\n{r.stderr[-8000:]}"
    res = json.loads((tmp_path / "results.json").read_text())
    grid = int(knobs["B2V_FF_GRID"])
    for cname, sname, ename in knob.cases(setting):
        shape = shapes[sname]
        tiles = knob.tile_count(shape)
        assert _layout_tiles(shape) == tiles, shape    # the restatement is right
        (tz, ty, tw), _ = knob.tile_shape(shape)
        assert ((tw, ty, tz) == (16, 16, 16)) == (sname == "canon"), (shape, tz, ty, tw)
        fallback = grid * knob.MAX_MINE < tiles
        assert fallback == (sname == "fallback"), (setting, sname, tiles)
        c = knob.case_inputs(setting, sname, ename)
        args = (c["data"], c["seeds"], c["t0"], c["t1"], c["fill"], c["strct"], c["out0"])
        want = _checker(orc, *args)
        assert ((want == c["fill"]) & (c["out0"] != c["fill"])).sum() > 5000, cname
        if ename in knob.SYMMETRIC:
            assert np.array_equal(_label_answer(*args), want), cname
        for engine in knob.ENGINES:
            key = f"{cname}__{engine}"
            got = np.load(tmp_path / f"{key}.npy")
            assert np.array_equal(got, want), (key, int((got != want).sum()))
            rec = res[key]
            assert rec["tiles"] == tiles, (key, rec)
            assert rec["rounds"] > 0, (key, rec)
            if engine == "persistent" and not fallback:
                assert rec["stats_rounds"] == rec["rounds"], (key, rec)
            else:       # host-driven rounds: the persistent kernel never ran
                assert rec["stats_rounds"] == 0, (key, rec)


# ------------------------------------------------------------------------------ B. > 1024 tiles
@pytest.fixture(scope="module")
def ct544():
    """A 544-slice CT: 34 x 32 x 1 = 1088 tiles, so the tile bitmap has 34 words and the tiles are
    ranked by the block-wide scan. The phantom's head ends near slice 490; rolled by half its height,
    the head reaches the top and tiles past index 1024 take part in the flood."""
    from invesalius3_b200 import phantom
    vol = np.roll(phantom.ct((544, 512, 512), seed=2), 272, axis=0)
    seeds = [phantom.first_seed_in_range(vol, 100, 226, 3071), phantom.first_seed_in_range(vol, 530, 226, 3071)]
    return vol, seeds


@pytest.mark.parametrize("conn", [1, 3])
def test_floodfill_more_than_1024_tiles(orc, ct544, engine, conn):
    import torch
    from invesalius3_b200 import device as dev
    vol, seeds = ct544
    st = generate_binary_structure(3, conn)
    out0 = np.zeros(vol.shape, np.uint8)

    def reference():
        want = _checker(orc, vol, seeds, 226, 3071, 254, st, out0)
        assert np.array_equal(_label_answer(vol, seeds, 226, 3071, 254, st, out0), want)
        return want

    want = _memo(("ct544", conn), reference)
    assert (want[512:] == 254).sum() > 100000      # tiles 1024.. are flooded
    out = torch.zeros(vol.shape, dtype=torch.uint8, device="cuda")
    stats = {}
    rounds = dev.floodfill_threshold(torch.from_numpy(vol).cuda(), seeds, 226, 3071, 254, st, out, stats=stats)
    assert stats["tiles"] == 1088 and rounds > 0
    got = out.cpu().numpy()
    assert np.array_equal(got, want), int((got != want).sum())


# --------------------------------------------------------------------------- C. long mazes, round cap
def serpentine(dz, dy, dx):
    """Corridor mask of a 3-D serpentine. Corridors along x, one voxel wide, on even rows of even
    planes; the rows of a plane are joined at alternating ends in y (x = dx - 1, 0, dx - 1, ...), and
    the planes at alternating ends in z (the end of a plane's path, then its start). Every other
    voxel is wall. The corridors form one path from (x, y, z) = (0, 0, 0), so the flood from there
    reaches exactly the corridors, one row per turn."""
    m = np.zeros((dz, dy, dx), bool)
    m[0::2, 0::2, :] = True
    rows, planes = (dy + 1) // 2, (dz + 1) // 2
    for k in range(rows - 1):
        m[0::2, 2 * k + 1, dx - 1 if k % 2 == 0 else 0] = True
    yend, xend = 2 * (rows - 1), (dx - 1 if (rows - 1) % 2 == 0 else 0)
    for j in range(planes - 1):
        m[2 * j + 1, yend if j % 2 == 0 else 0, xend if j % 2 == 0 else 0] = True
    assert m.sum() == planes * rows * dx + planes * (rows - 1) + planes - 1
    return m


@pytest.mark.parametrize("conn", [1, 3])
def test_floodfill_serpentine_maze(rs, orc, engine, conn):
    """1024 turns (32 planes x 32 rows of 600 voxels): a visit runs one sweep set, so every turn
    costs at least one round. Measured on an H100 80GB HBM3 at a 700 W power limit: 2148 rounds on
    the persistent engine and 2172 on the host-driven one (which counts whole batches), for 6- and
    26-connectivity alike: a row of 19 words spans two tiles, and the hand-over costs a round."""
    import torch
    from invesalius3_b200 import device as dev
    maze = serpentine(64, 64, 600)
    data = maze.astype(np.int16) * 1000
    st = generate_binary_structure(3, conn)
    out0 = np.zeros(maze.shape, np.uint8)
    want = _checker(orc, data, [(0, 0, 0)], 500, 1500, 1, st, out0)
    assert np.array_equal(want == 1, maze)
    out = torch.zeros(maze.shape, dtype=torch.uint8, device="cuda")
    rounds = dev.floodfill_threshold(torch.from_numpy(data).cuda(), [(0, 0, 0)], 500, 1500, 1, st, out)
    assert np.array_equal(out.cpu().numpy(), want)
    print(f"serpentine 64x64x600, {conn=}, {engine}: {rounds} rounds")
    assert rounds >= 1024, rounds
    got = out0.copy()
    rs.floodfill_threshold(data, [(0, 0, 0)], 500, 1500, 1, st, got)
    assert np.array_equal(got, want)


def test_floodfill_maze_beyond_round_cap(rs, orc, engine):
    """67 584 turns (264 planes x 256 rows of 64 voxels) are more rounds than the cap of 65 536
    (kMaxRounds): the flood stops with a clean error (B2V_ERR_NOCONV, raised as B2VError) on both
    engines, although the serial checker fills the maze. The numpy API leaves `out` unchanged.
    The device API leaves `out` unchanged on the host-driven engine, which fails before the
    write-back; the persistent engine queues the write-back behind its kernel before it reads the
    verdict, so `out` then holds the part of the path reached within the cap."""
    import torch
    from invesalius3_b200 import device as dev
    from invesalius3_b200._lib import B2VError
    maze = _memo("maze-cap", lambda: serpentine(528, 512, 64))
    data = maze.astype(np.int16) * 1000
    st = generate_binary_structure(3, 1)
    seeds = [(0, 0, 0)]
    assert _memo("maze-cap-checker", lambda: np.array_equal(
        _checker(orc, data, seeds, 500, 1500, 1, st, np.zeros(maze.shape, np.uint8)) == 1, maze))
    out = np.zeros(maze.shape, np.uint8)
    with pytest.raises(B2VError, match="no convergence"):
        rs.floodfill_threshold(data, seeds, 500, 1500, 1, st, out)
    assert not out.any()
    o = torch.zeros(maze.shape, dtype=torch.uint8, device="cuda")
    with pytest.raises(B2VError, match="no convergence"):
        dev.floodfill_threshold(torch.from_numpy(data).cuda(), seeds, 500, 1500, 1, st, o)
    got = o.cpu().numpy()
    if engine == "persistent":
        reached = got == 1
        assert np.array_equal(got.astype(bool), reached) and not (reached & ~maze).any()
        assert maze.sum() // 2 < reached.sum() < maze.sum(), int(reached.sum())
    else:
        assert not got.any()


# ----------------------------------------------------------------- D. int16 limits, build matrix
FILL = 1
THRESHOLDS = [(-32768, -32768), (32767, 32767), (-32768, 32767), (-32767, 32766), (0, 0), (5, 4),
              (-40000, -32768), (32767, 40000), (-0.5, 0.5)]
# name -> (dx, data offset in elements, out offset in bytes). 512: the vectorised build with
# dx % 32 == 0; 200: vectorised, padded rows; the rest take the ballot build (bitpack_model).
LAYOUTS = {"dx512": (512, 0, 0), "dx200": (200, 0, 0), "dx203": (203, 0, 0), "data+1": (512, 1, 0),
           **{f"out+{k}": (512, 0, k) for k in range(1, 8)}}
LIMIT_ELEMENTS = [generate_binary_structure(3, 1), generate_binary_structure(3, 3), generate_binary_structure(3, 2)]


def _limits_volume(dx):
    """(15, 63, dx) int16: smooth noise saturated at both limits over a fifth of the volume, a plateau
    at 0, and the first 65 536 voxels (raveled) holding every int16 value in order; out with walls
    (`FILL`), markers and other values."""
    def make():
        shape = (15, 63, dx)
        rng = np.random.default_rng(dx)
        f = ndimage.gaussian_filter(rng.normal(size=shape), 3.0)
        f /= np.quantile(np.abs(f), 0.8)
        v = np.clip(np.rint(f * 32767.0), -32768, 32767)
        v[np.abs(v) < 8000] = 0
        v = v.astype(np.int16)
        v.reshape(-1)[:65536] = np.arange(-32768, 32768)
        out0 = np.zeros(shape, np.uint8)
        for val, p in ((FILL, 0.02), (2, 0.01), (200, 0.01), (253, 0.01), (254, 0.01)):
            out0[rng.random(shape) < p] = val
        return v, out0
    return _memo(("limits", dx), make)


def _placed(a, offset):
    """A dense device copy of `a` that starts `offset` elements into its allocation."""
    import torch
    from invesalius3_b200 import device as dev
    t = dev.to_device(np.ascontiguousarray(a))
    buf = torch.zeros(a.size + offset + 64, dtype=t.dtype, device="cuda")
    v = buf[offset:offset + a.size].view(a.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == offset * a.itemsize % 16
    return v


def _seeds_in(data, lo, hi, rng):
    inr = (data >= lo) & (data <= hi)
    idx = np.flatnonzero(inr)
    pick = list(rng.choice(idx, min(6, idx.size), replace=False)) + ([idx[0], idx[-1]] if idx.size else [])
    out = np.flatnonzero(~inr)
    pick += [out[out.size // 2]] if out.size else []
    return [(int(x), int(y), int(z)) for z, y, x in (np.unravel_index(i, data.shape) for i in pick)]


def _nonempty(data, lo, hi):
    return bool(((data >= lo) & (data <= hi)).any())


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_floodfill_threshold_int16_limits(rs, orc, engine, layout):
    from invesalius3_b200 import device as dev
    dx, doff, ooff = LAYOUTS[layout]
    data, out0 = _limits_volume(dx)
    d = _placed(data, doff)
    for i, (t0, t1) in enumerate(THRESHOLDS):
        st = LIMIT_ELEMENTS[i % 3]
        seeds = _seeds_in(data, t0, t1, np.random.default_rng(i))

        def reference():   # the checker on float64 data: any bound, exactly
            want = out0.copy()
            orc._floodfill_threshold_core(data.astype(np.float64), seeds, float(t0), float(t1), FILL,
                                          np.ascontiguousarray(st, np.uint8), want)
            return want
        want = _memo(("thr", dx, i), reference)
        if _nonempty(data, t0, t1):
            assert ((want == FILL) & (out0 != FILL)).sum() > 1000, (t0, t1)
        else:
            assert np.array_equal(want, out0)
        o = _placed(out0, ooff)
        dev.floodfill_threshold(d, seeds, t0, t1, FILL, st, o)
        got = o.cpu().numpy()
        assert np.array_equal(got, want), (layout, t0, t1, int((got != want).sum()))
        if doff or ooff:
            continue
        got = out0.copy()
        if all(float(t).is_integer() and -32768 <= t <= 32767 for t in (t0, t1)):
            rs.floodfill_threshold(data, seeds, t0, t1, FILL, st, got)
            assert np.array_equal(got, want), (layout, t0, t1)
        elif isinstance(t0, int):   # PyO3 rejects bounds outside int16
            with pytest.raises(OverflowError):
                rs.floodfill_threshold(data, seeds, t0, t1, FILL, st, got)


# fill of the in-place flood per threshold of THRESHOLDS (the limits themselves included)
INPLACE_FILLS = [1, -1, 32767, -32768, 32767, 0, 32767, -32768, 5]


@pytest.mark.parametrize("layout", ["dx512", "dx200", "dx203", "data+1"])
def test_floodfill_inplace_int16_limits(orc, engine, layout):
    from invesalius3_b200 import device as dev
    dx, doff, _ = LAYOUTS[layout]
    data, _ = _limits_volume(dx)
    for i, (t0, t1) in enumerate(THRESHOLDS):
        st, fill = LIMIT_ELEMENTS[i % 3], INPLACE_FILLS[i]
        seeds = _seeds_in(data, t0, t1, np.random.default_rng(100 + i))

        def reference():
            a = data.astype(np.float64)
            orc.floodfill_threshold_inplace(a, seeds, float(t0), float(t1), float(fill), st)
            return a.astype(np.int16)
        want = _memo(("inplace", dx, i), reference)
        if _nonempty(data, t0, t1):
            assert (want != data).sum() > 1000, (t0, t1, fill)
        d = _placed(data, doff)
        dev.floodfill_threshold_inplace(d, seeds, t0, t1, fill, st)
        got = d.cpu().numpy()
        assert np.array_equal(got, want), (layout, t0, t1, fill, int((got != want).sum()))


# equality flood values: both limits, 0, a non-integer and one outside int16 (these two match
# nothing; the seed is still marked)
EQUAL_VALUES = [-32768, 32767, 0, 0.5, 40000]


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_floodfill_equal_int16_limits(rs, orc, engine, layout):
    from invesalius3_b200 import device as dev
    dx, doff, ooff = LAYOUTS[layout]
    data, out0 = _limits_volume(dx)
    d = _placed(data, doff)
    for v in EQUAL_VALUES:
        # seed in the largest 6-connected region of data == v (any voxel if there is none)
        lab, n = ndimage.label((data == v) & (out0 != FILL))
        if n:
            idx = np.flatnonzero(lab == 1 + np.argmax(np.bincount(lab.ravel())[1:]))
            i = idx[idx.size // 2]
        else:
            idx, i = np.array([]), data.size // 3
        z, y, x = (int(c) for c in np.unravel_index(i, data.shape))

        def reference():
            want = out0.copy()
            orc.floodfill(data.astype(np.float64), x, y, z, float(v), FILL, want)
            return want
        want = _memo(("eq", dx, v), reference)
        if idx.size:
            assert ((want == FILL) & (out0 != FILL)).sum() > 500, v
        else:
            expect = out0.copy()
            expect[z, y, x] = FILL
            assert np.array_equal(want, expect)
        o = _placed(out0, ooff)
        dev.floodfill(d, x, y, z, v, FILL, o)
        got = o.cpu().numpy()
        assert np.array_equal(got, want), (layout, v, int((got != want).sum()))
        if doff or ooff:
            continue
        got = out0.copy()
        if isinstance(v, float):
            with pytest.raises(TypeError):
                rs.floodfill(data, x, y, z, v, FILL, got)
        elif not -32768 <= v <= 32767:
            with pytest.raises(OverflowError):
                rs.floodfill(data, x, y, z, v, FILL, got)
        else:
            rs.floodfill(data, x, y, z, v, FILL, got)
            assert np.array_equal(got, want), (layout, v)


@pytest.mark.parametrize("layout", ["dx512", "dx200", "dx203", "data+1", "out+3"])
def test_threshold_int16_limits(orc, layout):
    """device.threshold on the same data and bounds: the vectorised kernel with a scalar tail
    (dx 200, 203) and the scalar kernel on unaligned buffers, with and without kept markers."""
    from invesalius3_b200 import device as dev
    dx, doff, ooff = LAYOUTS[layout]
    data, out0 = _limits_volume(dx)
    d = _placed(data, doff)
    for lo, hi in THRESHOLDS:
        for keep in (False, True):
            want = out0.copy()
            orc.threshold(data, lo, hi, want, keep)
            o = _placed(out0, ooff)
            dev.threshold(d, lo, hi, o, keep)
            got = o.cpu().numpy()
            assert np.array_equal(got, want), (layout, lo, hi, keep, int((got != want).sum()))


# ----------------------------------------------------------------- E. uint8 limits, build matrix
U8_THRESHOLDS = [(0, 0), (255, 255), (0, 255), (127, 128), (128, 255), (0, 127), (1, 254), (128, 127), (-40, 0),
                 (255, 400), (-40, -1), (256, 400), (-0.5, 0.5), (127.2, 127.8)]
# as LAYOUTS for uint8 data: 512 and 208 (a multiple of 16 with padded rows) take the vectorised build, the widths
# 200 and 203, the misaligned data and every misaligned out (16-byte loads) the ballot build
U8_LAYOUTS = {"dx512": (512, 0, 0), "dx208": (208, 0, 0), "dx200": (200, 0, 0), "dx203": (203, 0, 0),
              "data+1": (512, 1, 0), **{f"out+{k}": (512, 0, k) for k in range(1, 16)}}
# equality flood values: both limits, the two plateaus, a non-integer and two outside uint8 (these three match
# nothing; the seed is still marked)
U8_EQUAL_VALUES = [0, 255, 127, 128, 0.5, 300, -1]


def test_layouts_reach_every_packing_kernel():
    """The flood's build matrices reach every packing kernel, and each vectorised one again with a
    misaligned data or out pointer (the ballot at that width)."""
    cases = [(np.int16, dx, 2 * doff, ooff) for dx, doff, ooff in LAYOUTS.values()]
    cases += [(np.uint8, dx, doff, ooff) for dx, doff, ooff in U8_LAYOUTS.values()]
    assert {bitpack_model.pack_kernel(*c) for c in cases} == set(bitpack_model.VEC + bitpack_model.BALLOT)
    misaligned = {bitpack_model.pack_kernel(dt, dx) for dt, dx, doff, ooff in cases
                  if bitpack_model.pack_kernel(dt, dx, doff, ooff).startswith("ballot<")}
    assert misaligned >= {"vec<int16,linear>", "vec<uint8,linear>"}
    assert {ooff for dt, dx, doff, ooff in cases if dt == np.uint8} >= set(range(16))


def _limits_volume_u8(dx):
    """(15, 63, dx) uint8: smooth noise saturated at 0 and 255 over a fifth of the volume, plateaus at 127
    and 128, and the first 512 voxels (raveled) holding every value twice in order; out as in
    _limits_volume."""
    def make():
        shape = (15, 63, dx)
        rng = np.random.default_rng(1000 + dx)
        f = ndimage.gaussian_filter(rng.normal(size=shape), 3.0)
        f /= np.quantile(np.abs(f), 0.8)
        v = np.clip(np.rint(127.5 + f * 127.5), 0, 255)
        v[np.abs(v - 127.5) < 30] = np.where(v[np.abs(v - 127.5) < 30] < 127.5, 127, 128)
        v = v.astype(np.uint8)
        v.reshape(-1)[:512] = np.tile(np.arange(256), 2)
        out0 = np.zeros(shape, np.uint8)
        for val, p in ((FILL, 0.02), (2, 0.01), (200, 0.01), (253, 0.01), (254, 0.01)):
            out0[rng.random(shape) < p] = val
        return v, out0
    return _memo(("limits-u8", dx), make)


@pytest.mark.parametrize("layout", list(U8_LAYOUTS))
def test_floodfill_threshold_uint8_limits(orc, engine, layout):
    from invesalius3_b200 import device as dev
    dx, doff, ooff = U8_LAYOUTS[layout]
    data, out0 = _limits_volume_u8(dx)
    d = _placed(data, doff)
    for i, (t0, t1) in enumerate(U8_THRESHOLDS):
        st = LIMIT_ELEMENTS[i % 3]
        seeds = _seeds_in(data, t0, t1, np.random.default_rng(i))

        def reference():   # the checker on float64 data: any bound, exactly
            want = out0.copy()
            orc._floodfill_threshold_core(data.astype(np.float64), seeds, float(t0), float(t1), FILL,
                                          np.ascontiguousarray(st, np.uint8), want)
            return want
        want = _memo(("thr-u8", dx, i), reference)
        if _nonempty(data, t0, t1):
            assert ((want == FILL) & (out0 != FILL)).sum() > 1000, (t0, t1)
        else:
            assert np.array_equal(want, out0)
        o = _placed(out0, ooff)
        dev.floodfill_threshold(d, seeds, t0, t1, FILL, st, o)
        got = o.cpu().numpy()
        assert np.array_equal(got, want), (layout, t0, t1, int((got != want).sum()))


@pytest.mark.parametrize("layout", list(U8_LAYOUTS))
def test_floodfill_equal_uint8_limits(orc, engine, layout):
    from invesalius3_b200 import device as dev
    dx, doff, ooff = U8_LAYOUTS[layout]
    data, out0 = _limits_volume_u8(dx)
    d = _placed(data, doff)
    for v in U8_EQUAL_VALUES:
        # seed in the largest 6-connected region of data == v (any voxel if there is none)
        lab, n = ndimage.label((data == v) & (out0 != FILL))
        if n:
            idx = np.flatnonzero(lab == 1 + np.argmax(np.bincount(lab.ravel())[1:]))
            i = idx[idx.size // 2]
        else:
            idx, i = np.array([]), data.size // 3
        z, y, x = (int(c) for c in np.unravel_index(i, data.shape))

        def reference():
            want = out0.copy()
            orc.floodfill(data.astype(np.float64), x, y, z, float(v), FILL, want)
            return want
        want = _memo(("eq-u8", dx, v), reference)
        if idx.size:
            assert ((want == FILL) & (out0 != FILL)).sum() > 500, v
        else:
            expect = out0.copy()
            expect[z, y, x] = FILL
            assert np.array_equal(want, expect)
        o = _placed(out0, ooff)
        dev.floodfill(d, x, y, z, v, FILL, o)
        got = o.cpu().numpy()
        assert np.array_equal(got, want), (layout, v, int((got != want).sum()))
