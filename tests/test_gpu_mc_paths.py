"""Marching-cubes paths that the parity tests of test_gpu_mc.py do not reach: every kernel that
loads the inside bits, with and without the 128-bit classify / emit (VEC), rows that straddle the
1024-word tiles, both shift splits of a word index, the iso -> integer threshold over the whole
range of both dtypes (including the byte-wise uint8 compare for thresholds >= 128), misaligned
device pointers, and the Z-shard entry points driven in one process.

Every device mesh is compared with the sequential C checker (oracle.marching_cubes): triangles
with np.array_equal, vertices bit for bit as uint32.

`variant` restates the dispatch of csrc/mc.cu and bitpack_model the packing kernel's;
test_case_lists_cover_every_variant (no GPU) checks that the case lists below reach every combination
they can produce."""
import math
import zlib

import numpy as np
import pytest
from scipy import ndimage

import bitpack_model

U8, I16 = np.dtype(np.uint8), np.dtype(np.int16)
DTYPES = {"uint8": U8, "int16": I16}
TILE_WORDS = 1024   # words per classify / emit tile (mc.cu:52-54)
VEC_BITS = bitpack_model.VEC
ALL_BITS = VEC_BITS + bitpack_model.BALLOT

SP = (0.5, 0.75, 1.25)     # (sx, sy, sz)
ORIGIN = (-1, 2, 3)        # (ox, oy, oz)


def variant(dtype, shape, byte_offset=0):
    """The kernels b2v_mc_count / b2v_mc_emit run for a [nz][ny][nx] volume whose device pointer
    lies byte_offset bytes past a 16-byte boundary (csrc/mc.cu)."""
    nz, ny, nx = shape
    bits = bitpack_model.pack_kernel(dtype, nx, byte_offset)   # mc_count_impl -> pack_bits
    wx = -(-nx // 32)                                     # make_geom, mc.cu:34
    ntiles = -(-(nz * ny * wx) // TILE_WORDS)             # mc.cu:670 and mc.cu:704
    pow2 = lambda v: v & (v - 1) == 0                     # make_geom's lg, mc.cu:37-39
    return dict(bits=bits,
                vec=wx % 4 == 0,                          # k_mc_classify / k_mc_emit_tris<VEC>, mc.cu:671, 717
                wx_sh=pow2(wx), ny_sh=pow2(ny),           # split_word, mc.cu:44-50
                wx=wx, ntiles=ntiles,
                straddle=any(TILE_WORDS * k % wx for k in range(1, ntiles)))


# ------------------------------------------------------------------------------------ case lists
GEOM_SHAPES = [
    (6, 40, 384),    # u8 linear / i16 vec, VEC (wx 12), 3 tiles with their boundaries inside rows
    (40, 16, 256),   # VEC with both shifts (wx 8, ny 16), 5 tiles
    (3, 17, 400),    # u8_vec<false> / i16 vec, rows (wx 13)
    (1, 24, 112),    # nz = 1; u8_vec<false> with VEC (wx 4)
    (2, 9, 128),     # nz = 2; u8 linear, VEC (wx 4)
    (5, 1, 96),      # ny = 1; u8 linear, rows (wx 3)
    (3, 6, 160),     # u8 linear, rows (wx 5)
    (7, 13, 24),     # u8 scalar / i16 vec, one word per row (wx_sh = 0)
    (1, 1, 1000),    # u8 scalar / i16 vec, VEC (wx 32) with both shifts
    (9, 20, 250),    # scalar for both dtypes, VEC (wx 8), 2 tiles
    (4, 7, 33),      # scalar for both dtypes, rows (wx 2)
]
CONTENTS = ["binary", "full", "smooth", "checker", "six_faces", "all_in", "all_out", "voxels"]

U8_ISOS = [-1e9, -1, 0, 0.5, 1, 126.5, 127, 127.000001, 128, 128.5, 200, 254.5, 255, 255.5, 256, math.inf, -math.inf]
I16_ISOS = [-40000, -32768.5, -32768, -32767.5, -1.5, -1, -0.5, -0.0, 0, 0.5, 226, 32766.5, 32767, 32767.5, 40000,
            math.inf, -math.inf]
SWEEP_SHAPES = {"uint8": [(4, 10, 384), (3, 11, 48), (4, 9, 37)], "int16": [(4, 10, 384), (4, 9, 37)]}

# device views at every misalignment, at widths that would otherwise take the vector loads
MISALIGNED = [("uint8", (5, 9, 128), k) for k in range(1, 16)] + \
             [("uint8", (4, 7, 48), k) for k in range(1, 16)] + \
             [("int16", (4, 6, 384), k) for k in range(2, 16, 2)] + \
             [("int16", (3, 7, 24), k) for k in range(2, 16, 2)]

# z-slabs t[z0:z1] of a resident volume; a slab starts z0 * ny * nx * itemsize bytes in
SLAB_VOLUMES = [("uint8", (20, 9, 48)), ("uint8", (20, 9, 37)), ("int16", (20, 9, 100)), ("int16", (20, 5, 27))]
SLABS = [(0, 1), (0, 2), (1, 2), (3, 8), (5, 6), (7, 20), (19, 20), (0, 20)]

# Z shards: shard i owns planes [bounds[i], bounds[i+1]) and is handed one more plane unless it is
# the last. `full` is a plane set entirely inside, `quiet` a shard given no surface at all, and
# `place` how the slabs are put on the device: their own buffers ("copy"), views of one resident
# volume ("view"), or at a byte offset past a 16-byte boundary (an int).
SHARDS = [
    dict(dtype="uint8", shape=(12, 20, 128), bounds=(0, 6, 12), full=6, quiet=None, place="copy"),
    dict(dtype="int16", shape=(13, 18, 384), bounds=(0, 1, 5, 13), full=5, quiet=0, place="copy"),
    dict(dtype="uint8", shape=(16, 17, 96), bounds=(0, 3, 4, 9, 15, 16), full=9, quiet=1, place="view"),
    dict(dtype="int16", shape=(14, 11, 100), bounds=(0, 5, 6, 7, 10, 14), full=10, quiet=2, place="view"),
    dict(dtype="uint8", shape=(12, 13, 384), bounds=(0, 4, 5, 12), full=4, quiet=None, place=5),
    dict(dtype="int16", shape=(10, 12, 128), bounds=(0, 1, 2, 10), full=2, quiet=None, place=6),
]


def _ext_bounds(bounds):
    n = len(bounds) - 1
    return [(bounds[i], bounds[i + 1] + (1 if i < n - 1 else 0)) for i in range(n)]


def _shard_offset(case, z0):
    itemsize = DTYPES[case["dtype"]].itemsize
    place = case["place"]
    if place == "view":
        return z0 * case["shape"][1] * case["shape"][2] * itemsize
    return 0 if place == "copy" else place


def _all_cases():
    """(dtype, shape, byte_offset) of every volume handed to the device below."""
    out = [(DTYPES[d], s, 0) for s in GEOM_SHAPES for d in DTYPES]
    out += [(DTYPES[d], s, 0) for d, shapes in SWEEP_SHAPES.items() for s in shapes]
    out += [(DTYPES[d], s, k) for d, s, k in MISALIGNED]
    for d, (nz, ny, nx) in SLAB_VOLUMES:
        out += [(DTYPES[d], (z1 - z0, ny, nx), z0 * ny * nx * DTYPES[d].itemsize) for z0, z1 in SLABS]
    for c in SHARDS:
        _, ny, nx = c["shape"]
        out += [(DTYPES[c["dtype"]], (z1 - z0, ny, nx), _shard_offset(c, z0)) for z0, z1 in _ext_bounds(c["bounds"])]
    return out


def test_case_lists_cover_every_variant():
    cases = [(d, s, k, variant(d, s, k)) for d, s, k in _all_cases()]
    seen = {(v["bits"], v["vec"]) for _, _, _, v in cases}
    # every bits kernel with both classify / emit forms (each combination can occur)
    missing = {(b, vec) for b in ALL_BITS for vec in (True, False)} - seen
    assert not missing, missing
    # VEC where a tile boundary falls inside a row
    assert any(v["vec"] and v["straddle"] for *_, v in cases)
    # both shift splits at once, on real rows and planes, over several tiles
    assert any(v["vec"] and v["wx_sh"] and v["ny_sh"] and v["wx"] > 1 and s[1] > 1 and v["ntiles"] > 1
               for _, s, _, v in cases)
    # division for both (the split the common shapes never take), and shifts with division
    assert any(not v["wx_sh"] and not v["ny_sh"] for *_, v in cases)
    assert any(v["wx_sh"] != v["ny_sh"] for *_, v in cases)
    # every vector bits kernel again with a misaligned pointer: the ballot at that width
    for b in VEC_BITS:
        assert any(k % 16 and variant(d, s, 0)["bits"] == b and v["bits"].startswith("ballot<")
                   for d, s, k, v in cases), b
    # the geometry matrix holds the degenerate extents and more than one tile
    assert any(s[0] == 1 for s in GEOM_SHAPES) and any(s[0] == 2 for s in GEOM_SHAPES)
    assert any(s[1] == 1 for s in GEOM_SHAPES)
    assert any(variant(U8, s)["ntiles"] > 1 for s in GEOM_SHAPES)
    # the Z shards: 2, 3 and 5 shards, single-plane shards, VEC and row widths, both dtypes, misalignment
    assert {len(c["bounds"]) - 1 for c in SHARDS} >= {2, 3, 5}
    assert any(b - a == 1 for c in SHARDS for a, b in zip(c["bounds"], c["bounds"][1:]))
    assert {c["shape"][2] for c in SHARDS} >= {128, 384, 96, 100}
    assert {c["dtype"] for c in SHARDS} == set(DTYPES)
    assert any(_shard_offset(c, z0) % 16 for c in SHARDS for z0, _ in _ext_bounds(c["bounds"]))
    assert any(c["quiet"] is not None for c in SHARDS) and all(c["full"] in c["bounds"] for c in SHARDS)


# ------------------------------------------------------------------------------------ helpers
def _sid(shape):
    return "x".join(map(str, shape))


def _seed(*key):
    return zlib.crc32(repr(key).encode())


ISO = {U8: 127.0, I16: 226.0}


def content(kind, dt, shape, seed):
    """A test volume of dtype dt: `kind` is one of CONTENTS."""
    rng = np.random.default_rng(seed)
    info = np.iinfo(dt)
    lo, hi = (0, 255) if dt == U8 else (-1024, 3071)
    scale = 120.0 if dt == U8 else 2500.0
    nz, ny, nx = shape
    if kind == "binary":
        v = np.where(rng.random(shape) < 0.5, hi, lo)
    elif kind == "full":
        v = rng.integers(int(info.min), int(info.max) + 1, shape)
    elif kind == "smooth":
        f = ndimage.gaussian_filter(rng.normal(size=shape), 1.5)
        v = ISO[dt] + f / max(float(np.abs(f).max()), 1e-12) * scale
    elif kind == "checker":   # every cell active, the densest tiles
        z, y, x = np.indices(shape)
        v = np.where((x + y + z) % 2 == 0, hi, lo)
    elif kind == "six_faces":  # a ball cut by all six faces: inside at every face centre, not at the corners
        z, y, x = np.indices(shape, dtype=np.float64)
        r2 = sum(((c - (n - 1) / 2) / (n / 2)) ** 2 for c, n in ((x, nx), (y, ny), (z, nz)))
        v = ISO[dt] + (1.15 - r2) * scale
    elif kind == "all_in":
        v = np.full(shape, hi)
    elif kind == "all_out":
        v = np.full(shape, lo)
    elif kind == "voxels":    # single inside voxels at the corners and at the word edges x = 31 / 32 / 63 / 64
        v = np.full(shape, lo)
        for z in {0, nz - 1}:
            for y in {0, ny - 1}:
                for x in {0, nx - 1}:
                    v[z, y, x] = hi
        for x, rows in ((31, [(0, 0), (nz - 1, ny - 1)]), (63, [(0, 0), (nz - 1, ny - 1)]),
                        (32, [(nz // 2, ny // 2), (0, ny - 1)]), (64, [(nz // 2, ny // 2), (0, ny - 1)])):
            if x < nx:
                for z, y in rows:
                    v[z, y, x] = hi
    else:
        raise ValueError(kind)
    return np.clip(np.rint(v), info.min, info.max).astype(dt)


def full_range(dt, shape, seed):
    """Uniform noise over the whole dtype range that holds every value next to the isos swept."""
    rng = np.random.default_rng(seed)
    info = np.iinfo(dt)
    flat = rng.integers(int(info.min), int(info.max) + 1, int(np.prod(shape)))
    if dt == U8:
        special = np.arange(256)
    else:
        special = np.array([-32768, -32767, -32766, -3, -2, -1, 0, 1, 2, 225, 226, 227, 32765, 32766, 32767])
    flat[:len(special)] = special
    rng.shuffle(flat)
    return flat.astype(dt).reshape(shape)


def crossing_edges(vol, iso):
    """Grid edges whose ends differ in (vol >= iso): the vertex count, without any case table."""
    inside = vol.astype(np.float64) >= iso
    return sum(int(np.count_nonzero(np.moveaxis(inside, a, 0)[1:] != np.moveaxis(inside, a, 0)[:-1]))
               for a in range(3))


def _at_offset(vol, k):
    """A device copy of vol whose data pointer lies k bytes past a 16-byte boundary."""
    import torch
    raw = np.ascontiguousarray(vol).view(np.uint8).reshape(-1)
    base = torch.zeros(raw.size + 32, dtype=torch.uint8, device="cuda")
    assert base.data_ptr() % 16 == 0
    t = base[k:k + raw.size]
    t.copy_(torch.from_numpy(raw))
    t = t.view(torch.int16 if vol.dtype == I16 else torch.uint8).view(vol.shape)
    assert t.data_ptr() % 16 == k % 16
    return t


def _same(got, want, what):
    (V, F), (Vo, Fo) = got, want
    assert V.shape == Vo.shape and F.shape == Fo.shape, (what, V.shape, Vo.shape, F.shape, Fo.shape)
    assert np.array_equal(F, Fo), what
    assert np.array_equal(V.view(np.uint32), Vo.view(np.uint32)), what


def _device_mesh(mesh, t, iso, origin=ORIGIN, flip=True):
    V, F = mesh.marching_cubes(t, iso, SP, origin, flip)
    return V.cpu().numpy(), F.cpu().numpy()


def _check(mesh, orc, vol, iso, t=None, origin=ORIGIN, flip=True, what=""):
    import torch
    if t is None:
        t = torch.from_numpy(np.ascontiguousarray(vol)).cuda()
    got = _device_mesh(mesh, t, iso, origin, flip)
    _same(got, orc.marching_cubes(vol, iso, SP, origin, flip), what)
    return got


@pytest.fixture(scope="module")
def mesh():
    from invesalius3_b200 import device, mesh
    device.require_cuda()
    return mesh


# ------------------------------------------------------------------------------------ 2. geometry
@pytest.mark.gpu
@pytest.mark.parametrize("kind", CONTENTS)
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("shape", GEOM_SHAPES, ids=_sid)
def test_geometry(mesh, orc, shape, dt, kind):
    vol = content(kind, DTYPES[dt], shape, _seed(shape, dt, kind))
    V, F = _check(mesh, orc, vol, ISO[DTYPES[dt]], flip=kind != "smooth", what=(shape, dt, kind))
    if kind in ("all_in", "all_out"):
        assert len(V) == 0 and len(F) == 0
    else:
        assert len(V) == crossing_edges(vol, ISO[DTYPES[dt]])


# ------------------------------------------------------------------------------------ 3. iso sweep
SWEEP = [(d, s, iso) for d, isos in (("uint8", U8_ISOS), ("int16", I16_ISOS)) for s in SWEEP_SHAPES[d] for iso in isos]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,shape,iso", SWEEP, ids=[f"{d}-{_sid(s)}-{iso!r}" for d, s, iso in SWEEP])
def test_iso_sweep(mesh, orc, dt, shape, iso):
    vol = full_range(DTYPES[dt], shape, _seed(dt, shape))
    V, F = _check(mesh, orc, vol, iso, what=(dt, shape, iso))
    assert len(V) == crossing_edges(vol, iso)
    if not math.isfinite(iso):
        assert len(V) == 0 and len(F) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DTYPES))
def test_nan_iso_is_rejected(mesh, dt):
    import torch
    t = torch.from_numpy(full_range(DTYPES[dt], (3, 5, 64), 1)).cuda()
    with pytest.raises(ValueError, match="NaN"):
        mesh.marching_cubes(t, math.nan, SP, ORIGIN, True)


# ------------------------------------------------------------------------------------ 4. misaligned
@pytest.mark.gpu
@pytest.mark.parametrize("dt,shape,k", MISALIGNED, ids=[f"{d}-{_sid(s)}-{k}" for d, s, k in MISALIGNED])
def test_misaligned_view(mesh, orc, dt, shape, k):
    for kind in ("full", "smooth"):
        vol = content(kind, DTYPES[dt], shape, _seed(dt, shape, kind))
        for iso in (ISO[DTYPES[dt]], 200.5):
            _check(mesh, orc, vol, iso, t=_at_offset(vol, k), what=(kind, iso))


@pytest.mark.gpu
@pytest.mark.parametrize("dt,shape", SLAB_VOLUMES, ids=[f"{d}-{_sid(s)}" for d, s in SLAB_VOLUMES])
def test_z_slab_of_resident_volume(mesh, orc, dt, shape):
    import torch
    vol = content("smooth", DTYPES[dt], shape, _seed(dt, shape, "slab"))
    t = torch.from_numpy(vol).cuda()
    for z0, z1 in SLABS:
        s = t[z0:z1]
        assert s.is_contiguous() and s.data_ptr() - t.data_ptr() == z0 * shape[1] * shape[2] * vol.itemsize
        _check(mesh, orc, vol[z0:z1], ISO[DTYPES[dt]], t=s, origin=(0, 0, z0), what=(z0, z1))


# ------------------------------------------------------------------------------------ 5. Z shards
def shard_volume(case, kind):
    dt = DTYPES[case["dtype"]]
    vol = content(kind, dt, case["shape"], _seed(case["shape"], case["dtype"], kind))
    lo, hi = (0, 255) if dt == U8 else (-1024, 3071)
    if kind == "smooth":
        vol[case["full"]] = hi
        if case["quiet"] is not None:   # the quiet shard's planes and the plane it is handed: no crossing
            z0, z1 = _ext_bounds(case["bounds"])[case["quiet"]]
            vol[z0:z1] = lo
    return vol


def owned_vertices(vol, iso, z0, z1):
    """Crossing edges owned by the voxels of planes [z0, z1) (an edge belongs to its lower end)."""
    inside = vol.astype(np.float64) >= iso
    own = inside[z0:z1]
    n = int(np.count_nonzero(own[:, :, 1:] != own[:, :, :-1])) + int(np.count_nonzero(own[:, 1:] != own[:, :-1]))
    up = inside[z0:min(z1 + 1, len(inside))]
    return n + int(np.count_nonzero(up[1:] != up[:-1]))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["binary", "smooth"])
@pytest.mark.parametrize("ci", range(len(SHARDS)))
def test_z_shards(orc, ci, kind):
    """The order dist.marching_cubes drives a Z-sharded volume in: count every shard (all but the
    last skip the vertices of the plane they share), vertex bases = the prefix sums of V, then emit
    with the next shard's plane-0 records and vertex base."""
    import torch
    from invesalius3_b200 import dist
    case = SHARDS[ci]
    vol = shard_volume(case, kind)
    iso = ISO[vol.dtype]
    be = dist.DeviceBackend()
    ext = _ext_bounds(case["bounds"])
    n = len(ext)
    resident = torch.from_numpy(vol).cuda()
    sts = []
    for i, (z0, z1) in enumerate(ext):
        if case["place"] == "view":
            t = resident[z0:z1]
        elif case["place"] == "copy":
            t = torch.from_numpy(np.ascontiguousarray(vol[z0:z1])).cuda()
        else:
            t = _at_offset(vol[z0:z1], case["place"])
        assert t.data_ptr() % 16 == _shard_offset(case, z0) % 16
        sts.append(be.mc_count(t, iso, skip_last=i < n - 1))
    counts = np.array([[st["V"], st["T"]] for st in sts], np.int64)
    vbases = np.concatenate([[0], np.cumsum(counts[:, 0])[:-1]])
    recs = [be.mc_plane0_records(st) for st in sts]
    flip = ci % 2 == 0
    Vs, Fs = [], []
    for i, st in enumerate(sts):
        last = i == n - 1
        v, f = be.mc_emit(st, SP, (ORIGIN[0], ORIGIN[1], ORIGIN[2] + case["bounds"][i]), flip, int(vbases[i]),
                          None if last else recs[i + 1], 0 if last else int(vbases[i + 1]))
        Vs.append(v.cpu().numpy())
        Fs.append(f.cpu().numpy())
    torch.cuda.synchronize()
    # per shard: V = the crossings its own planes own, T = the triangles of its slab's cells
    for i, (z0, z1) in enumerate(ext):
        assert counts[i, 0] == owned_vertices(vol, iso, case["bounds"][i], case["bounds"][i + 1]), i
        assert counts[i, 1] == len(orc.marching_cubes(vol[z0:z1], iso, SP, ORIGIN, flip)[1]), i
        assert len(Vs[i]) == counts[i, 0] and len(Fs[i]) == counts[i, 1]
    if kind == "smooth" and case["quiet"] is not None:
        assert tuple(counts[case["quiet"]]) == (0, 0)
    want = orc.marching_cubes(vol, iso, SP, ORIGIN, flip)
    assert counts[:, 0].sum() == len(want[0]) and counts[:, 1].sum() == len(want[1])
    _same((np.concatenate(Vs), np.concatenate(Fs)), want, (ci, kind))
