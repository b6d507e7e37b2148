"""Flood-fill cases under the tuning knob B2V_FF_GRID.

The knob is read once per process (`FloodKnobs` in csrc/floodfill.cu), so every setting floods
in a process of its own:

    python tests/ff_knob_child.py SETTING OUTDIR

floods every case of SETTING on both engines and writes OUTDIR/<case>__<engine>.npy (the mask)
and OUTDIR/results.json (returned round count and `stats` per flood). The cases are seeded, so
tests/test_gpu_floodfill_paths.py rebuilds the same inputs for the serial checker."""
from __future__ import annotations

import json
import sys
import zlib
from pathlib import Path

import numpy as np
from scipy import ndimage
from scipy.ndimage import generate_binary_structure

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

FILL = 1
ENGINES = ("persistent", "host-rounds")
MAX_MINE = 256     # tiles one block of the persistent kernel may own in a round (kMaxMine)

# a one-sided element: the walk is directed, so this cannot be symmetrised
ASYM = np.zeros((3, 3, 3), np.uint8)
for _z, _y, _x in ((1, 1, 2), (1, 2, 1), (0, 1, 1), (2, 0, 0), (1, 0, 2)):
    ASYM[_z, _y, _x] = 1
ELEMENTS = {"6": generate_binary_structure(3, 1), "18": generate_binary_structure(3, 2),
            "26": generate_binary_structure(3, 3), "asym": ASYM}
SYMMETRIC = ("6", "18", "26")

CANON = (37, 45, 1100)      # canonical tiles: 16 x 16 rows x 16 words
NONCANON = (60, 90, 250)    # 8-word rows: generic tiles (32 x 16 x 8 words)

# name -> (environment, {case shape name: (z, y, x)}). "own": a few hundred tiles, one seed in each,
# so that a block owns up to MAX_MINE tiles in the first round; "fallback": more tiles than
# grid * MAX_MINE, which the persistent engine hands to the host-driven rounds.
SETTINGS = {
    "grid1": ({"B2V_FF_GRID": "1"}, {"canon": CANON, "noncanon": NONCANON, "own": (4, 4096, 64),
                                      "fallback": (4, 4112, 64)}),
    "grid3": ({"B2V_FF_GRID": "3"}, {"canon": CANON, "noncanon": NONCANON, "own": (4, 4800, 64),
                                      "fallback": (4, 12304, 64)}),
}


def tile_shape(shape):
    """make_bitvol() restated: tile dims (planes, rows, words) and the tile grid."""
    dz, dy, dx = shape
    wx = -(-dx // 32)

    def pow2ceil(v, cap):
        p = 1
        while p < v and p < cap:
            p <<= 1
        return p

    tw = pow2ceil(wx, 16)
    ty = pow2ceil(dy, 16)
    tz = pow2ceil(dz, 4096 // (tw * ty))
    while tz > 1 and (tz + 2) * (ty + 2) * (tw + 2) * 8 > 48 * 1024:
        tz >>= 1
    return (tz, ty, tw), (-(-dz // tz), -(-dy // ty), -(-wx // tw))


def tile_count(shape) -> int:
    _, (nz, ny, nw) = tile_shape(shape)
    return nz * ny * nw


def cases(setting: str):
    """(case name, shape name, element name) of every flood of the setting."""
    return [(f"{sname}-{ename}", sname, ename) for sname in SETTINGS[setting][1] for ename in ELEMENTS]


def case_inputs(setting: str, sname: str, ename: str) -> dict:
    shape = SETTINGS[setting][1][sname]
    key = zlib.crc32(f"{setting}/{sname}/{ename}".encode())
    rng = np.random.default_rng(key)
    f = ndimage.gaussian_filter(rng.normal(size=shape), 2.0)
    f = (f - f.min()) / (f.max() - f.min() + 1e-9)
    data = (-1000 + f * 3000).astype(np.int16)
    # the directed element needs a denser passable set to get anywhere
    t0, t1 = (300, 2000) if ename in SYMMETRIC else (-100, 2000)
    inr = (data >= t0) & (data <= t1)
    seeds = []
    if sname in ("own", "fallback"):
        ty = tile_shape(shape)[0][1]
        for y0 in range(0, shape[1], ty):          # the tiles are bands of ty rows: one seed in each
            band = inr[:, y0:y0 + ty]
            idx = np.flatnonzero(band)
            if idx.size:
                z, y, x = np.unravel_index(idx[idx.size // 2], band.shape)
                seeds.append((int(x), int(y0 + y), int(z)))
    zz, yy, xx = np.nonzero(inr)
    for i in rng.choice(zz.size, 6, replace=False):
        seeds.append((int(xx[i]), int(yy[i]), int(zz[i])))
    for _ in range(2):                             # anywhere: in range or not
        seeds.append((int(rng.integers(shape[2])), int(rng.integers(shape[1])), int(rng.integers(shape[0]))))
    out0 = np.zeros(shape, np.uint8)
    out0[rng.random(shape) < 0.02] = FILL          # walls
    out0[rng.random(shape) < 0.01] = 200           # other values stay untouched
    return dict(data=data, seeds=seeds, t0=t0, t1=t1, fill=FILL, strct=ELEMENTS[ename], out0=out0)


def main() -> None:
    setting, outdir = sys.argv[1], Path(sys.argv[2])
    import torch
    from invesalius3_b200 import _lib, device as dev
    dev.require_cuda()
    lib = _lib.load()
    results = {}
    for cname, sname, ename in cases(setting):
        c = case_inputs(setting, sname, ename)
        d = torch.from_numpy(c["data"]).cuda()
        for engine in ENGINES:
            lib.b2v_floodfill_set_engine(1 if engine == "persistent" else 0)
            o = torch.from_numpy(c["out0"]).cuda()
            stats = {}
            rounds = dev.floodfill_threshold(d, c["seeds"], c["t0"], c["t1"], c["fill"], c["strct"], o, stats=stats)
            np.save(outdir / f"{cname}__{engine}.npy", o.cpu().numpy())
            results[f"{cname}__{engine}"] = {"rounds": rounds, "stats_rounds": stats["rounds"],
                                             "tiles": stats["tiles"]}
        del d
    lib.b2v_floodfill_set_engine(1)
    (outdir / "results.json").write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
