"""Timings of the porous-creation plugin's TPMS and Blobs scaffolds on the device (invesalius3_b200.porous), printed
as one JSON line.

Device, from CUDA events over warmed repeats (median), for each of the six surfaces at the dialog's default 250^3 and
at its largest 1000^3, bounds -10 .. 10 on every axis: b2v_tpms_f64 (8 B written per voxel) and b2v_tpms_i16, the
OK step's two launches (2 B written per voxel). For Blobs at 250^3 and sigma 5: the three Gaussian passes
(filters._gaussian, 3 x (8 B read + 8 B written) per voxel) and b2v_image_normalize_f64_i16 (2 x 8 B read + 2 B
written). Algorithmic bytes are set against the 3.35 TB/s HBM3 data sheet.
Wall times (host clock around calls that end in a synchronise) of the numpy API: create_schwarzp and
create_schwarzp_i16 at 250^3 and create_schwarzp_i16 at 1000^3 (tables, launches, download), and create_blobs_i16 at
250^3, whose host draw and upload are timed apart.
Host: the plugin's flow once at 250^3 (create_schwarzp or create_blobs, then image_normalize to -1000 .. 1000), in
the checker's NumPy / SciPy restatement; the int16 results are compared byte for byte.
Run: python tools/bench_porous.py [--reps N]"""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
from bench_mask_editor import HBM_TBPS, card, events, wall  # noqa: E402
from invesalius3_b200 import _lib, filters, porous  # noqa: E402
from invesalius3_b200.device import _p, _stream  # noqa: E402
from oracle import porous as op  # noqa: E402

BOUNDS = (-10.0, 10.0, -10.0, 10.0, -10.0, 10.0)
SIGMA = 5.0


def share(nbytes, ms):
    return round(nbytes / (ms * 1e-3) / (HBM_TBPS * 1e12), 3)


def host_once(fn):
    t0 = time.perf_counter()
    r = fn()
    return r, round((time.perf_counter() - t0) * 1e3, 1)


def tpms_device(n, reps):
    """Event times of both TPMS entries for every surface on an n^3 volume."""
    shape = (n, n, n)
    z, y, x = porous._axes(*BOUNDS, n, n, n)
    tab = torch.from_numpy(porous._tables(z, y, x)).cuda()
    f64 = torch.empty(shape, dtype=torch.float64, device="cuda")
    i16 = torch.empty(shape, dtype=torch.int16, device="cuda")
    ws = torch.empty(_lib.load().b2v_tpms_i16_workspace_bytes(*shape), dtype=torch.uint8, device="cuda")
    res = {}
    for code, name in enumerate(porous.SURFACES):
        ms_f = events(lambda: _lib.call("b2v_tpms_f64", _p(tab), *shape, code, _p(f64), _stream()), reps)
        ms_i = events(lambda: _lib.call("b2v_tpms_i16", _p(tab), *shape, code, 2000.0, -1000.0, -1000, _p(ws), _p(i16),
                                        _stream()), reps)
        res[name] = {"f64_ms": round(ms_f, 3), "f64_share_of_hbm_peak": share(8 * n ** 3, ms_f),
                     "i16_ms": round(ms_i, 3), "i16_share_of_hbm_peak": share(2 * n ** 3, ms_i)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, plim = card()
    res = {"metric": "porous_tpms_blobs", "gpu": name, "power_limit": plim, "bounds": BOUNDS, "blobs_sigma": SIGMA}

    res["device_ms"] = {"tpms_250": tpms_device(250, args.reps), "tpms_1000": tpms_device(1000, max(3, args.reps // 2))}
    torch.cuda.empty_cache()

    n3 = 250 ** 3
    np.random.seed(0)
    blob = torch.from_numpy(np.random.random((250, 250, 250))).cuda()
    ms_g = events(lambda: filters._gaussian(blob, SIGMA, torch.float64), args.reps)
    blurred = filters._gaussian(blob, SIGMA, torch.float64)
    ms_n = events(lambda: porous.image_normalize_device(blurred, -1000, 1000), args.reps)
    res["device_ms"]["blobs_250"] = {"gaussian_3_passes_ms": round(ms_g, 3),
                                     "gaussian_share_of_hbm_peak": share(3 * 16 * n3, ms_g),
                                     "normalize_ms": round(ms_n, 3), "normalize_share_of_hbm_peak": share(18 * n3, ms_n)}
    del blob, blurred
    torch.cuda.empty_cache()

    draw = np.random.random((250, 250, 250))
    res["wall_ms"] = {
        "create_schwarzp Schwarz D 250 (float64 download)": round(
            wall(lambda: porous.create_schwarzp("Schwarz D", *BOUNDS, 250, 250, 250), args.reps), 1),
        "create_schwarzp_i16 Schwarz D 250": round(
            wall(lambda: porous.create_schwarzp_i16("Schwarz D", *BOUNDS, 250, 250, 250), args.reps), 1),
        "create_schwarzp_i16 Schwarz D 1000": round(
            wall(lambda: porous.create_schwarzp_i16("Schwarz D", *BOUNDS, 1000, 1000, 1000), 3), 1),
        "create_blobs_i16 250": round(wall(lambda: porous.create_blobs_i16(250, 250, 250, SIGMA), args.reps), 1),
        "blobs host draw 250": round(wall(lambda: np.random.random((250, 250, 250)), args.reps), 1),
        "blobs upload 250": round(wall(lambda: torch.from_numpy(draw).cuda(), args.reps), 1),
    }

    # host: the plugin's flow once, against the device's int16
    host_ms, equal = {}, {}
    for method in ("Schwarz P", "Schwarz D"):
        f, ms_f = host_once(lambda: op.create_schwarzp(method, *BOUNDS, 250, 250, 250))
        h, ms_n = host_once(lambda: op.image_normalize(f, -1000, 1000))
        host_ms[method] = {"create_schwarzp": ms_f, "image_normalize": ms_n}
        equal[method] = bool(np.array_equal(porous.create_schwarzp_i16(method, *BOUNDS, 250, 250, 250), h))
    np.random.seed(3)
    f, ms_f = host_once(lambda: op.create_blobs(250, 250, 250, SIGMA))
    h, ms_n = host_once(lambda: op.image_normalize(f, -1000, 1000))
    host_ms["Blobs"] = {"create_blobs": ms_f, "image_normalize": ms_n}
    np.random.seed(3)
    equal["Blobs"] = bool(np.array_equal(porous.create_blobs_i16(250, 250, 250, SIGMA), h))
    res["host_ms"] = host_ms
    res["equal"] = equal
    print(json.dumps(res))


if __name__ == "__main__":
    main()
