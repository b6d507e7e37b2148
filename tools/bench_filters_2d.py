"""Timings of the image-filter action's "2D" branch on the device (invesalius3_b200.filters.apply_image_filter) at
512^3, printed as one JSON line.

Input: phantom.ct((512,)*3, seed=2), int16. Cases: the dialog choices Gaussian sigma 1, median (dialog value 3 ->
size 5), mean (dialog "kernel size" 3 -> size 7), sharpening 1, despeckle sigma 1 and border detection sigma 1,
each on every axial, coronal and sagittal slice; and the image histogram of the border-detection result.

Reports, per case: the device time of apply_image_filter_device from CUDA events over warmed repeats (median),
the wall time of apply_image_filter (numpy in / numpy out, PCIe included), the compulsory bytes (the int16 image
read and the result written, 4 B per voxel) and the bytes of the passes the device makes (each pass reading its
inputs and writing its output once), that traffic against the 3.35 TB/s HBM3 data sheet, and whether the result
equals the per-slice SciPy loop (tests/filters_2d_model.py) on a slab of SLAB slices, so that the run stays short.
Run: python tools/bench_filters_2d.py [--reps N]"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
sys.path.insert(0, str(ROOT / "tests"))
import filters_2d_model as fm  # noqa: E402
from bench_mask_editor import HBM_TBPS, card, events, wall  # noqa: E402
from invesalius3_b200 import device as dev, filters, phantom  # noqa: E402

SHAPE = (512, 512, 512)
SLAB = 8
CASES = [("gaussian", 0, 1.0), ("median", 1, 3.0), ("mean", 2, 3.0), ("sharpen", 3, 1.0), ("despeckle", 4, 1.0),
         ("border", 5, 1.0)]
# bytes per voxel of each pass: (read, written)
CAST, GAUSS_I16, GAUSS_F64 = (2, 8), (2, 2), (8, 8)
PASSES = {
    0: [GAUSS_I16] * 2,
    1: [(2, 2)],
    2: [(2, 2)] * 2,
    3: [CAST] + [GAUSS_F64] * 2 + [(2, 0), (2 + 8, 2)],                 # per-slice min / max, sharpen
    4: [GAUSS_I16] * 2,
    5: [CAST] + [GAUSS_F64] * 2 + [GAUSS_F64] * 4 + [(16, 8), (2, 0), (8, 0), (8, 2)],   # sobel, magnitude, stats, cast
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, plim = card()
    vol = phantom.ct(SHAPE, seed=2)
    t = dev.to_device(vol)
    n = vol.size
    res = {"metric": "image_filter_2d_512", "gpu": name, "power_limit": plim, "shape": SHAPE, "cases": {}}
    checks = {}
    for label, ft, value in CASES:
        for orientation, axis in fm.AXIS.items():
            key = f"{label}_{orientation.lower()}"
            run = lambda: filters.apply_image_filter_device(t, ft, value, "2D", orientation)   # noqa: E731
            ms = events(run, args.reps)
            api = wall(lambda: filters.apply_image_filter(vol, ft, value, "2D", orientation), max(3, args.reps // 3))
            got = run()
            k0 = SHAPE[axis] // 2 - SLAB // 2
            idx = [slice(None)] * 3
            idx[axis] = slice(k0, k0 + SLAB)
            slab = np.ascontiguousarray(vol[tuple(idx)])
            checks[key] = bool(np.array_equal(got[tuple(idx)].cpu().numpy(), fm.loop_2d(slab, ft, value, orientation)))
            nbytes = sum(r + w for r, w in PASSES[ft]) * n
            res["cases"][key] = {
                "device_ms": round(ms, 3), "apply_image_filter_wall_ms": round(api, 1),
                "compulsory_gb": round(4 * n / 1e9, 3), "pass_gb": round(nbytes / 1e9, 3), "passes": len(PASSES[ft]),
                "hbm_share_of_datasheet": round(nbytes / (ms * 1e-3) / (HBM_TBPS * 1e12), 3),
            }
            del got
    border = filters.apply_image_filter_device(t, 5, 1.0, "2D", "Axial")
    ms = events(lambda: filters.image_histogram_device(border), args.reps)
    host = border.cpu().numpy()
    api = wall(lambda: filters.image_histogram(host), max(3, args.reps // 3))
    h, i, e = filters.image_histogram(host)
    checks["histogram"] = bool(np.array_equal(h, np.histogram(host, int(e) - int(i), (i, e))[0]) and
                               (i, e) == (host.min(), host.max()))
    res["cases"]["histogram"] = {"device_ms": round(ms, 3), "image_histogram_wall_ms": round(api, 1), "bins": int(e) - int(i),
                                 "read_gb": round(4 * n / 1e9, 3),        # the min / max pass and the counting pass
                                 "hbm_share_of_datasheet": round(4 * n / (ms * 1e-3) / (HBM_TBPS * 1e12), 3)}
    res["checks"] = checks
    res["verified"] = all(checks.values())
    print(json.dumps(res))
    return 0 if res["verified"] else 1


if __name__ == "__main__":
    sys.exit(main())
