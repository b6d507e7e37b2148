"""Timings of the low-quality surface resample (invesalius3_b200.resample) at 512^3, printed as one JSON line.

Inputs: phantom.ct((512,)*3, seed=3) as int16, and its bone mask (> 226 -> 255) in the padded layout of
mask.matrix (513^3 uint8, the first plane, row and column 0), both zoomed by 1/2 and 1/3 at order 2 as
SurfaceManager.AddNewActor does for the "Medium" and "Low" qualities (surface.py:1352-1353).

Reports, per case: the device time of zoom_device from CUDA events over warmed repeats (median), the
algorithmic bytes of the prefilter and gather over that time against the 3.35 TB/s HBM3 data sheet, the
wall time of resize_image_array (numpy in / numpy out, PCIe dominates), the wall time of SciPy's zoom on
the host (run once), and whether the device output equals SciPy's.
Run: python tools/bench_zoom.py [--reps N]"""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch
from scipy import ndimage as ndi

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
from bench_mask_editor import card, events, wall  # noqa: E402
from invesalius3_b200 import device as dev, phantom, resample  # noqa: E402

SHAPE = (512, 512, 512)


def algorithmic_bytes(n_in: int, in_size: int, n_out: int, out_size: int) -> int:
    """z pass: two reads of the input dtype, three float64 accesses; y and x passes: five float64
    accesses each; gather: one float64 read per input voxel (its taps hit cache) and the output."""
    return n_in * (2 * in_size + 3 * 8 + 2 * 5 * 8 + 8) + n_out * out_size


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, plim = card()
    vol = phantom.ct(SHAPE, seed=3)
    mask = np.zeros(tuple(n + 1 for n in SHAPE), np.uint8)
    mask[1:, 1:, 1:] = np.where(vol > 226, 255, 0)
    mask[1:, 0, 0] = 1
    res = {"metric": "zoom_512_order2", "gpu": name, "power_limit": plim, "order": 2, "cases": {}}
    checks = {}
    for label, arr in (("image_int16", vol), ("mask_uint8_padded", mask)):
        t = dev.to_device(arr)
        for fname, f in (("1/2", 0.5), ("1/3", 1 / 3)):
            key = f"{label}@{fname}"
            tdt = t.dtype
            out = resample.zoom_device(t, f, 2, tdt)
            ms = events(lambda: resample.zoom_device(t, f, 2, tdt), args.reps)
            api = wall(lambda: resample.resize_image_array(arr, f), max(3, args.reps // 2))
            t0 = time.perf_counter()
            ref = ndi.zoom(arr, f, arr.dtype, order=2)
            scipy_ms = (time.perf_counter() - t0) * 1e3
            got = out.cpu().numpy()
            checks[key] = bool(got.shape == ref.shape and np.array_equal(got, ref))
            checks[key + " numpy_api"] = bool(np.array_equal(resample.resize_image_array(arr, f), ref))
            nbytes = algorithmic_bytes(arr.size, arr.itemsize, ref.size, ref.itemsize)
            res["cases"][key] = {
                "in_shape": list(arr.shape), "out_shape": list(ref.shape),
                "device_ms": round(ms, 3), "numpy_api_wall_ms": round(api, 1), "scipy_host_ms": round(scipy_ms, 0),
                "algorithmic_gb": round(nbytes / 1e9, 3),
                "hbm_share_of_datasheet": round(nbytes / (ms * 1e-3) / 3.35e12, 3),
            }
        del t
        torch.cuda.empty_cache()
    res["checks"] = checks
    res["verified"] = all(checks.values())
    print(json.dumps(res))
    return 0 if res["verified"] else 1


if __name__ == "__main__":
    sys.exit(main())
