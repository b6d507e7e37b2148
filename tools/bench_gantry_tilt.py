"""Timings of the gantry-tilt correction (invesalius3_b200.resample) at 512^3, printed as one JSON line.

Input: phantom.ct((512,)*3, seed=2) as int16, tilted by 15 degrees with spacing (0.5, 0.5, 1.0), as the DICOM
import runs imagedata_utils.FixGantryTilt on a tilted series (control.py:1331, :1334).

Reports: the device time of fix_gantry_tilt_device from CUDA events over warmed repeats (median, min and max; the
volume is restored outside the timed window), its algorithmic bytes over that time against the 3.35 TB/s HBM3
data sheet, the wall time of fix_gantry_tilt through the numpy API (PCIe included), the wall time of the
sequential SciPy loop (run once), and whether both device paths equal the loop.
Run: python tools/bench_gantry_tilt.py [--reps N]"""
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
sys.path.insert(0, str(ROOT / "tests"))
from bench_mask_editor import card, wall  # noqa: E402
from invesalius3_b200 import device as dev, phantom, resample  # noqa: E402
import shift_model as sm  # noqa: E402

SHAPE = (512, 512, 512)
SPACING = (0.5, 0.5, 1.0)
TILT = 15


def algorithmic_bytes(n: int) -> int:
    """Original slice minima: 2 B read; y pass: 2 B + 3 x 8 B read, 2 x 8 B written; x pass: 3 x 8 B read,
    2 x 8 B written; gather: ~8 B read (its taps hit cache), 2 B written. The fill's writes are not counted."""
    return n * (2 + (2 + 24 + 16) + (24 + 16) + (8 + 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, plim = card()
    vol = phantom.ct(SHAPE, seed=2)
    src = dev.to_device(vol)
    t = src.clone()

    def restore():
        t.copy_(src)

    def run():
        resample.fix_gantry_tilt_device(t, SPACING, TILT)

    for _ in range(2):
        restore()
        run()
    times = []
    for _ in range(args.reps):
        restore()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); run(); e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    ms = float(np.median(times))
    got = t.cpu().numpy()

    arr = vol.copy()
    api = wall(lambda: resample.fix_gantry_tilt(arr, SPACING, TILT), max(3, args.reps // 2), before=lambda: arr.__setitem__(..., vol))
    arr[...] = vol
    resample.fix_gantry_tilt(arr, SPACING, TILT)

    t0 = time.perf_counter()
    ref, _ = sm.reference_loop(vol, SPACING, TILT)
    scipy_ms = (time.perf_counter() - t0) * 1e3

    nbytes = algorithmic_bytes(vol.size)
    checks = {"device_equals_loop": bool(np.array_equal(got, ref)), "numpy_api_equals_loop": bool(np.array_equal(arr, ref))}
    res = {"metric": "gantry_tilt_512", "gpu": name, "power_limit": plim, "tilt_deg": TILT, "spacing": SPACING,
           "device_ms": round(ms, 3), "device_ms_min": round(min(times), 3), "device_ms_max": round(max(times), 3),
           "reps": args.reps, "algorithmic_gb": round(nbytes / 1e9, 3),
           "hbm_share_of_datasheet": round(nbytes / (ms * 1e-3) / 3.35e12, 3),
           "numpy_api_wall_ms": round(api, 1), "scipy_loop_host_ms": round(scipy_ms, 0), "checks": checks,
           "verified": all(checks.values())}
    print(json.dumps(res))
    return 0 if res["verified"] else 1


if __name__ == "__main__":
    sys.exit(main())
