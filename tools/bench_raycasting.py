"""Timings of the volume rendering's data preparation on the device (invesalius3_b200.raycasting), printed as one
JSON line per input.

Inputs: the Cranium crop of tests/golden/cranium_crop.npz and phantom.ct((512,)*3, seed=2). For each, the median
device time from CUDA events over warmed repeats of: the upload of the int16 matrix, the flip and shift (the
minmax pass included), one and two passes of the presets' "Basic Smooth 5x5", the histogram (minmax and two
histogram passes, including its synchronise), and the download of the uint16 result to a host array. The C
checker (one host core, sequential) is timed once for the flip and shift and for one smoothing pass; that is the
checker's time, not VTK's, which is not measured. One smoothing pass is also set against its data-sheet bounds
on an H100 SXM: 4 B per voxel at 3.35 TB/s, and 50 float64 operations per voxel (25 multiplies and 25 adds, no
FMA) at 64 lanes x 132 SMs x 1.98 GHz. The equality flags compare the device with the checker on the same input;
the card name and power limit are read in the same run.
Run: python tools/bench_raycasting.py [--reps N]"""
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
from bench_mask_editor import card, events  # noqa: E402
from invesalius3_b200 import device as dev, phantom, raycasting as rc  # noqa: E402
from oracle import raycasting as orc  # noqa: E402

SMOOTH = [i / 60.0 for i in (1, 1, 1, 1, 1, 1, 4, 4, 4, 1, 1, 4, 12, 4, 1, 1, 4, 4, 4, 1, 1, 1, 1, 1, 1)]
HBM_BPS = 3.35e12
FP64_OPS = 64 * 132 * 1.98e9


def measure(name, m, reps):
    n = m.size
    t = dev.to_device(m)
    u, rng = rc.flip_shift_device(t)
    a, b = torch.empty_like(u), torch.empty_like(u)
    host = np.empty(m.shape, np.uint16)
    ms = {
        "upload": events(lambda: dev.to_device(m), reps),
        "flip_shift": events(lambda: rc.flip_shift_device(t), reps),
        "smooth_1": events(lambda: rc.convolve5x5_device(u, SMOOTH, a), reps),
        "smooth_2": events(lambda: rc.convolve5x5_device(rc.convolve5x5_device(u, SMOOTH, a), SMOOTH, b), reps),
        "histogram": events(lambda: rc.accumulate_histogram_device(t), reps),
        "download": events(lambda: dev.to_host(a, host), reps),
    }
    counts, lo, hi = rc.accumulate_histogram_device(t)
    one = rc.convolve5x5_device(u, SMOOTH, a).cpu().numpy()
    two = rc.convolve5x5_device(rc.convolve5x5_device(u, SMOOTH, a), SMOOTH, b).cpu().numpy()
    t0 = time.perf_counter()
    want_u, want_rng = orc.flip_shift(m)
    cpu_flip = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    want_one = orc.convolve(want_u, SMOOTH)
    cpu_smooth = (time.perf_counter() - t0) * 1e3
    want_counts, wlo, whi = orc.histogram(m)
    equal = {
        "flip_shift": bool(rng == want_rng and np.array_equal(u.cpu().numpy(), want_u)),
        "smooth_1": bool(np.array_equal(one, want_one)),
        "smooth_2": bool(np.array_equal(two, orc.convolve(want_one, SMOOTH))),
        "histogram": bool((lo, hi) == (wlo, whi) and np.array_equal(counts.cpu().numpy(), want_counts)),
    }
    bounds = {"hbm_ms": round(4 * n / HBM_BPS * 1e3, 3), "fp64_ms": round(50 * n / FP64_OPS * 1e3, 3)}
    return {"metric": "raycasting_prep", "input": name, "shape": list(m.shape), "voxels": n,
            "device_ms": {k: round(v, 3) for k, v in ms.items()},
            "smooth_1_gvoxel_per_s": round(n / ms["smooth_1"] / 1e6, 2),
            "smooth_1_datasheet_bounds": bounds,
            "checker_one_core_ms": {"flip_shift": round(cpu_flip, 1), "smooth_1": round(cpu_smooth, 1)},
            "equal": equal, "verified": all(equal.values())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, plim = card()
    crop = np.load(ROOT / "tests" / "golden" / "cranium_crop.npz")["matrix_crop"]
    for label, m in (("cranium_crop", crop), ("phantom_512", phantom.ct((512, 512, 512), seed=2))):
        res = measure(label, m, args.reps)
        res.update(gpu=name, power_limit=plim)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
