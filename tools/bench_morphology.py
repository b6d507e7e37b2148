"""Timings of the mask-morphology plugin on the device (invesalius3_b200.morphology) at 512^3, printed as
one JSON line.

Input: the bone mask (> 226 -> 255) of phantom.ct((512,)*3, seed=2) in the padded layout of mask.matrix
(513^3 uint8, the first plane, row and column 0 but for the slice flags). Cases: erosion and dilation with
ball(1), ball(3), ball(10) and disk(10) on every axial slice, as MaskMorphologyPanel.OnApply applies them.

Reports, per case: the device time of binary_morphology_device from CUDA events over warmed repeats (median),
its algorithmic bytes (planar: the input read and the output written, 2 B per voxel; ball: also the
workspace written and read, 4 B) against the 3.35 TB/s HBM3 data sheet, the wall time of mask_morphology
(numpy in / numpy out, PCIe included), SciPy's host time once for r <= 3 (ball(10) dilation in SciPy takes
minutes at this size), and whether the device result equals the NumPy restatement oracle/morphology.py (and
SciPy's, where it ran). tests/test_morphology_model.py pins the restatement to SciPy.
Run: python tools/bench_morphology.py [--reps N]"""
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
from bench_mask_editor import HBM_TBPS, card, events, wall  # noqa: E402
from invesalius3_b200 import device as dev, morphology as mm, phantom  # noqa: E402
from oracle import morphology as om  # noqa: E402

SHAPE = (512, 512, 512)
CASES = [("ball", 1), ("ball", 3), ("ball", 10), ("disk", 10)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, plim = card()
    vol = phantom.ct(SHAPE, seed=2)
    mask = np.zeros(tuple(n + 1 for n in SHAPE), np.uint8)
    mask[1:, 1:, 1:] = np.where(vol > 226, 255, 0)
    mask[1:, 0, 0] = 1
    del vol
    body = mask[1:, 1:, 1:]
    a = body > 0
    t = dev.to_device(body)
    res = {"metric": "mask_morphology_512", "gpu": name, "power_limit": plim, "shape": SHAPE,
           "set_voxels": int(a.sum()), "cases": {}}
    checks = {}
    for op_i, op in enumerate(("erosion", "dilation")):
        for struct, r in CASES:
            planar = struct == "disk"
            key = f"{op}_{struct}{r}"
            out, counts = mm.binary_morphology_device(t, op, r, planar, set_value=255)
            ms = events(lambda: mm.binary_morphology_device(t, op, r, planar, set_value=255, out=out), args.reps)
            api = wall(lambda: mm.mask_morphology(mask, op_i, r, int(not planar)), max(3, args.reps // 3))
            got = out.cpu().numpy() == 255
            n_in, n_out = (int(v) for v in counts.cpu())
            want = om.binary_morphology(a, op, r, planar)
            checks[key] = bool(np.array_equal(got, want))
            checks[key + "_counts"] = (n_in, n_out) == (int(a.sum()), int(want.sum()))
            new, n0, n1 = mm.mask_morphology(mask, op_i, r, int(not planar))
            checks[key + "_mask_morphology"] = bool(new is not None and (n0, n1) == (n_in, n_out) and
                                                    np.array_equal(new[1:, 1:, 1:] == 255, want))
            scipy_ms = None
            if r <= 3:   # the ball cases
                t0 = time.perf_counter()
                ref = (ndi.binary_erosion(a, mm.ball(r), border_value=1) if op == "erosion" else
                       ndi.binary_dilation(a, mm.ball(r), border_value=0))
                scipy_ms = round((time.perf_counter() - t0) * 1e3, 0)
                checks[key + "_scipy"] = bool(np.array_equal(got, ref))
            nbytes = (2 if planar else 4) * a.size
            res["cases"][key] = {
                "device_ms": round(ms, 3), "mask_morphology_wall_ms": round(api, 1), "scipy_host_ms": scipy_ms,
                "result_voxels": n_out, "algorithmic_gb": round(nbytes / 1e9, 3),
                "hbm_share_of_datasheet": round(nbytes / (ms * 1e-3) / (HBM_TBPS * 1e12), 3),
            }
    res["checks"] = checks
    res["verified"] = all(checks.values())
    print(json.dumps(res))
    return 0 if res["verified"] else 1


if __name__ == "__main__":
    sys.exit(main())
