"""Timings of "Remove non-visible faces" on the device (invesalius3_b200.visible_faces) for the bone surface
of the 512^3 phantom, printed as one JSON line.

Input: phantom.ct((512,)*3, seed=2) thresholded at (226, 3071), then mesh.marching_cubes at iso 127 with unit
spacing (the surface stays on the device). Reports V and T of that surface; the time of
remove_non_visible_faces_device with the six default positions from CUDA events over warmed repeats (median;
the call synchronises twice, so this is the whole call as a caller sees it); the time of the C checker
(oracle/visibility.c, one host core, sequential) once; V' and T' of the result, and whether the device
result equals the checker's. The card name and power limit are read in the same run.
Run: python tools/bench_visibility.py [--reps N]"""
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
from invesalius3_b200 import device as dev, phantom, visible_faces as vf  # noqa: E402
from invesalius3_b200.mesh import marching_cubes  # noqa: E402
from oracle import visibility as ov  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, plim = card()
    vol = phantom.ct((512, 512, 512), seed=2)
    mask = dev.threshold(torch.from_numpy(vol).cuda(), 226, 3071)
    del vol
    V, F = marching_cubes(mask, 127, (1.0, 1.0, 1.0), (0, 0, 0), True)
    del mask
    vo, fo = vf.remove_non_visible_faces_device(V, F)
    ms = events(lambda: vf.remove_non_visible_faces_device(V, F), args.reps)
    v, f = V.cpu().numpy(), F.cpu().numpy()
    t0 = time.perf_counter()
    wv, wf = ov.remove_non_visible_faces(v, f)
    oracle_ms = (time.perf_counter() - t0) * 1e3
    same = bool(np.array_equal(vo.cpu().numpy().view(np.uint32), wv.view(np.uint32)) and
                np.array_equal(fo.cpu().numpy(), wf))
    res = {"metric": "remove_non_visible_faces_512_bone", "gpu": name, "power_limit": plim,
           "V": int(V.shape[0]), "T": int(F.shape[0]), "V_out": int(vo.shape[0]), "T_out": int(fo.shape[0]),
           "device_call_ms": round(ms, 3), "oracle_cpu_ms": round(oracle_ms, 0), "verified": same}
    print(json.dumps(res))
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
