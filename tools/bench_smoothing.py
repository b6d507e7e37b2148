"""Timings of the Laplacian surface smoothing on the device (invesalius3_b200.surface_smoothing), printed as one
JSON line.

Inputs: (1) the bone surface of phantom.ct((512,)*3, seed=2) thresholded at (226, 3071), contoured by
mesh.marching_cubes at iso 127, with polydata_utils.ApplySmoothFilter's settings (20 iterations, relaxation
0.4, feature angle 80, feature-edge and boundary smoothing off); (2) a strip of 200 000 triangles with
decimate_polydata's settings (15 iterations, VTK's defaults, boundary smoothing on), where every point waits
for the one two ids below it: the longest dependency chain a mesh can have. Both stay on the device. For each:
V, T, the dependency levels of one iteration and the steps of the run (levels x iterations), the median
device time of smooth_polydata_device from CUDA events over warmed repeats (the call synchronises the host
three times for its counts), the C checker's time once (one host core, sequential), and whether the device
result equals the checker's bit for bit. The card name and power limit are read in the same run.
Run: python tools/bench_smoothing.py [--reps N]"""
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
from bench_mask_editor import card, events  # noqa: E402
from invesalius3_b200 import device as dev, phantom, surface_smoothing as ss  # noqa: E402
from invesalius3_b200.mesh import marching_cubes  # noqa: E402
from oracle import smoothing as osm  # noqa: E402
from connectivity_meshes import strip  # noqa: E402
from smoothing_meshes import APPLY_SMOOTH, DECIMATE  # noqa: E402


def measure(label, settings, V, F, kw, reps):
    r = ss.smooth_polydata_device(V, F, **kw)
    res = {"input": label, "settings": settings, "V": int(V.shape[0]), "T": int(F.shape[0]), "levels": r.levels,
           "iterations": r.iterations, "steps": r.steps}
    res["device_ms"] = round(events(lambda: ss.smooth_polydata_device(V, F, **kw), reps), 3)
    v, f = V.cpu().numpy(), F.cpu().numpy()
    t0 = time.perf_counter()
    want = osm.smooth(v, f, **kw)
    res["oracle_cpu_ms"] = round((time.perf_counter() - t0) * 1e3, 0)
    res["verified"] = bool(np.array_equal(r.vertices.cpu().numpy().view(np.uint32), want["vertices"].view(np.uint32))
                           and np.array_equal(r.point_types.cpu().numpy(), want["types"])
                           and r.iterations == want["iterations"])
    return res


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
    bone = measure("phantom_512_bone", "ApplySmoothFilter", V, F, APPLY_SMOOTH, args.reps)
    del V, F
    v, f = strip(200_000)
    chain = measure("strip_200000", "decimate_polydata", torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(),
                    DECIMATE, args.reps)
    res = {"metric": "surface_smoothing", "gpu": name, "power_limit": plim, "results": [bone, chain],
           "verified": bone["verified"] and chain["verified"]}
    print(json.dumps(res))
    return 0 if res["verified"] else 1


if __name__ == "__main__":
    sys.exit(main())
