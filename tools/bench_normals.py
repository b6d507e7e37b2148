"""Timings of surface normals and mass properties on the device (invesalius3_b200.surface_normals), printed as
one JSON line.

Input: phantom.ct((512,)*3, seed=2) thresholded at (226, 3071) and contoured by mesh.marching_cubes at iso
127 without padding, kept on the device: the 512^3 phantom's bone surface. It runs at the settings of
join_process_surface (feature angle 80, auto-orientation) and of the context-aware-smoothing branch (30
degrees, no auto-orientation). For each: V, T, the regions, flips, new points and waves, the median device time
of compute_normals_device from CUDA events over warmed repeats (the call synchronises the host), the C
checker's time once (one host core, sequential), both as triangles/s, and whether the device result equals
the checker's exactly. mass_properties_device is timed the same way. The card name and power limit are read in
the same run.
Run: python tools/bench_normals.py [--reps N]"""
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
from invesalius3_b200 import device as dev, phantom, surface_normals as sn  # noqa: E402
from invesalius3_b200.mesh import marching_cubes  # noqa: E402
from oracle import normals as on  # noqa: E402


def measure(V, F, angle, auto_orient, reps):
    r = sn.compute_normals_device(V, F, angle, auto_orient)
    nt = int(F.shape[0])
    res = {"feature_angle": angle, "auto_orient": auto_orient, "V": int(V.shape[0]), "T": nt,
           "regions": r.regions, "flips": r.flips, "new_points": r.new_points, "waves": r.waves}
    ms = events(lambda: sn.compute_normals_device(V, F, angle, auto_orient), reps)
    v, f = V.cpu().numpy(), F.cpu().numpy()
    t0 = time.perf_counter()
    want = on.compute_normals(v, f, angle, auto_orient)
    cpu_ms = (time.perf_counter() - t0) * 1e3
    res.update(device_ms=round(ms, 3), oracle_cpu_ms=round(cpu_ms, 0), device_tri_per_s=round(nt / ms * 1e3),
               oracle_tri_per_s=round(nt / cpu_ms * 1e3))
    res["verified"] = bool(
        np.array_equal(r.faces.cpu().numpy(), want["faces"])
        and all(np.array_equal(getattr(r, k).cpu().numpy().view(np.uint32), want[k].view(np.uint32))
                for k in ("points", "point_normals", "cell_normals"))
        and (r.regions, r.flips, r.new_points, r.waves)
        == (want["regions"], want["flips"], want["new_points"], want["waves"]))
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
    results = [measure(V, F, 80.0, True, args.reps), measure(V, F, 30.0, False, args.reps)]
    nt = int(F.shape[0])
    got = sn.mass_properties_device(V, F)
    ms = events(lambda: sn.mass_properties_device(V, F), args.reps)
    v, f = V.cpu().numpy(), F.cpu().numpy()
    t0 = time.perf_counter()
    want = on.mass_properties(v, f)
    cpu_ms = (time.perf_counter() - t0) * 1e3
    mass = {"T": nt, "volume": got[0], "area": got[1], "device_ms": round(ms, 3), "oracle_cpu_ms": round(cpu_ms, 0),
            "device_tri_per_s": round(nt / ms * 1e3), "oracle_tri_per_s": round(nt / cpu_ms * 1e3),
            "verified": bool(got == want)}
    res = {"metric": "surface_normals", "input": "phantom_512_bone", "gpu": name, "power_limit": plim,
           "normals": results, "mass_properties": mass,
           "verified": all(r["verified"] for r in results) and mass["verified"]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
