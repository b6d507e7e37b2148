"""Timings of the surface clean and triangle filter on the device (invesalius3_b200.surface_clean) for the bone
surface of the 512^3 phantom, printed as one JSON line.

Input: phantom.ct((512,)*3, seed=2) thresholded at (226, 3071), mesh.marching_cubes at iso 127 with unit
spacing, then compute_normals_device at 30 degrees (the feature splitting duplicates points along the sharp
edges; this is the mesh the "Context aware smoothing" branch cleans). Reports V and T of the split surface;
the time of clean_polydata_device on it, and of triangle_filter_device on the same surface given as strips
(runs of 3 to 7 points cut from the faces' connectivity in order, as offsets + connectivity), from CUDA events
over --reps warmed repeats (median; each call synchronises twice, so this is the whole call as a caller sees it); the time of the C checker
(oracle/clean.c, one host core, sequential) once for each; and whether the device results equal the checker's.
The card name and power limit are read in the same run.
Run: python tools/bench_clean.py [--reps N]"""
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
from invesalius3_b200 import device as dev, phantom, surface_clean as sc, surface_normals as sn  # noqa: E402
from invesalius3_b200.mesh import marching_cubes  # noqa: E402
from oracle import clean as oc  # noqa: E402


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
    n = sn.compute_normals_device(V, F, 30.0)
    P, Fs = n.points, n.faces
    conn = Fs.reshape(-1).to(torch.int64)
    sizes = np.random.default_rng(0).integers(3, 8, conn.numel() // 3 + 1)
    offs = np.concatenate([[0], np.cumsum(sizes)])
    offs = np.concatenate([offs[offs < conn.numel()], [conn.numel()]])
    strips = (torch.from_numpy(offs.astype(np.int64)).cuda(), conn)
    c = sc.clean_polydata_device(P, Fs)
    clean_ms = events(lambda: sc.clean_polydata_device(P, Fs), args.reps)
    t = sc.triangle_filter_device(P, None, strips)
    tri_ms = events(lambda: sc.triangle_filter_device(P, None, strips), args.reps)

    p, f = P.cpu().numpy(), Fs.cpu().numpy()
    s = tuple(x.cpu().numpy() for x in strips)
    t0 = time.perf_counter()
    wc = oc.clean_polydata(p, f)
    clean_cpu = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    wt = oc.triangle_filter(p, None, s)
    tri_cpu = (time.perf_counter() - t0) * 1e3
    same = bool(np.array_equal(c.points.cpu().numpy().view(np.uint32), wc["points"].view(np.uint32)) and
                np.array_equal(c.polys.cpu().numpy().reshape(-1), wc["polys"][1]) and
                np.array_equal(c.cell_ids.cpu().numpy(), wc["cell_ids"]) and
                np.array_equal(t.faces.cpu().numpy(), wt["faces"]) and
                np.array_equal(t.cell_ids.cpu().numpy(), wt["cell_ids"]))
    res = {"metric": "clean_triangle_filter_512_bone", "gpu": name, "power_limit": plim, "reps": args.reps,
           "V": int(P.shape[0]), "T": int(Fs.shape[0]), "V_out": int(c.points.shape[0]), "strips": len(offs) - 1,
           "strip_triangles": int(t.faces.shape[0]),
           "clean_device_ms": round(clean_ms, 3), "clean_oracle_cpu_ms": round(clean_cpu, 0),
           "triangle_filter_device_ms": round(tri_ms, 3), "triangle_filter_oracle_cpu_ms": round(tri_cpu, 0),
           "verified": same}
    print(json.dumps(res))
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
