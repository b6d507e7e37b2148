"""Timings of the surface hole filling on the device (invesalius3_b200.surface_holes), printed as one JSON line.

Inputs, all contoured by mesh.marching_cubes at iso 127 without padding and kept on the device: (1) the Cranium
bone mask of tests/golden/cranium_crop.npz; (2) phantom.ct((512,)*3, seed=2) thresholded at (226, 3071) with z
cropped to [128, 384), open where the crop cuts it; (3) connectivity_meshes.noise_volume(128, 0.5, 1), thousands
of small loops; (4) the whole 512^3 phantom's bone surface, closed. Each runs at HoleSize 1000, as
ApplySmoothFilter uses it. For each: V, T, the boundary lines, the loops and the loops filled, the longest
loop, the median device time of fill_holes_device from CUDA events over warmed repeats (the call synchronises
the host twice), the C checker's time once (one host core, sequential), and whether the device result equals
the checker's exactly. The card name and power limit are read in the same run.
Run: python tools/bench_fill_holes.py [--reps N]"""
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
from invesalius3_b200 import device as dev, phantom, surface_holes as sh  # noqa: E402
from invesalius3_b200.mesh import marching_cubes  # noqa: E402
from oracle import fill_holes as ofh  # noqa: E402
from connectivity_meshes import noise_volume  # noqa: E402

HOLE_SIZE = 1000.0


def measure(label, V, F, reps):
    r = sh.fill_holes_device(V, F, HOLE_SIZE)
    pts = r.points.cpu().numpy()
    res = {"input": label, "V": int(V.shape[0]), "T": int(F.shape[0]), "lines": r.lines, "loops": int(len(pts)),
           "filled": int((r.status.cpu().numpy() == sh.FILLED).sum()), "longest_loop": int(pts.max(initial=0))}
    res["device_ms"] = round(events(lambda: sh.fill_holes_device(V, F, HOLE_SIZE), reps), 3)
    v, f = V.cpu().numpy(), F.cpu().numpy()
    t0 = time.perf_counter()
    want = ofh.fill_holes(v, f, HOLE_SIZE)
    res["oracle_cpu_ms"] = round((time.perf_counter() - t0) * 1e3, 0)
    res["verified"] = bool(np.array_equal(r.faces.cpu().numpy(), want["faces"]) and r.lines == want["lines"]
                           and np.array_equal(r.first_line.cpu().numpy(), want["first_line"])
                           and np.array_equal(pts, want["npts"])
                           and np.array_equal(r.radius.cpu().numpy().view(np.uint64), want["radius"].view(np.uint64))
                           and np.array_equal(r.status.cpu().numpy(), want["status"]))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, plim = card()
    results = []
    cr = np.load(ROOT / "tests" / "golden" / "cranium_crop.npz")
    full = tuple(int(s) for s in cr["full_shape"])
    mask = np.unpackbits(cr["mask_0_bits_full"])[:np.prod(full)].reshape(full) * np.uint8(255)
    sx, sy, sz = (float(s) for s in cr["spacing"])
    results.append(measure("cranium", *marching_cubes(torch.from_numpy(mask).cuda(), 127, (sx, sy, sz), (0, 0, 0),
                                                      True), args.reps))
    vol = phantom.ct((512, 512, 512), seed=2)
    mask = dev.threshold(torch.from_numpy(vol).cuda(), 226, 3071)
    del vol
    results.append(measure("phantom_512_z128_384", *marching_cubes(mask[128:384].contiguous(), 127,
                                                                   (1.0, 1.0, 1.0), (0, 0, 0), True), args.reps))
    whole = marching_cubes(mask, 127, (1.0, 1.0, 1.0), (0, 0, 0), True)
    del mask
    noise = torch.from_numpy(noise_volume(128, 0.5, 1)).cuda()
    results.append(measure("noise_128", *marching_cubes(noise, 127, (1.0, 1.0, 1.0), (0, 0, 0), True), args.reps))
    results.append(measure("phantom_512_closed", *whole, args.reps))
    res = {"metric": "surface_fill_holes", "gpu": name, "power_limit": plim, "hole_size": HOLE_SIZE,
           "results": results, "verified": all(r["verified"] for r in results)}
    print(json.dumps(res))
    return 0 if res["verified"] else 1


if __name__ == "__main__":
    sys.exit(main())
