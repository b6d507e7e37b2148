"""Timings of the surface connectivity tools on the device (invesalius3_b200.surface_connectivity), printed as
one JSON line.

Inputs: (1) the bone surface of phantom.ct((512,)*3, seed=2) thresholded at (226, 3071), contoured by
mesh.marching_cubes at iso 127 (few, large regions); (2) the surface of a 160^3 noise mask (each voxel set
with probability 0.03, numpy seed 5), about 10^5 fragments. Both stay on the device. For each: V, T, the
region count, the deepest region's wave count, the median device time of each tool from CUDA events over
warmed repeats (each call synchronises once for its counts; the split also copies the region offsets to the
host), the C checker's time once (one host core, sequential), and whether the device state and the largest
part equal the checker's. The card name and power limit are read in the same run.
Run: python tools/bench_connectivity.py [--reps N]"""
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
from connectivity_meshes import noise_volume  # noqa: E402
from invesalius3_b200 import device as dev, phantom, surface_connectivity as sc  # noqa: E402
from invesalius3_b200.mesh import marching_cubes  # noqa: E402
from oracle import connectivity as oc  # noqa: E402


def measure(label, V, F, reps):
    seeds = [int(F[0, 0])]
    c = sc.connectivity_device(V, F)
    res = {"input": label, "V": int(V.shape[0]), "T": int(F.shape[0]), "regions": int(c.sizes.shape[0]),
           "max_wave_depth": c.depth}
    res["largest_ms"] = round(events(lambda: sc.select_largest_part_device(V, F), reps), 3)
    res["split_ms"] = round(events(lambda: sc.split_disconnected_parts_device(V, F), max(2, reps // 4)), 3)
    res["seeds_ms"] = round(events(lambda: sc.join_seeds_parts_device(V, F, seeds), reps), 3)
    v, f = V.cpu().numpy(), F.cpu().numpy()
    t0 = time.perf_counter()
    st = oc.traverse(len(v), f)
    res["oracle_cpu_ms"] = round((time.perf_counter() - t0) * 1e3, 0)
    wv, wf, wp, wc = oc.select_largest_part(v, f)
    gv, gf, gp, gc = (t.cpu().numpy() for t in sc.select_largest_part_device(V, F))
    res["verified"] = bool(np.array_equal(c.region.cpu().numpy(), st["region"]) and
                           np.array_equal(c.point_map.cpu().numpy(), st["point_map"]) and
                           np.array_equal(c.sizes.cpu().numpy(), st["sizes"]) and c.depth == st["depth"] and
                           np.array_equal(gv.view(np.uint32), wv.view(np.uint32)) and np.array_equal(gf, wf) and
                           np.array_equal(gp, wp) and np.array_equal(gc, wc))
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
    bone = measure("phantom_512_bone", V, F, args.reps)
    del V, F
    V, F = marching_cubes(torch.from_numpy(noise_volume(160, 0.03, 5)).cuda(), 127, (1.0, 1.0, 1.0), (0, 0, 0), True)
    noise = measure("noise_160_p0.03", V, F, args.reps)
    res = {"metric": "surface_connectivity", "gpu": name, "power_limit": plim, "results": [bone, noise],
           "verified": bone["verified"] and noise["verified"]}
    print(json.dumps(res))
    return 0 if res["verified"] else 1


if __name__ == "__main__":
    sys.exit(main())
