"""Timings of the geodesic measurement on the device (invesalius3_b200.surface_geodesic), printed as one JSON line.

Input: phantom.ct((512,)*3, seed=2) thresholded at (226, 3071) and contoured by mesh.marching_cubes at iso 127
without padding, kept on the device: the 512^3 phantom's bone surface. The start pick is the surface point with
the largest z; the near pick is the point whose straight-line distance from it is closest to 20 mm, the far pick
the point of its connected part with the largest geodesic distance (across the skull). Median device times
from CUDA events over warmed repeats, each call ending in a host synchronise, of:
  links       GeodesicSurface(V, F): faces, point -> cell links and the bucket width, once per surface
  closest     the closest points of two picks
  near, far   GeodesicSurface.path for the pick pair: closest points, distances with early exit, trace
  full        the whole distance field from the start (GetCumulativeWeights)
and the C checker's time once on one host core for the near pair (what the reference does per click: the graph,
a Dijkstra over the whole connected part, the trace). `verified`: the device paths and lengths equal the
checker's (an ambiguous path is checked by its end points only), and the full field equals it bit for bit. The
card name and power limit are read in the same run.
Run: python tools/bench_geodesic.py [--reps N]"""
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
from invesalius3_b200 import device as dev, phantom, surface_geodesic as sg  # noqa: E402
from invesalius3_b200.mesh import marching_cubes  # noqa: E402
from oracle import geodesic as og  # noqa: E402


def same_path(got, want):
    ok = got.ambiguous == list(want["ambiguous"]) and got.unreached == list(want["unreached"])
    for g, w, a in zip(got.ids, want["ids"], want["ambiguous"]):
        g = g.cpu().numpy()
        ok &= bool(np.array_equal(g, w) if not a else (g[0] == w[0] and g[-1] == w[-1]))
    return ok and (any(want["ambiguous"]) or got.total == want["total"])


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
    v, f = V.cpu().numpy(), F.cpu().numpy()
    s = sg.GeodesicSurface(V, F)
    start = int(np.argmax(v[:, 2]))
    full = s.distances(start)
    d = full.cpu().numpy()
    far = int(np.argmax(np.where(np.isfinite(d), d, -1.0)))
    e = np.sqrt(((v.astype(np.float64) - v[start]) ** 2).sum(1))
    near = int(np.argmin(np.where(np.isfinite(d), np.abs(e - 20.0), np.inf)))
    picks = {"near": v[[start, near]].astype(np.float64), "far": v[[start, far]].astype(np.float64)}

    res = {"metric": "geodesic", "input": "phantom_512_bone", "gpu": name, "power_limit": plim,
           "V": int(V.shape[0]), "T": int(F.shape[0])}
    res["links_ms"] = round(events(lambda: sg.GeodesicSurface(V, F), args.reps), 3)
    res["closest_ms"] = round(events(lambda: s.closest_points(picks["near"]), args.reps), 3)
    verified = True
    for k, p in picks.items():
        got = s.path(p)
        want = og.geodesic_path(v, f, p)
        s.distances(start, int(got.ids[0][0]))
        res[k] = {"ms": round(events(lambda: s.path(p), args.reps), 3), "points": int(len(got.ids[0])),
                  "length_mm": got.total, "euclidean_mm": float(e[near if k == "near" else far]),
                  "rounds": s.rounds, "buckets": s.buckets, "ambiguous": got.ambiguous[0]}
        verified &= bool(same_path(got, want))
    res["full_ms"] = round(events(lambda: s.distances(start), args.reps), 3)
    res["full_rounds"], res["full_buckets"] = s.rounds, s.buckets
    t0 = time.perf_counter()
    want = og.geodesic_path(v, f, picks["near"])
    res["checker_cpu_ms"] = round((time.perf_counter() - t0) * 1e3, 0)
    verified &= bool(np.array_equal(d.view(np.uint64), og.distances(v, f, start)["dist"].view(np.uint64)))
    res["verified"] = verified
    print(json.dumps(res))


if __name__ == "__main__":
    main()
