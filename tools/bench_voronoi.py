"""Timings of jump flooding and the porous-scaffold Voronoi generator (invesalius3_b200.voronoi), printed as
one JSON line.

Cases: jump_flooding_device on zeroed volumes at 256^3 with 1000 random sites (the tool's default) and 512^3
with 5000, normalize off; the numpy-in, numpy-out jump_flooding at 256^3; a whole create_voronoi() (256^3,
1000 sites, borders, float32 gaussian) and image_normalize(-1000, 1000) after it, as gui.py:199, 237 run.

Reports, per case: the device time from CUDA events over warmed repeats (median), the two byte counts per
Jacobi step (compulsory: owner and distance read and written, 16 B per voxel; gathered: 26 neighbour owners,
104 B per voxel) and the compulsory bytes over the device time against the 3.35 TB/s HBM3 data sheet; wall
times of the numpy API; and, on the host of the same run, the threaded C checker (oracle/voronoi.c with
every core) plus NumPy's gradient and SciPy's gaussian_filter (the crate itself is not built here). Every
device output is compared with the checker's in the same run.
Run: python tools/bench_voronoi.py [--reps N]"""
import argparse
import json
import os
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
from bench_mask_editor import card, events, wall  # noqa: E402
from invesalius3_b200 import voronoi  # noqa: E402
from oracle import voronoi as ov  # noqa: E402

COMPULSORY_B, GATHERED_B = 16, 26 * 4


def n_steps(shape) -> int:
    return max(shape).bit_length() - 1


def host(fn):
    t0 = time.perf_counter()
    r = fn()
    return r, (time.perf_counter() - t0) * 1e3


def jfa_case(shape, n_sites, reps, seed):
    sites = np.random.default_rng(seed).integers((0, 0, 0), shape, size=(n_sites, 3)).astype(np.int32)
    s = torch.from_numpy(sites).cuda()
    dist = torch.zeros(shape, dtype=torch.float32, device="cuda")
    own = torch.zeros(shape, dtype=torch.int32, device="cuda")

    def reset():
        dist.zero_()
        own.zero_()

    ms = events(lambda: voronoi.jump_flooding_device(dist, own, s, False), reps, before=reset)
    reset()
    voronoi.jump_flooding_device(dist, own, s, False)
    ref_d, ref_o = np.zeros(shape, np.float32), np.zeros(shape, np.int32)
    _, checker_ms = host(lambda: ov.jump_flooding(ref_d, ref_o, sites, False))
    ok = bool(np.array_equal(dist.cpu().numpy(), ref_d) and np.array_equal(own.cpu().numpy(), ref_o))
    nvox, steps = int(np.prod(shape)), n_steps(shape)
    res = {
        "shape": list(shape), "sites": n_sites, "steps": steps, "device_ms": round(ms, 3),
        "compulsory_gb_per_step": round(nvox * COMPULSORY_B / 1e9, 3),
        "gathered_gb_per_step": round(nvox * GATHERED_B / 1e9, 3),
        "compulsory_hbm_share_of_datasheet": round(nvox * COMPULSORY_B * steps / (ms * 1e-3) / 3.35e12, 3),
        "checker_host_ms": round(checker_ms, 0),
    }
    return res, ok, sites, (ref_d, ref_o)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, plim = card()
    res = {"metric": "voronoi_jump_flooding", "gpu": name, "power_limit": plim, "host_cpus": os.cpu_count(),
           "cases": {}}
    checks = {}

    small = (256, 256, 256)
    r, checks["jump_flooding_device 256^3"], sites, (ref_d, ref_o) = jfa_case(small, 1000, args.reps, 1)
    d, o = np.zeros(small, np.float32), np.zeros(small, np.int32)

    def numpy_call():
        d[...] = 0
        o[...] = 0
        voronoi.jump_flooding(d, o, sites, False)

    r["numpy_api_wall_ms"] = round(wall(numpy_call, max(3, args.reps // 2)), 1)
    checks["jump_flooding numpy 256^3"] = bool(np.array_equal(d, ref_d) and np.array_equal(o, ref_o))
    res["cases"]["jump_flooding 256^3"] = r
    torch.cuda.empty_cache()

    r, checks["jump_flooding_device 512^3"], _, _ = jfa_case((512, 512, 512), 5000, max(3, args.reps // 2), 2)
    res["cases"]["jump_flooding 512^3"] = r
    torch.cuda.empty_cache()

    def seeded(fn):
        np.random.seed(99)
        return fn()

    got = seeded(voronoi.create_voronoi)
    create_ms = wall(lambda: seeded(voronoi.create_voronoi), max(3, args.reps // 2))
    norm_ms = wall(lambda: voronoi.image_normalize(got, min_=-1000, max_=1000), max(3, args.reps // 2))
    want, host_create_ms = host(lambda: seeded(ov.create_voronoi))
    want_i16, host_norm_ms = host(lambda: ov.image_normalize(want, min_=-1000, max_=1000))
    checks["create_voronoi 256^3"] = bool(np.array_equal(got, want))
    checks["image_normalize 256^3"] = bool(np.array_equal(voronoi.image_normalize(got, min_=-1000, max_=1000),
                                                          want_i16))
    res["cases"]["create_voronoi 256^3 1000 sites, borders"] = {
        "numpy_api_wall_ms": round(create_ms, 1), "image_normalize_wall_ms": round(norm_ms, 1),
        "host_checker_gradient_gaussian_ms": round(host_create_ms, 0), "host_image_normalize_ms": round(host_norm_ms, 0),
    }
    res["checks"] = checks
    res["verified"] = all(checks.values())
    print(json.dumps(res))
    return 0 if res["verified"] else 1


if __name__ == "__main__":
    sys.exit(main())
