"""Timings of the region growing tool (invesalius3_b200.region_grow) at 512^3, printed as one JSON line.

Input: phantom.ct((512,)*3, seed=2), WW/WL 406 / -18, a seed at the volume's centre (inside the skull),
26-connectivity, 3 confidence iterations at multiplier 2.5 (the tool's defaults).

Reports device times from CUDA events over warmed repeats (median per call) for the LUT, one moments
call over the bone voxels and a whole confidence click; wall times of the numpy API and of a resident
RegionGrower; the wall time of today's path (the reference's NumPy statements of do_rg_confidence
around the existing floodfill_threshold binding, which ships the image over PCIe on every flood);
and whether every result equals the NumPy restatement of tests/test_region_grow_model.py.
Run: python tools/bench_region_grow.py [--reps N]"""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))
import oracle  # noqa: E402
from bench_mask_editor import card, events, wall  # noqa: E402
from invesalius3_b200 import invesalius_rs, phantom, region_grow as rg  # noqa: E402
from test_region_grow_model import image_density, lut255, rg_confidence, structure  # noqa: E402

SHAPE, WW, WL, SEED, ITERS, MULT = (512, 512, 512), 406, -18, (256, 256, 256), 3, 2.5


def todays_path(image, mask, p, bstruct):
    """do_rg_confidence's statements (styles.py:3220-3251) with use_ww_wl, the flood bound to the
    existing numpy binding."""
    x, y, z = p
    image = lut255(image, WW, WL)
    bool_mask = np.zeros_like(mask, dtype="bool")
    out_mask = np.zeros_like(mask)
    bool_mask[z - 1: z + 2, y - 1: y + 2, x - 1: x + 2] = True
    for _ in range(ITERS):
        var = np.std(image[bool_mask])
        mean = np.mean(image[bool_mask])
        t0, t1 = mean - var * MULT, mean + var * MULT
        invesalius_rs.floodfill_threshold(image, ((x, y, z),), t0, t1, 1, bstruct, out_mask)
        bool_mask[out_mask == 1] = True
    return out_mask


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, plim = card()
    vol = phantom.ct(SHAPE, seed=2)
    st = structure(26)
    mask = np.zeros(SHAPE, np.uint8)
    res = {"metric": "region_grow_512", "gpu": name, "power_limit": plim, "shape": SHAPE, "ww": WW, "wl": WL,
           "seed_xyz": SEED, "connectivity": 26, "confid_iters": ITERS, "confid_mult": MULT}
    checks = {}

    # ---- device (CUDA events)
    t = torch.from_numpy(vol).cuda()
    lut_t = rg.lut255_device(t, WW, WL)
    bone = torch.from_numpy(np.where(vol > 226, 255, 0).astype(np.uint8)).cuda()
    ws = torch.empty(rg._lib.load().b2v_masked_moments_workspace_bytes(*SHAPE), dtype=torch.uint8, device="cuda")
    out_t = torch.zeros(SHAPE, dtype=torch.uint8, device="cuda")
    dev_ms = {
        "lut255": events(lambda: rg.lut255_device(t, WW, WL, lut_t), args.reps),
        "masked_moments_bone": events(lambda: rg.masked_moments_device(t, bone, "gt127", workspace=ws), args.reps),
        "confidence_click": events(lambda: rg.confidence_grow_device(lut_t, SEED, st, ITERS, MULT, out_t, workspace=ws),
                                   args.reps),
    }
    res["device_ms"] = {k: round(v, 4) for k, v in dev_ms.items()}
    res["bone_voxels"] = int((vol > 226).sum())
    res["grown_voxels"] = int(out_t.sum().item())
    res["lut255_hbm_share_of_datasheet"] = round(vol.nbytes * 2 / (dev_ms["lut255"] * 1e-3) / 3.35e12, 3)

    # ---- wall clock
    grower = rg.RegionGrower(vol)
    api_ms = {
        "get_LUT_value_255": wall(lambda: rg.get_LUT_value_255(vol, WW, WL), max(3, args.reps // 2)),
        "do_rg_confidence": wall(lambda: rg.do_rg_confidence(vol, mask, SEED, st, ITERS, MULT, True, WW, WL),
                                 max(3, args.reps // 2)),
        "region_grower_confidence": wall(lambda: grower.confidence(SEED, st, ITERS, MULT, True, WW, WL), args.reps),
        "calc_image_density": wall(lambda: rg.calc_image_density(vol, mask), max(3, args.reps // 2)),
    }
    res["numpy_api_wall_ms"] = {k: round(v, 2) for k, v in api_ms.items()}
    t0 = time.perf_counter(); todays = todays_path(vol, mask, SEED, st); t1 = time.perf_counter()
    t2 = time.perf_counter(); want_lut = lut255(vol, WW, WL); t3 = time.perf_counter()
    res["todays_path_wall_ms"] = {"do_rg_confidence": round((t1 - t0) * 1e3, 1),
                                  "get_LUT_value_255_numpy": round((t3 - t2) * 1e3, 1)}

    # ---- checks against the NumPy restatement
    th_w, th_g = [], []
    want = rg_confidence(oracle, vol, SEED, st, ITERS, MULT, True, WW, WL, thresholds=th_w)
    got = grower.confidence(SEED, st, ITERS, MULT, True, WW, WL, thresholds=th_g)
    checks["lut255"] = bool(np.array_equal(rg.get_LUT_value_255(vol, WW, WL), want_lut))
    checks["confidence_thresholds"] = th_g == th_w
    checks["confidence_mask"] = bool(np.array_equal(got, want))
    checks["numpy_api_mask"] = bool(np.array_equal(rg.do_rg_confidence(vol, mask, SEED, st, ITERS, MULT, True, WW, WL),
                                                   want))
    checks["todays_path_mask"] = bool(np.array_equal(todays, want))
    checks["device_click_mask"] = bool(np.array_equal(out_t.cpu().numpy(), want))
    body = np.where(vol > 226, 255, 0).astype(np.uint8)
    checks["calc_image_density"] = rg.calc_image_density(vol, body) == image_density(vol, body)
    m = rg.masked_moments_device(t, bone, "gt127", workspace=ws)
    v = vol[body > 127]
    checks["masked_moments_bone"] = (m.mean, m.std) == (np.mean(v), np.std(v))
    res["thresholds"] = [[float(a), float(b)] for a, b in th_w]
    res["checks"] = checks
    res["verified"] = all(checks.values())
    print(json.dumps(res))
    return 0 if res["verified"] else 1


if __name__ == "__main__":
    sys.exit(main())
