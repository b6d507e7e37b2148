"""Timings of the surface join on the device (surface_process.join_surface_device), one JSON line per case.

Cases: the Cranium full-size mask_0 (108 x 256 x 256, tests/golden) in AddNewActor's 6 pieces; the bone
surface of phantom.ct((512,)*3, seed=2) thresholded at (226, 3071), in 26 pieces and as one whole-volume
piece. Pieces are made by contour_piece (create_surface_piece's mesh, padded) and uploaded before timing.
Settings: "Binary" with the largest part and hole filling; "ca_smoothing" at the GUI's defaults (angle 0.7,
max distance 3.0, min weight 0.5, 10 steps) without either.

Per case: the whole join_surface_device call, and each of its module calls made one by one in the join's order
on the same pieces (whose final result must equal the join's), each the median over --reps calls after one
warm-up call, from CUDA events; every module synchronises to bring its counts to the host, so these are the
times a caller sees. Also the time to copy the result to the host and write the .vtp, the time of the
sequential checker (oracle/join.py, one host core) once, and whether the device result equals it bit for bit. The card name and power limit are read in the same run.
Run: python tools/bench_join.py [--reps N] [--no-checker]"""
import argparse
import json
import os
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
sys.path.insert(0, str(ROOT / "tests"))
from bench_mask_editor import card  # noqa: E402
from join_cases import CA_OPTIONS, padded_mask, rois  # noqa: E402
from invesalius3_b200 import device as dev, phantom, surface_process as sp  # noqa: E402
from invesalius3_b200.mesh_ops import smooth_device  # noqa: E402
from invesalius3_b200.surface_connectivity import select_largest_part_device  # noqa: E402
from invesalius3_b200.surface_holes import fill_holes_device  # noqa: E402
from invesalius3_b200.surface_normals import compute_normals_device, mass_properties_device  # noqa: E402

SETTINGS = [("Binary", True, True), ("ca_smoothing", False, False)]


def _timed(times, name, fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    e1.synchronize()
    times[name] = e0.elapsed_time(e1)
    return r


def one_join(pieces, setting):
    """(result, ms) of one join_surface_device call."""
    t = {}
    r = _timed(t, "total", lambda: sp.join_surface_device(pieces, *setting, CA_OPTIONS))
    return r, t["total"]


def staged(pieces, setting):
    """The join's module calls one by one, in its order, each timed: (final normals, {step: ms})."""
    algorithm, keep_largest, fill_holes = setting
    t = {}
    points, faces = _timed(t, "append", lambda: sp._append(pieces))
    points, faces, _, _ = _timed(t, "clean", lambda: sp._clean(points, faces))
    if algorithm == "ca_smoothing":
        n = _timed(t, "ca_normals", lambda: compute_normals_device(points, faces, 30.0, False))
        points, faces, ids, _ = _timed(t, "ca_clean", lambda: sp._clean(n.points, n.faces))
        cn = n.cell_normals[ids].contiguous()
        f4 = torch.cat((torch.full((faces.shape[0], 1), 3, dtype=torch.int64, device=faces.device), faces), 1)
        opts = [CA_OPTIONS[k] for k in ("angle", "max distance", "min weight", "steps")]
        _timed(t, "ca_smoothing", lambda: smooth_device(points, f4, cn, *opts))
    if keep_largest:
        points, faces, _, _ = _timed(t, "largest_part", lambda: select_largest_part_device(points, faces))
    if fill_holes:
        faces = _timed(t, "fill_holes", lambda: fill_holes_device(points, faces, 300.0).faces)
    _timed(t, "volume_area", lambda: mass_properties_device(points, faces))
    n = _timed(t, "final_normals", lambda: compute_normals_device(points, faces, 80.0, True))
    return n, t


def run_case(name, pieces_np, setting, reps, checker):
    pieces = [(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()) for v, f in pieces_np]
    one_join(pieces, setting)
    runs = [one_join(pieces, setting) for _ in range(reps)]
    r = runs[-1][0]
    staged(pieces, setting)
    stage_runs = [staged(pieces, setting) for _ in range(reps)]
    steps = {k: round(float(np.median([s[k] for _, s in stage_runs])), 3) for k in stage_runs[0][1]}
    n = stage_runs[-1][0]
    staged_same = all(torch.equal(a, b) for a, b in ((n.points, r.points), (n.faces, r.faces),
                                                     (n.point_normals, r.point_normals)))
    fd, fn = tempfile.mkstemp(suffix="_full.vtp")
    os.close(fd)
    t0 = time.perf_counter()
    sp.write_vtp(fn, *(t.cpu().numpy() for t in (r.points, r.faces, r.point_normals, r.cell_normals)))
    write_ms = (time.perf_counter() - t0) * 1e3
    size = os.path.getsize(fn)
    os.unlink(fn)
    res = {"metric": "join_surface", "case": name, "algorithm": setting[0], "keep_largest": setting[1],
           "fill_holes": setting[2], "pieces": len(pieces), "T_in": int(sum(len(f) for _, f in pieces_np)),
           "V_out": int(r.points.shape[0]), "T_out": int(r.faces.shape[0]), "reps": reps,
           "join_ms": round(float(np.median([ms for _, ms in runs])), 3), "step_ms": steps, "steps_equal_join": staged_same,
           "write_vtp_ms": round(write_ms, 1), "vtp_bytes": size}
    if checker:
        from oracle import join as oj
        t0 = time.perf_counter()
        w = oj.join(pieces_np, *setting, CA_OPTIONS)
        res["checker_cpu_ms"] = round((time.perf_counter() - t0) * 1e3, 0)
        res["verified"] = bool(
            all(np.array_equal(getattr(r, k).cpu().numpy(), w[k]) for k in ("points", "faces", "point_normals",
                                                                            "cell_normals"))
            and (r.volume, r.area, r.dropped_cells) == (w["volume"], w["area"], w["dropped_cells"]))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-checker", action="store_true")
    args = ap.parse_args()
    dev.require_cuda()
    torch.cuda.set_device(0)
    gpu, plim = card()

    cr = np.load(ROOT / "tests" / "golden" / "cranium_crop.npz")
    full = tuple(int(s) for s in cr["full_shape"])
    mm = padded_mask(np.unpackbits(cr["mask_0_bits_full"])[:np.prod(full)].reshape(full) * np.uint8(255))
    spacing = tuple(float(s) for s in cr["spacing"])
    cases = [("cranium_mask0_6_pieces", [sp.contour_piece(None, mm, roi, spacing, index_dtype=np.int64)
                                         for roi in rois(full[0])])]
    vol = phantom.ct((512, 512, 512), seed=2)
    mm = padded_mask(dev.threshold(torch.from_numpy(vol).cuda(), 226, 3071).cpu().numpy())
    del vol
    cases.append(("phantom512_bone_26_pieces", [sp.contour_piece(None, mm, roi, (1.0, 1.0, 1.0), index_dtype=np.int64)
                                                for roi in rois(512)]))
    cases.append(("phantom512_bone_whole", [sp.contour_piece(None, mm, slice(0, 512), (1.0, 1.0, 1.0),
                                                             index_dtype=np.int64)]))
    del mm
    ok = True
    for name, pieces in cases:
        for setting in SETTINGS:
            res = run_case(name, pieces, setting, args.reps, not args.no_checker)
            res.update(gpu=gpu, power_limit=plim)
            ok = ok and res["steps_equal_join"] and res.get("verified", True)
            print(json.dumps(res), flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
