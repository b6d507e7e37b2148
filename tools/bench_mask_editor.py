"""Timings of the 3-D mask editor (invesalius3_b200.mask_editor) at 512^3, printed as one JSON line.

Inputs: the bone mask (226..3071) of phantom.ct((512,)*3, seed=2) at 0.5 mm spacing, a perspective
camera that sees the whole volume in a 1280x800 viewport, a 40-vertex polygon covering about a quarter
of the viewport, and a 30 mm brush (InVesalius' BRUSH_SIZE; radius 15 mm) at the volume's centre.

Reports device times from CUDA events over warmed repeats (median per call), wall times through the
numpy API, the single-threaded C restatement's time on the host cores (the crate itself runs on rayon
threads: this is not the reference's time), and whether every device result equals the restatement.
Run: python tools/bench_mask_editor.py [--reps N]"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import editor as oracle  # noqa: E402
from invesalius3_b200 import mask_editor as me, phantom  # noqa: E402

SHAPE, SP, VP = (512, 512, 512), (0.5, 0.5, 0.5), (1280, 800)
HBM_TBPS = 3.35          # H100 SXM data-sheet HBM3 bandwidth


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        name, plim = (s.strip() for s in r.stdout.splitlines()[0].split(","))
        return name, plim
    except Exception:
        return torch.cuda.get_device_name(0), "not measured"


def camera(w, h):
    """Look-at from a fixed oblique direction at a distance where a 30-degree frustum holds the
    volume's bounding sphere, VTK-style projection, then the editor's inv_Y flip."""
    dz, dy, dx = SHAPE
    centre = np.array([dx * SP[0], -dy * SP[1], dz * SP[2]]) / 2
    radius = np.linalg.norm(centre)
    d = np.array([0.4, -0.5, 0.77]); d /= np.linalg.norm(d)
    fovy = 30.0
    dist = 1.05 * radius / np.sin(np.radians(fovy / 2) * min(1.0, w / h))
    eye = centre + d * dist
    f = (centre - eye) / dist
    s = np.cross(f, [0.0, 0.0, 1.0]); s /= np.linalg.norm(s)
    u = np.cross(s, f)
    V = np.eye(4)
    V[0, :3], V[1, :3], V[2, :3] = s, u, -f
    V[:3, 3] = -V[:3, :3] @ eye
    near, far = dist - radius, dist + radius
    P = np.zeros((4, 4))
    ff = 1.0 / np.tan(np.radians(fovy) / 2)
    P[0, 0], P[1, 1] = ff / (w / h), ff
    P[2, 2], P[2, 3], P[3, 2] = (far + near) / (near - far), 2 * far * near / (near - far), -1.0
    inv_y = np.eye(4); inv_y[1, 1] = -1
    return np.ascontiguousarray(P @ V @ inv_y), np.ascontiguousarray(V @ inv_y), near, far


def polygon(w, h, n=40, seed=4):
    """A star-shaped polygon with area ~ w h / 4, centred a quarter of the way across the viewport so
    that it covers part of the bone (which projects about the viewport's centre), not all of it."""
    rng = np.random.default_rng(seed)
    a = np.sort(rng.uniform(0, 2 * np.pi, n))
    r = 0.28 * rng.uniform(0.85, 1.15, n)
    return np.stack([w / 4 + r * w * np.cos(a), h / 2 + r * h * np.sin(a)], axis=1)


def events(fn, reps, before=None):
    """Median device time (ms) of fn() over `reps` warmed calls; before() runs outside the window."""
    for _ in range(2):
        if before:
            before()
        fn()
    times = []
    for _ in range(reps):
        if before:
            before()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(np.median(times))


def wall(fn, reps, before=None):
    for _ in range(2):
        if before:
            before()
        fn()
    times = []
    for _ in range(reps):
        if before:
            before()
        torch.cuda.synchronize()
        t0 = time.perf_counter(); fn(); t1 = time.perf_counter()
        times.append((t1 - t0) * 1e3)
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, plim = card()
    w, h = VP
    vol = phantom.ct(SHAPE, seed=2)
    mask = np.where((vol >= 226) & (vol <= 3071), 255, 0).astype(np.uint8)
    M, MV, near, far = camera(w, h)
    poly = polygon(w, h)
    centre = tuple(np.array(SHAPE[::-1]) * np.array(SP) / 2)
    radius = 15.0
    res = {"metric": "mask_editor_512", "gpu": name, "power_limit": plim, "shape": SHAPE, "spacing": SP,
           "viewport": VP, "polygon_vertices": len(poly), "brush_radius_mm": radius,
           "selected_voxels": int((mask > 127).sum())}
    checks = {}

    # ---- device kernels (CUDA events)
    dev_ms = {}
    dev_ms["polygon2mask_device"] = events(lambda: me.polygon2mask_device((w, h), poly), args.reps)
    filt_excl = me.polygon2mask_device((w, h), poly).T.contiguous()
    filt_incl = 1 - filt_excl
    pristine = torch.from_numpy(mask).cuda()
    t = torch.empty_like(pristine)
    restore = lambda: t.copy_(pristine)                                        # noqa: E731
    for mode, f in ((0, filt_incl), (1, filt_excl)):
        dev_ms[f"mask_cut_device_mode{mode}"] = events(lambda: me.mask_cut_device(t, SP, far, f, M, MV, mode), args.reps,
                                                       restore)
    zeros, full = torch.zeros_like(pristine), torch.full_like(pristine, 255)
    dev_ms["mask_cut_device_empty_mask"] = events(lambda: me.mask_cut_device(zeros, SP, far, filt_excl, M, MV, 1),
                                                  args.reps)
    dev_ms["mask_cut_device_full_mask"] = events(lambda: me.mask_cut_device(t, SP, far, filt_excl, M, MV, 1), args.reps,
                                                 lambda: t.copy_(full))
    for mode in (0, 1):
        dev_ms[f"brush_mask_device_mode{mode}"] = events(
            lambda: me.brush_mask_device(t, None, SP, centre, radius, mode), args.reps, restore)
    res["device_ms"] = {k: round(v, 4) for k, v in dev_ms.items()}
    n = mask.size
    res["mask_cut_hbm_share_of_datasheet"] = {
        k: round(n / (dev_ms[k] * 1e-3) / (HBM_TBPS * 1e12), 3) for k in ("mask_cut_device_empty_mask",
                                                                          "mask_cut_device_mode1")}

    # ---- numpy API (wall clock), the editor's padded [1:, 1:, 1:] view
    padded = np.zeros(tuple(s + 1 for s in SHAPE), np.uint8)
    view = padded[1:, 1:, 1:]
    reset = lambda: view.__setitem__(Ellipsis, mask)                           # noqa: E731
    filt_np = {1: me.polygon2mask_rs((w, h), poly).T}
    filt_np[0] = np.logical_not(filt_np[1])
    api_ms = {}
    for mode in (0, 1):
        api_ms[f"mask_cut_mode{mode}"] = wall(lambda: me.mask_cut(vol, *SP, far, filt_np[mode], M, MV, view, mode),
                                              max(3, args.reps // 4), reset)
    api_ms["brush_mask_rs_mode1"] = wall(lambda: me.brush_mask_rs(view, None, SP, centre, radius, 1), args.reps, reset)
    api_ms["polygon2mask_rs"] = wall(lambda: me.polygon2mask_rs((w, h), poly), args.reps)
    res["numpy_api_wall_ms"] = {k: round(v, 3) for k, v in api_ms.items()}

    # ---- C restatement, one host thread, and the checks
    ref_ms = {}
    t0 = time.perf_counter(); want_poly = oracle.polygon2mask_rs((w, h), poly); ref_ms["polygon2mask"] = time.perf_counter() - t0
    checks["polygon2mask"] = bool(np.array_equal(me.polygon2mask_rs((w, h), poly), want_poly))
    for mode in (0, 1):
        want = mask.copy()
        t0 = time.perf_counter()
        oracle.mask_cut(vol, *SP, far, filt_np[mode], M, MV, want, mode)
        ref_ms[f"mask_cut_mode{mode}"] = time.perf_counter() - t0
        reset()
        me.mask_cut(vol, *SP, far, filt_np[mode], M, MV, view, mode)
        checks[f"mask_cut_mode{mode}"] = bool(np.array_equal(view, want))
        checks[f"mask_cut_mode{mode}_changed_voxels"] = int((want != mask).sum())
        t.copy_(pristine)
        me.mask_cut_device(t, SP, far, filt_incl if mode == 0 else filt_excl, M, MV, mode)
        checks[f"mask_cut_device_mode{mode}"] = bool(np.array_equal(t.cpu().numpy(), want))
    for mode in (0, 1):
        want = mask.copy()
        t0 = time.perf_counter()
        oracle.brush_mask_rs(want, None, SP, centre, radius, mode)
        ref_ms[f"brush_mode{mode}"] = time.perf_counter() - t0
        reset()
        me.brush_mask_rs(view, None, SP, centre, radius, mode)
        checks[f"brush_mode{mode}"] = bool(np.array_equal(view, want))
        checks[f"brush_mode{mode}_changed_voxels"] = int((want != mask).sum())
    res["restatement_single_thread_host_ms"] = {k: round(v * 1e3, 1) for k, v in ref_ms.items()}
    res["checks"] = checks
    res["verified"] = all(v for k, v in checks.items() if not k.endswith("_voxels"))
    print(json.dumps(res))
    return 0 if res["verified"] else 1


if __name__ == "__main__":
    sys.exit(main())
