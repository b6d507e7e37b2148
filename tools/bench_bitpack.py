"""The bit-volume packer of flood fill and marching cubes (csrc/bitpack.cuh), timed against another build of
libb2v.so loaded in the same process, printed as one JSON line per workload.

At 512^3 (phantom.ct, seed 2, and its 0/255 bone mask) it times, with CUDA events around each call:
  - the flood's pack: b2v_floodfill_threshold_staged with stage BEGIN only (the control-region clear, the
    pack and no seeds), for int16 data with `out` at dx 512 (rows a multiple of 32) and dx 504 (padded rows),
    and for the uint8 mask with the range [255, 255];
  - b2v_mc_count on the uint8 mask (iso 127.5) and on the int16 data (iso 226), each including its
    classify, scan and synchronise.
The two libraries alternate call by call. Each of --rounds rounds takes the median of --reps calls per
library; the spread is the range of those medians over the rounds, so a difference between the libraries
can be set against the difference between repeats of one. The packed words (flood) and the counts and
inside bits (marching cubes) of the two libraries are compared. The card name and power limit are read in
the same run.
Run: python tools/bench_bitpack.py --other path/to/libb2v.so [--reps N] [--rounds R]"""
import argparse
import ctypes as C
import json
import sys
from pathlib import Path

import numpy as np
import torch
from scipy.ndimage import generate_binary_structure

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
from bench_mask_editor import card  # noqa: E402
from invesalius3_b200 import _lib, device as dev, phantom  # noqa: E402

N = 512
P, I64, F64 = C.c_void_p, C.c_int64, C.c_double
STRCT = np.ascontiguousarray(generate_binary_structure(3, 1), np.uint8)   # any element: BEGIN only packs


def load(path):
    lib = C.CDLL(str(path))
    lib.b2v_floodfill_workspace_bytes.restype = I64
    lib.b2v_floodfill_workspace_bytes.argtypes = [I64] * 4
    lib.b2v_floodfill_layout.argtypes = [I64] * 4 + [P]
    lib.b2v_floodfill_threshold_staged.argtypes = [C.c_int, P, C.c_int, I64, I64, I64, P, I64, F64, F64, C.c_uint8,
                                                   P, I64, I64, I64, P, P, P, P]
    lib.b2v_mc_workspace_bytes.restype = I64
    lib.b2v_mc_workspace_bytes.argtypes = [I64] * 3
    lib.b2v_mc_count.argtypes = [P, C.c_int, I64, I64, I64, F64, P, P, P, P]
    return lib


def flood_pack(lib, data, code, t0, t1, out, ws):
    dz, dy, dx = data.shape
    rnd = C.c_int(0)
    rc = lib.b2v_floodfill_threshold_staged(1, data.data_ptr(), code, dz, dy, dx, None, 0, t0, t1, 254,
                                            STRCT.ctypes.data, 3, 3, 3, out.data_ptr(), ws.data_ptr(),
                                            torch.cuda.current_stream().cuda_stream, C.byref(rnd))
    assert rc == 0, rc


def mc_count(lib, vol, code, iso, ws):
    nz, ny, nx = vol.shape
    nv, nt = C.c_int64(0), C.c_int64(0)
    rc = lib.b2v_mc_count(vol.data_ptr(), code, nz, ny, nx, iso, ws.data_ptr(),
                          torch.cuda.current_stream().cuda_stream, C.byref(nv), C.byref(nt))
    assert rc == 0, rc
    return nv.value, nt.value


def workloads(vol16, vol16p, mask):
    zeros = {s: torch.zeros(s, dtype=torch.uint8, device="cuda") for s in {vol16.shape, vol16p.shape}}
    return {
        "flood_pack_int16_dx512": ("flood", vol16, _lib.I16, (226.0, 3071.0), zeros[vol16.shape]),
        "flood_pack_int16_dx504": ("flood", vol16p, _lib.I16, (226.0, 3071.0), zeros[vol16p.shape]),
        "flood_pack_uint8_mask": ("flood", mask, _lib.U8, (255.0, 255.0), zeros[mask.shape]),
        "mc_count_uint8_mask": ("mc", mask, _lib.U8, 127.5, None),
        "mc_count_int16": ("mc", vol16, _lib.I16, 226.0, None),
    }


def setup(lib, kind, vol, code, arg, out):
    """The call to time, and a function that returns what it computed (bytes of the workspace, counts)."""
    dz, dy, dx = vol.shape
    nwords = dz * dy * ((dx + 31) // 32)
    if kind == "flood":
        ws = torch.empty(lib.b2v_floodfill_workspace_bytes(dz, dy, dx, 0), dtype=torch.uint8, device="cuda")
        lay = (I64 * 8)()
        assert lib.b2v_floodfill_layout(dz, dy, dx, 0, lay) == 0
        fn = lambda: flood_pack(lib, vol, code, *arg, out, ws)  # noqa: E731
        res = lambda: (ws[lay[0]:lay[0] + nwords * 4].cpu().numpy(), ws[lay[1]:lay[1] + nwords * 4].cpu().numpy())  # noqa: E731
        return fn, res
    ws = torch.empty(lib.b2v_mc_workspace_bytes(dz, dy, dx), dtype=torch.uint8, device="cuda")
    counts = {}
    fn = lambda: counts.update(c=mc_count(lib, vol, code, arg, ws))  # noqa: E731
    res = lambda: (counts["c"], ws[:nwords * 4].cpu().numpy())  # noqa: E731
    return fn, res


def same(a, b):
    if isinstance(a, tuple):
        return all(same(x, y) for x, y in zip(a, b))
    return bool(np.array_equal(a, b)) if isinstance(a, np.ndarray) else a == b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", required=True, help="the libb2v.so to compare with")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dev.require_cuda()
    libs = {"this": load(_lib.LIB_PATH), "other": load(Path(args.other).resolve())}
    vol16 = torch.from_numpy(phantom.ct((N, N, N), seed=2)).cuda()
    vol16p = vol16[:, :, :N - 8].contiguous()
    mask = dev.threshold(vol16, 226, 3071)
    name, plim = card()
    for wname, (kind, vol, code, arg, out) in workloads(vol16, vol16p, mask).items():
        calls = {k: setup(lib, kind, vol, code, arg, out) for k, lib in libs.items()}
        results = {}
        for k, (fn, res) in calls.items():
            fn()
            torch.cuda.synchronize()
            results[k] = res()
        for _ in range(2):
            for fn, _ in calls.values():
                fn()
        medians = {k: [] for k in calls}
        for _ in range(args.rounds):
            times = {k: [] for k in calls}
            for _ in range(args.reps):
                for k, (fn, _) in calls.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(); fn(); e1.record()
                    e1.synchronize()
                    times[k].append(e0.elapsed_time(e1))
            for k in calls:
                medians[k].append(float(np.median(times[k])))
        rec = {"workload": wname, "shape": list(vol.shape), "card": name, "power_limit": plim,
               "same_output": same(results["this"], results["other"])}
        for k in calls:
            m = medians[k]
            rec[k] = {"ms_median": round(float(np.median(m)), 4), "ms_spread": round(max(m) - min(m), 4),
                      "ms_rounds": [round(x, 4) for x in m]}
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
