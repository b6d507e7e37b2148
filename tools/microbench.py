"""Per-op device-timed microbenchmarks (CUDA events, L2 flush between iterations)."""
import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from invesalius3_b200 import device as dev  # noqa: E402

PEAK = 3350.0   # GB/s, HBM3 of the H100 SXM data sheet


def timeit(fn, iters=10, warmup=3, flush=None):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.add_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--ops", default="threshold,mip")
    args = ap.parse_args()
    n = args.n
    g = torch.Generator(device="cuda").manual_seed(0)
    vol = torch.randint(-1024, 3072, (n, n, n), dtype=torch.int16, device="cuda", generator=g)
    vol[0, 0, 0] = -1024; vol[0, 0, 1] = 3071
    flush = torch.zeros(256 << 20, dtype=torch.uint8, device="cuda")
    N = vol.numel()
    res = {}
    ops = args.ops.split(",")
    if "threshold" in ops:
        out = torch.empty((n, n, n), dtype=torch.uint8, device="cuda")
        med, best = timeit(lambda: dev.threshold(vol, 226, 3071, out=out), flush=flush)
        res["threshold"] = dict(ms=med, best_ms=best, gbs=3 * N / med / 1e6, frac=3 * N / med / 1e6 / PEAK)
        med, best = timeit(lambda: dev.threshold(vol, 226, 3071, out=out, preserve_markers=True), flush=flush)
        res["threshold_preserve"] = dict(ms=med, best_ms=best, gbs=4 * N / med / 1e6, frac=4 * N / med / 1e6 / PEAK)
    if "mip" in ops:
        for axis in (0, 1, 2):
            for kind in ("max", "mean"):
                o = dev.mip(vol, axis, kind)
                med, best = timeit(lambda: dev.mip(vol, axis, kind, out=o), flush=flush)
                res[f"mip_{kind}_axis{axis}"] = dict(ms=med, best_ms=best, gbs=2 * N / med / 1e6,
                                                     frac=2 * N / med / 1e6 / PEAK)
    if "mida" in ops:
        from invesalius3_b200 import projection
        for axis in (0, 1, 2):
            o = projection.mida(vol, axis, 300, 300)
            med, best = timeit(lambda: projection.mida(vol, axis, 300, 300, out=o), flush=flush)
            res[f"mida_axis{axis}_earlyexit"] = dict(ms=med, best_ms=best, gbs=4 * N / med / 1e6,
                                                     frac=4 * N / med / 1e6 / PEAK)
            # opacity 0 everywhere: no ray terminates, the whole volume is read twice (min/max + rays)
            med, best = timeit(lambda: projection.mida(vol, axis, 32000, 2, out=o), flush=flush)
            res[f"mida_axis{axis}_fullrays"] = dict(ms=med, best_ms=best, gbs=4 * N / med / 1e6,
                                                    frac=4 * N / med / 1e6 / PEAK)
            o = projection.lmip(vol, axis, 700, 3033)
            med, best = timeit(lambda: projection.lmip(vol, axis, 700, 3033, out=o), flush=flush)
            res[f"lmip_axis{axis}"] = dict(ms=med, best_ms=best, gbs=2 * N / med / 1e6, frac=2 * N / med / 1e6 / PEAK)
    if "fcm" in ops:
        from invesalius3_b200 import projection
        for axis in (0, 2):
            for tmip in (0, 2):
                o = projection.fast_countour_mip(vol, 2.0, axis, 300, 300, tmip)
                med, best = timeit(lambda: projection.fast_countour_mip(vol, 2.0, axis, 300, 300, tmip, out=o), iters=5,
                                   flush=flush)
                b = 2 if tmip == 0 else 4
                res[f"fcm_tmip{tmip}_axis{axis}"] = dict(ms=med, best_ms=best, gbs=b * N / med / 1e6,
                                                         frac=b * N / med / 1e6 / PEAK)
    if "minmax" in ops:
        med, best = timeit(lambda: dev.minmax(vol), flush=flush)
        res["minmax"] = dict(ms=med, best_ms=best, gbs=2 * N / med / 1e6, frac=2 * N / med / 1e6 / PEAK)
    for k, v in res.items():
        print(f"{k:28s} {v['ms']:8.3f} ms (best {v['best_ms']:.3f})  {v['gbs']:8.1f} GB/s  {100 * v['frac']:5.1f}% of the data-sheet {PEAK}")
    Path("bench_out").mkdir(exist_ok=True)
    json.dump(res, open(f"bench_out/microbench_{n}.json", "w"), indent=1)


if __name__ == "__main__":
    main()
