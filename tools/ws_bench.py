"""BASELINE config 4: 512^3 watershed with 8 seed markers (4 foreground, 4 background balls
of radius 4), ww=406 / wl=-18, mg_size 3, 6-connectivity, both algorithms. Device-resident
timing (CUDA events) + agreement with the CPU checker on a 128^3 crop-sized phantom."""
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from scipy.ndimage import generate_binary_structure  # noqa: E402

from invesalius3_b200 import phantom, watershed_process as wp  # noqa: E402


def markers_for(vol, seed):
    rng = np.random.default_rng(seed)
    m = np.zeros(vol.shape, np.uint8)
    zz, yy, xx = np.ogrid[:vol.shape[0], :vol.shape[1], :vol.shape[2]]
    ins = np.argwhere(vol > 600)
    outs = np.argwhere(vol < -900)
    for lab, pool in ((1, ins), (2, outs)):
        for _ in range(4):
            c = pool[rng.integers(len(pool))]
            m[(zz - c[0]) ** 2 + (yy - c[1]) ** 2 + (xx - c[2]) ** 2 <= 16] = lab
    return m


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 512
    vol = phantom.ct((n, n, n), seed=4)
    mk = markers_for(vol, 4)
    st = generate_binary_structure(3, 1)
    t_vol, t_mk = torch.from_numpy(vol).cuda(), torch.from_numpy(mk).cuda()
    res = {}
    for alg in ("Watershed", "Watershed IFT"):
        wp.watershed_device(t_vol, t_mk, st, alg, 3, True, -18, 406)
        ts = []
        for _ in range(3):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            lab = wp.watershed_device(t_vol, t_mk, st, alg, 3, True, -18, 406)
            b.record(); torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        res[alg] = {"ms": min(ts), "Mvoxel/s": vol.size / min(ts) / 1e3,
                    "labels": {int(k): int(v) for k, v in zip(*np.unique(lab.cpu().numpy(), return_counts=True))}}
    # CPU checker on a bounded sample (SciPy IFT ~5 Mvox/s): 128^3
    from oracle import watershed as W
    m = 128
    v2 = phantom.ct((m, m, m), seed=4)
    mk2 = markers_for(v2, 4)
    for alg in ("Watershed", "Watershed IFT"):
        t0 = time.perf_counter()
        want = W.do_watershed_array(v2, mk2, st, alg, 3, True, -18, 406)
        cpu_s = time.perf_counter() - t0
        got = wp.watershed_device(torch.from_numpy(v2).cuda(), torch.from_numpy(mk2).cuda(), st, alg, 3, True, -18,
                                  406).cpu().numpy()
        res[alg].update(cpu_128_Mvoxel_s=v2.size / cpu_s / 1e6, agreement_128=float((got == want).mean()))
    print(json.dumps(res, indent=1))
    Path("bench_out").mkdir(exist_ok=True)
    json.dump(res, open(f"bench_out/ws_bench_{n}.json", "w"), indent=1)


if __name__ == "__main__":
    main()
