"""Timings of the "Remove tiny objects" plugin on the device (invesalius3_b200.tiny_objects) at 512^3, printed as one
JSON line.

Input: the bone mask (226 <= v <= 3071 -> 255) of phantom.ct((512,)*3, seed=2) in the padded layout of mask.matrix
(513^3 uint8, flags 1 in the column x = 0), and min_size 10, the plugin's initial value.

Device, from CUDA events over warmed repeats (median): the labelling (label_device), the size table
(region_sizes_device, 4 B read per voxel), one preview into a resident buffer (4 B read + 1 B written) and one
removal on a resident padded mask (4 B read + at most 1 B written). Their algorithmic bytes are set against the
3.35 TB/s HBM3 data sheet. Wall times (host clock around calls that end in a synchronise): TinyObjects(mask)
(upload, label, size table), preview(10, out) (launch + the 128 MB download) and remove(mask, 10) (upload, launch,
download). A size table over random int32 labels (every value different from its neighbours, the case the
run aggregation does not help) is timed too.
Host: the plugin's own flow once: nd.label, count_regions restated as np.bincount(labels)[labels], the preview
`(counts <= 10) * 255` into a uint8 array and `m[preview > 127] = 1`. Both results are compared byte for byte.
Run: python tools/bench_tiny_objects.py [--reps N]"""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch
from scipy import ndimage

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
from bench_mask_editor import HBM_TBPS, card, events, wall  # noqa: E402
from invesalius3_b200 import _lib, device as dev, labeling, phantom  # noqa: E402
from invesalius3_b200.device import _p, _stream  # noqa: E402
from invesalius3_b200.tiny_objects import TinyObjects  # noqa: E402

SHAPE = (512, 512, 512)
MIN_SIZE = 10


def host_once(fn):
    t0 = time.perf_counter()
    r = fn()
    return r, round((time.perf_counter() - t0) * 1e3, 1)


def share(nbytes, ms):
    return round(nbytes / (ms * 1e-3) / (HBM_TBPS * 1e12), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, plim = card()
    vol = phantom.ct(SHAPE, seed=2)
    mask = np.zeros(tuple(s + 1 for s in SHAPE), np.uint8)
    mask[1:, 1:, 1:] = np.where((vol >= 226) & (vol <= 3071), 255, 0)
    mask[1:, 0, 0] = 1
    del vol
    nvox = int(np.prod(SHAPE))
    res = {"metric": "tiny_objects_512", "gpu": name, "power_limit": plim, "shape": SHAPE, "min_size": MIN_SIZE}

    # device
    body = dev.to_device(mask[1:, 1:, 1:])
    t = TinyObjects(mask)
    n = t.num_labels
    out = torch.empty(SHAPE, dtype=torch.uint8, device="cuda")
    pad = dev.to_device(mask)
    dz, dy, dx = SHAPE

    def remove_kernel():
        _lib.call("b2v_tiny_objects_remove", _p(t.labels), dz, dy, dx, _p(t.sizes), t.sizes.numel(), MIN_SIZE, _p(pad),
                  _stream())

    dev_ms = {
        "label": events(lambda: labeling.label_device(body, None), args.reps),
        "size_table": events(lambda: labeling.region_sizes_device(t.labels, n), args.reps),
        "preview": events(lambda: t.preview_device(MIN_SIZE, out), args.reps),
        "remove": events(remove_kernel, args.reps),
    }
    noise = torch.randint(0, 1 << 20, SHAPE, dtype=torch.int32, device="cuda")
    dev_ms["size_table_random_labels"] = events(lambda: labeling.region_sizes_device(noise, (1 << 20) - 1), args.reps)
    del noise
    res["labels"] = n
    res["device_ms"] = {k: round(v, 3) for k, v in dev_ms.items()}
    res["share_of_hbm_peak"] = {"size_table": share(4 * nvox, dev_ms["size_table"]),
                                "preview": share(5 * nvox, dev_ms["preview"]),
                                "remove": share(4 * nvox, dev_ms["remove"])}
    prev = np.empty(SHAPE, np.uint8)
    scratch = mask.copy()
    res["wall_ms"] = {
        "open (upload + label + size table)": round(wall(lambda: t.refresh(mask), max(3, args.reps // 3)), 1),
        "preview + download": round(wall(lambda: t.preview(MIN_SIZE, out=prev), args.reps), 1),
        "remove (upload + launch + download)": round(
            wall(lambda: t.remove(scratch, MIN_SIZE), max(3, args.reps // 3), before=lambda: np.copyto(scratch, mask)), 1),
    }

    # host: the plugin's flow
    (labels, nh), ms_label = host_once(lambda: ndimage.label(mask[1:, 1:, 1:]))
    counts, ms_count = host_once(lambda: np.bincount(labels.ravel(), minlength=nh + 1).astype(np.uint32)[labels])
    host_prev = np.empty(SHAPE, np.uint8)

    def host_preview():
        host_prev[:] = (counts <= MIN_SIZE) * 255
    _, ms_prev = host_once(host_preview)
    host_mask = mask.copy()

    def host_remove():
        m = host_mask[1:, 1:, 1:]
        m[host_prev > 127] = 1
    _, ms_rem = host_once(host_remove)
    res["host_ms"] = {"label": ms_label, "count_regions": ms_count, "preview": ms_prev, "remove": ms_rem}

    dev_mask = mask.copy()
    t.remove(dev_mask, MIN_SIZE)
    res["equal"] = {"num_labels": n == nh, "preview": bool(np.array_equal(prev, host_prev)),
                    "mask": bool(np.array_equal(dev_mask, host_mask))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
