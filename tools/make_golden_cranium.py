"""Generate tests/golden/cranium_crop.npz and tests/golden/cranium_thr_matrix.npy.xz from
samples/Cranium.inv3 of an InVesalius 3 checkout:

    python tools/make_golden_cranium.py <invesalius3>/samples/Cranium.inv3

The .inv3 format is a tar of main.plist + matrix.dat + mask_N.dat/.plist
(invesalius/project.py:378-470, invesalius/data/mask.py:315-366). We keep a crop of the
int16 matrix plus the two shipped, reference-produced threshold masks (bit-packed), and
whole-volume voxel counts; and the whole matrix reduced to what thresholding at the
shipped masks' bounds can see (thr_matrix below).
"""
import io
import lzma
import plistlib
import sys
import tarfile
from pathlib import Path

import numpy as np

GOLDEN = Path(__file__).resolve().parents[1] / "tests" / "golden"
DST = GOLDEN / "cranium_crop.npz"
DST_THR = GOLDEN / "cranium_thr_matrix.npy.xz"
CROP = (slice(30, 78), slice(64, 192), slice(64, 192))  # z, y, x


def load_inv3(path):
    with tarfile.open(path, "r:*") as tf:
        files = {Path(m.name).name: tf.extractfile(m).read() for m in tf.getmembers() if m.isfile()}
    main = plistlib.loads(files["main.plist"])
    shape = tuple(main["matrix"]["shape"])
    matrix = np.frombuffer(files[main["matrix"]["filename"]], dtype=main["matrix"]["dtype"]).reshape(shape)
    masks = []
    for key in sorted(main["masks"], key=int):
        mp = plistlib.loads(files[main["masks"][key]])
        mshape = tuple(mp["mask_shape"])
        m = np.frombuffer(files[mp["mask_file"]], dtype=np.uint8).reshape(mshape)
        masks.append((tuple(mp["threshold_range"]), m))
    return main, matrix, masks


def thr_matrix(matrix, bounds):
    """The matrix with every value more than two away from a threshold edge (lo, or hi + 1, of
    each range in `bounds`) replaced by the smallest value of the matrix between the same two
    edges. Thresholding at those bounds gives the same answer on it as on the matrix, and it
    compresses to a fraction of the size."""
    edges = np.array(sorted({lo for lo, _ in bounds} | {hi + 1 for _, hi in bounds}))
    cls = np.searchsorted(edges, matrix, side="right")
    near = np.zeros(matrix.shape, bool)
    for e in edges:
        near |= (matrix >= e - 2) & (matrix <= e + 1)
    rep = np.array([matrix[cls == i].min() if (cls == i).any() else 0 for i in range(len(edges) + 1)], matrix.dtype)
    return np.where(near, matrix, rep[cls]).astype(matrix.dtype)


def main():
    src = Path(sys.argv[1])
    meta, matrix, masks = load_inv3(src)
    out = {"matrix_crop": np.ascontiguousarray(matrix[CROP]), "crop": np.array([[s.start, s.stop] for s in CROP]),
           "full_shape": np.array(matrix.shape), "spacing": np.array(meta["spacing"], dtype=np.float64)}
    for i, (thr, m) in enumerate(masks):
        body = m[1:, 1:, 1:]
        assert set(np.unique(body)) <= {0, 255}
        out[f"thr_{i}"] = np.array(thr, dtype=np.int64)
        out[f"mask_{i}_crop_bits"] = np.packbits(body[CROP] == 255)
        out[f"mask_{i}_count_full"] = np.array(int((body == 255).sum()))
        # per-slice counts pin the whole volume without shipping it
        out[f"mask_{i}_slice_counts"] = (body == 255).sum(axis=(1, 2)).astype(np.int64)
    out["matrix_slice_sums"] = matrix.astype(np.int64).sum(axis=(1, 2))
    # the two WHOLE reference masks, bit-packed (the marching-cubes envelope check contours them), and
    # what the reference recorded for the surfaces it built from them (surface_N.plist: volume in mm^3
    # of the smoothed / decimated mesh shipped in the project — an envelope, not a golden mesh)
    with tarfile.open(src, "r:*") as tf:
        files = {Path(m.name).name: tf.extractfile(m).read() for m in tf.getmembers() if m.isfile()}
    for i, (thr, m) in enumerate(masks):
        out[f"mask_{i}_bits_full"] = np.packbits(m[1:, 1:, 1:] == 255)
        out[f"surface_{i}_volume_mm3"] = np.array(float(plistlib.loads(files[f"surface_{i}.plist"])["volume"]))
    np.savez_compressed(DST, **out)
    print(DST, DST.stat().st_size, {k: v.shape for k, v in out.items()})
    buf = io.BytesIO()
    np.save(buf, thr_matrix(matrix, [thr for thr, _ in masks]))
    DST_THR.write_bytes(lzma.compress(buf.getvalue(), preset=9 | lzma.PRESET_EXTREME))
    print(DST_THR, DST_THR.stat().st_size)


if __name__ == "__main__":
    sys.exit(main())
