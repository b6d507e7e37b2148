"""Inputs of the surface join: masks and images cut into Z pieces as SurfaceManager.AddNewActor cuts them
(surface.py:1362-1381: pieces of 20 slices plus one shared slice), and those pieces contoured on the host
by the marching-cubes checker with create_surface_piece's padding."""
import numpy as np
from scipy import ndimage

PIECE_SIZE, OVERLAP = 20, 1
CA_OPTIONS = {"angle": 0.7, "max distance": 3.0, "min weight": 0.5, "steps": 10}   # the GUI's defaults
SPACING = (0.9570312, 0.9570312, 1.5)


def rois(dz: int):
    n = int(round(dz / PIECE_SIZE + 0.5))
    return [slice(i * PIECE_SIZE, (i + 1) * PIECE_SIZE + OVERLAP) for i in range(n)]


def padded_mask(body: np.ndarray) -> np.ndarray:
    """The Mask memmap's layout: [dz+1][dy+1][dx+1] with a zero first slice, row and column."""
    dz, dy, dx = body.shape
    mm = np.zeros((dz + 1, dy + 1, dx + 1), np.uint8)
    mm[1:, 1:, 1:] = body
    return mm


def noise_case(seed: int, shape=(45, 40, 48)):
    """(padded mask, int16 image) of smoothed noise: many parts, holes where they touch the border."""
    rng = np.random.default_rng(seed)
    body = (ndimage.gaussian_filter(rng.normal(size=shape), 1.3) > 0).astype(np.uint8) * np.uint8(255)
    img = (ndimage.gaussian_filter(rng.normal(size=shape), 1.3) * 3000).astype(np.int16)
    return padded_mask(body), img


def host_pieces(orc, data: np.ndarray, isovalues, spacing=SPACING, fill_border_holes=True):
    """create_surface_piece's meshes with the checker: data is the unpadded mask (iso 127) or image
    (isovalues tmin, tmax), padded with 0 or the int16 minimum."""
    pad_value = 0 if data.dtype == np.uint8 else int(np.iinfo(np.int16).min)
    dz, dy, dx = data.shape
    out = []
    for roi in rois(dz):
        a = data[roi]
        if a.shape[0] == 0:
            out.append((np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64)))
            continue
        pb, pt = roi.start == 0, roi.stop >= dz
        padding = (0, 0, 0)
        if fill_border_holes:
            pad = np.full((a.shape[0] + pb + pt, dy + 2, dx + 2), pad_value, data.dtype)
            pad[int(pb):int(pb) + a.shape[0], 1:-1, 1:-1] = a
            a, padding = pad, (1, 1, int(pb))
        vs, fs, base = [], [], 0
        for iso in isovalues:
            v, f = orc.marching_cubes(a, iso, spacing, (-padding[0], -padding[1], roi.start - padding[2]), True)
            vs.append(v)
            fs.append(f + base)
            base += len(v)
        out.append((np.concatenate(vs), np.concatenate(fs)))
    return out


def triangle_rows(points: np.ndarray, faces: np.ndarray) -> np.ndarray:
    """The triangles as rows of their 9 corner coordinates' bits, corners in order, rows sorted."""
    rows = points[np.asarray(faces, np.int64).reshape(-1, 3)].reshape(-1, 9).view(np.uint32)
    return rows[np.lexsort(rows.T[::-1])] if len(rows) else rows
