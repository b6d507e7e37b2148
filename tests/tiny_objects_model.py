"""A NumPy / SciPy restatement of the "Remove tiny objects" plugin (plugins/remove_tiny_objects/gui.py), the
model the device's TinyObjects is compared with. Its three steps, on the padded mask matrix
[dz + 1][dy + 1][dx + 1] whose body is matrix[1:, 1:, 1:]:

  find_regions   label the body with SciPy's default structure (6-connected, any non-zero voxel a feature)
                 and give every voxel the number of voxels of its region, background included
  preview        255 where that number is at most min_size, else 0, as uint8
  remove         a copy of the matrix with the body set to 1 where the preview is above 127
"""
import numpy as np
from scipy import ndimage


def find_regions(matrix: np.ndarray):
    """(labels int32, number of labels, uint32 region size of every body voxel)."""
    labels, n = ndimage.label(matrix[1:, 1:, 1:])
    sizes = np.bincount(labels.ravel(), minlength=n + 1).astype(np.uint32)
    return labels, n, sizes[labels]


def preview(counts: np.ndarray, min_size) -> np.ndarray:
    out = np.empty(counts.shape, np.uint8)
    out[:] = (counts <= min_size) * 255
    return out


def remove(matrix: np.ndarray, preview_matrix: np.ndarray) -> np.ndarray:
    out = matrix.copy()
    body = out[1:, 1:, 1:]
    body[preview_matrix > 127] = 1
    return out


def padded(body: np.ndarray, rng=None) -> np.ndarray:
    """The mask matrix around `body`; the flag planes z = 0, y = 0 and x = 0 hold 0, 1 or 2 at random
    (any values will do: nothing may change them)."""
    rng = rng or np.random.default_rng(0)
    m = rng.integers(0, 3, size=tuple(s + 1 for s in body.shape), dtype=np.uint8)
    m[1:, 1:, 1:] = body
    return m
