"""Binary erosion and dilation with disk and ball footprints on the device: the mask-morphology plugin.

  disk(radius, dtype), ball(radius, dtype)                      skimage.morphology.disk / ball
  binary_erosion(image, footprint, out), binary_dilation(...)   skimage.morphology.binary_erosion / _dilation
      (plugins/mask_morphology/gui.py:5), for 2-D or 3-D bool / uint8 images and the footprints disk(r) (2-D)
      or ball(r) (3-D), r = 0 .. 15
  mask_morphology(mask_matrix, operation, radius, struct_type)   the body of MaskMorphologyPanel.OnApply
      (gui.py:98-175) in one upload, one launch sequence and one download

Under them, binary_morphology_device works on dense uint8 device tensors. skimage's functions are
scipy.ndimage.binary_erosion(border_value=True) / binary_dilation(border_value=False); every result here
equals SciPy's bit for bit (libb2v computes the bounded squared distance to the nearest source voxel one
axis at a time, in integers).
"""
from __future__ import annotations

import operator

import numpy as np
import torch

from . import _lib
from . import device as dev
from .device import _dense, _p, _stream

MAX_RADIUS = 15
_OPS = {"erosion": _lib.MORPH_ERODE, "dilation": _lib.MORPH_DILATE}
EROSION, DILATION = 0, 1     # the plugin's operation choice (gui.py:31)
DISK, BALL = 0, 1            # the plugin's structuring-element choice (gui.py:35)


def _radius(radius) -> int:
    r = operator.index(radius)
    if r < 0:
        raise ValueError(f"radius must be >= 0, got {r}")
    return r


def disk(radius, dtype=np.uint8) -> np.ndarray:
    """skimage.morphology.disk: (x^2 + y^2 <= r^2) on the (2r + 1)^2 grid."""
    r = _radius(radius)
    y, x = np.mgrid[-r:r + 1, -r:r + 1]
    return (x * x + y * y <= r * r).astype(dtype)


def ball(radius, dtype=np.uint8) -> np.ndarray:
    """skimage.morphology.ball: (x^2 + y^2 + z^2 <= r^2) on the (2r + 1)^3 grid."""
    r = _radius(radius)
    z, y, x = np.mgrid[-r:r + 1, -r:r + 1, -r:r + 1]
    return (x * x + y * y + z * z <= r * r).astype(dtype)


def _check_radius(r: int) -> None:
    if r > MAX_RADIUS:
        raise NotImplementedError(f"binary morphology: radius {r} > {MAX_RADIUS} is not supported")


def binary_morphology_device(t: torch.Tensor, op: str, radius: int, planar: bool, threshold: int = 0,
                             set_value: int = 1, out: torch.Tensor | None = None):
    """Erode (op "erosion", outside the volume counts as set) or dilate (op "dilation", outside counts as
    unset) the voxels of a dense uint8 [dz][dy][dx] tensor that exceed `threshold`, with disk(radius) on
    every z-slice (planar) or ball(radius). Returns (out, counts): out uint8 holding set_value where the
    result is set and 0 elsewhere, counts a device int64 [2] tensor with the set voxels of the input and
    of the result. Does not synchronise."""
    _dense(t, "image")
    if t.dtype != torch.uint8 or t.dim() != 3:
        raise TypeError("binary_morphology_device: uint8 3-D tensor expected")
    if op not in _OPS:
        raise ValueError(f"binary_morphology_device: op must be 'erosion' or 'dilation', not {op!r}")
    r = _radius(radius)
    _check_radius(r)
    if out is None:
        out = torch.empty(t.shape, dtype=torch.uint8, device=t.device)
    _dense(out, "out")
    if out.dtype != torch.uint8 or out.shape != t.shape:
        raise TypeError("binary_morphology_device: out must be uint8 with the image's shape")
    if out.device != t.device or out.data_ptr() == t.data_ptr():
        raise ValueError("binary_morphology_device: out must be a separate tensor on the image's device")
    counts = torch.empty(2, dtype=torch.int64, device=t.device)
    lib = _lib.load()
    ws = dev._workspace(lib.b2v_binary_morphology_workspace_bytes(*t.shape, int(bool(planar))), t.device)
    with torch.cuda.device(t.device):
        _lib.call("b2v_binary_morphology", _p(t), *t.shape, int(threshold), _OPS[op], r, int(bool(planar)),
                  int(set_value), _p(out), _p(counts), _p(ws), _stream())
    return out, counts


def _footprint_radius(footprint, ndim: int) -> int:
    """r when `footprint` is disk(r) for a 2-D image or ball(r) for a 3-D one (None: r = 1, skimage's
    default generate_binary_structure(ndim, 1)); SciPy's RuntimeError on a rank mismatch."""
    if footprint is None:
        return 1
    fp = np.asarray(footprint)
    if fp.ndim != ndim:
        raise RuntimeError("structure and input must have same dimensionality")
    n = fp.shape[0]
    if n % 2 == 0 or any(s != n for s in fp.shape):
        raise NotImplementedError(f"binary morphology: only disk / ball footprints are supported, not {fp.shape}")
    r = n // 2
    if not np.array_equal(fp != 0, (disk(r) if ndim == 2 else ball(r)) != 0):
        raise NotImplementedError("binary morphology: only disk / ball footprints are supported")
    _check_radius(r)
    return r


def _morphology(image, footprint, out, op: str) -> np.ndarray:
    a = np.asarray(image)
    if a.dtype not in (np.bool_, np.uint8):
        raise NotImplementedError(f"binary morphology: bool or uint8 images only, not {a.dtype}")
    if a.ndim not in (2, 3):
        raise NotImplementedError(f"binary morphology: 2-D or 3-D images only, not {a.ndim}-D")
    r = _footprint_radius(footprint, a.ndim)
    if out is None:
        out = np.empty(a.shape, bool)
    elif not isinstance(out, np.ndarray) or out.dtype != np.bool_ or out.shape != a.shape:
        raise NotImplementedError("binary morphology: out must be a bool array of the image's shape")
    if a.size == 0:
        return out
    planar = a.ndim == 2
    vol = a.reshape((1,) + a.shape) if planar else a
    t = dev.to_device(vol.view(np.uint8))
    res, _ = binary_morphology_device(t, op, r, planar)
    dev.to_host(res, (out[None] if planar else out).view(np.uint8))
    return out


def binary_erosion(image, footprint=None, out=None) -> np.ndarray:
    """skimage.morphology.binary_erosion: a voxel stays set when every footprint voxel inside the image is
    set (outside counts as set). Returns a bool array (`out` when given)."""
    return _morphology(image, footprint, out, "erosion")


def binary_dilation(image, footprint=None, out=None) -> np.ndarray:
    """skimage.morphology.binary_dilation: a voxel is set when a footprint voxel inside the image is set.
    Returns a bool array (`out` when given)."""
    return _morphology(image, footprint, out, "dilation")


def mask_morphology(mask_matrix, operation: int, radius: int, struct_type: int):
    """MaskMorphologyPanel.OnApply on mask.matrix (the padded [dz + 1][dy + 1][dx + 1] uint8 array, memmaps
    included): the body's voxels > 0 (edit and watershed markers included) eroded (operation 0) or dilated
    (1) with disk(radius) on every axial slice (struct_type 0) or ball(radius) (1). Returns
    (new_matrix, n_before, n_after), the set voxels before and after; new_matrix is a fresh array of the
    padded shape with the planes [0, :, :], [:, 0, :] and [:, :, 0] all 1 and the body 255 / 0, or None
    where the plugin leaves the mask unchanged: an empty mask, or an erosion that empties it."""
    m = np.asarray(mask_matrix)
    if m.dtype != np.uint8 or m.ndim != 3 or min(m.shape) < 1:
        raise TypeError("mask_morphology: the padded 3-D uint8 mask matrix expected")
    if operation not in (EROSION, DILATION) or struct_type not in (DISK, BALL):
        raise ValueError(f"mask_morphology: operation {operation!r} / struct_type {struct_type!r} out of range")
    op = "erosion" if operation == EROSION else "dilation"
    r = _radius(radius)
    _check_radius(r)
    body = m[1:, 1:, 1:]
    if body.size == 0:
        return None, 0, 0
    t = dev.to_device(body)
    res, counts = binary_morphology_device(t, op, r, struct_type == DISK, threshold=0, set_value=255)
    n_before, n_after = (int(v) for v in counts.cpu())
    if n_before == 0:
        return None, 0, 0
    if n_after == 0:      # only an erosion can empty a non-empty mask
        return None, n_before, 0
    new = np.empty(m.shape, np.uint8)
    new[0, :, :] = 1
    new[:, 0, :] = 1
    new[:, :, 0] = 1
    dev.to_host(res, new[1:, 1:, 1:])
    return new, n_before, n_after
