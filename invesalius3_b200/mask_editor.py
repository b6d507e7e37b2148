"""The 3-D mask editor's crate functions on the device (invesalius/data/mask3d_editor_state.py:14):

  polygon2mask_rs(shape, polygon)                                 polygon_mask_py.rs:7-27 -> polygon_mask.rs:4-79
  mask_cut(image, sx, sy, sz, max_depth, mask, M, MV, out, edit_mode)   mask_cut_py.rs:8-69 -> mask_cut.rs:7-62
  brush_mask_rs(out, orig, spacing, center, radius, edit_mode)    brush_mask_py.rs:7-28 -> brush_mask.rs:5-71

The numpy functions keep the crate's names, argument order and in-place writes, so the editor binds
them with one import line. They validate every argument before any device work. Under them is a
device-tensor layer (polygon2mask_device, mask_cut_device, brush_mask_device) for callers that keep
the mask in HBM across cuts and strokes.

Deviations from the crate, where it panics: a non-finite polygon vertex, an M or MV that is not a
C-contiguous 4x4 block of 16 doubles, and an `orig` whose shape differs from `out` raise ValueError.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from . import device as dev
from .device import _dense, _p, _stream

_IMAGE_DTYPES = (np.dtype(np.int16), np.dtype(np.uint8), np.dtype(np.float64))


def _i32(v, name: str) -> int:
    """PyO3 `i32` extraction: floats are a TypeError, out-of-range integers an OverflowError."""
    if isinstance(v, (float, np.floating)) or not hasattr(v, "__index__"):
        raise TypeError(f"{name}: 'float' object cannot be interpreted as an integer")
    v = int(v)
    if not -(2 ** 31) <= v < 2 ** 31:
        raise OverflowError("out of range integral type conversion attempted")
    return v


def _dbl3(v, name: str) -> np.ndarray:
    t = tuple(float(x) for x in v)
    if len(t) != 3:
        raise TypeError(f"{name}: a tuple of three floats expected")
    return np.array(t, np.float64)


def _mat4(a, name: str) -> np.ndarray:
    if not isinstance(a, np.ndarray) or a.dtype != np.float64 or a.ndim != 2:
        raise TypeError(f"{name}: 2-D float64 array expected")
    if not a.flags.c_contiguous or a.size != 16:
        raise ValueError(f"{name}: a C-contiguous array of 16 elements expected (the crate panics here)")
    return a.reshape(16)


def _writeable_u8_3d(a, what: str) -> None:
    if not isinstance(a, np.ndarray) or a.dtype != np.uint8 or a.ndim != 3 or not a.flags.writeable:
        raise TypeError(what)


# ----------------------------------------------------------------------------- polygon2mask
def _polygon(polygon) -> np.ndarray:
    p = polygon.numpy() if isinstance(polygon, torch.Tensor) else polygon
    if not isinstance(p, np.ndarray) or p.dtype != np.float64 or p.ndim != 2:
        raise TypeError("polygon: 2-D float64 array of (x, y) points expected")
    if len(p) and p.shape[1] < 2:
        raise ValueError("polygon: every point needs an x and a y")
    pts = np.ascontiguousarray(p[:, :2]) if len(p) else np.zeros((0, 2), np.float64)
    if not np.isfinite(pts).all():
        raise ValueError("polygon: coordinates must be finite (the crate overflows on them)")
    return pts


def _shape2(shape) -> tuple[int, int]:
    w, h = (int(s) for s in shape)
    if w < 0 or h < 0:
        raise OverflowError("can't convert negative int to unsigned")
    return w, h


def polygon2mask_device(shape, polygon, device=None) -> torch.Tensor:
    """(w, h) uint8 tensor, 1 where the screen point (row, column) lies inside `polygon` (even-odd
    rule, N x 2 float64 (x, y) points on the host), 0 elsewhere."""
    w, h = _shape2(shape)
    pts = _polygon(polygon)
    dev.require_cuda()
    device = torch.device("cuda" if device is None else device)
    out = torch.empty((w, h), dtype=torch.uint8, device=device)
    ws = torch.empty(max(1, pts.size) * 8, dtype=torch.uint8, device=device)
    with torch.cuda.device(device):
        _lib.call("b2v_polygon2mask", C.c_void_p(pts.ctypes.data), len(pts), w, h, _p(out), _p(ws), _stream())
    return out


def polygon2mask_rs(shape, polygon) -> np.ndarray:
    """invesalius_rs.polygon2mask_rs: bool array of shape (w, h)."""
    t = polygon2mask_device(shape, polygon)
    res = np.empty(tuple(t.shape), np.bool_)
    if res.size:
        dev.to_host(t, res.view(np.uint8))
    return res


# ----------------------------------------------------------------------------- mask_cut
def mask_cut_device(out: torch.Tensor, spacing, max_depth: float, filt: torch.Tensor, m, mv, edit_mode: int) -> torch.Tensor:
    """mask_cut on a dense uint8 [dz][dy][dx] device mask, in place. filt: dense (h, w) uint8 device
    image, non-zero = inside the cutting polygon(s); m, mv: 4x4 float64 (world -> screen, world ->
    camera). Returns `out`."""
    _dense(out, "out"); _dense(filt, "filter")
    if out.dtype != torch.uint8 or out.dim() != 3:
        raise TypeError("mask_cut_device: out must be a 3-D uint8 tensor")
    if filt.dtype not in (torch.uint8, torch.bool) or filt.dim() != 2:
        raise TypeError("mask_cut_device: filter must be a 2-D uint8 or bool tensor")
    if out.data_ptr() % 16:
        raise ValueError("mask_cut_device: out must be 16-byte aligned")
    mm = _mat4(np.asarray(m, dtype=np.float64), "M")
    vv = _mat4(np.asarray(mv, dtype=np.float64), "MV")
    sp = _dbl3(spacing, "spacing")
    h, w = filt.shape
    with torch.cuda.device(out.device):
        _lib.call("b2v_mask_cut", _p(out), *out.shape, C.c_void_p(sp.ctypes.data), float(max_depth),
                  _p(filt.view(torch.uint8)), h, w, C.c_void_p(mm.ctypes.data), C.c_void_p(vv.ctypes.data),
                  _i32(edit_mode, "edit_mode"), _stream())
    return out


def mask_cut(image, sx, sy, sz, max_depth, mask, m, mv, out, edit_mode) -> None:
    """invesalius_rs.mask_cut: zero the voxels of `out` (> 127) that the camera sees inside `mask`
    (include mode 0 also zeroes those it sees off-screen). `image` only selects the dtype and is
    never read; `mask` is (h, w) bool with any strides; `out` is edited in place (strided views
    welcome)."""
    if not isinstance(image, np.ndarray) or image.dtype not in _IMAGE_DTYPES or image.ndim != 3:
        raise TypeError("Invalid image or mask type")
    _writeable_u8_3d(out, "Invalid image or mask type")
    if not isinstance(mask, np.ndarray) or mask.dtype != np.bool_ or mask.ndim != 2:
        raise TypeError("mask: 2-D bool array expected")
    mm, vv = _mat4(m, "M"), _mat4(mv, "MV")
    sp = (float(sx), float(sy), float(sz))
    max_depth = float(max_depth)
    edit_mode = _i32(edit_mode, "edit_mode")
    if out.size == 0:
        return
    t = dev.to_device(out)
    f = dev.to_device(np.ascontiguousarray(mask).view(np.uint8), t.device)
    mask_cut_device(t, sp, max_depth, f, mm.reshape(4, 4), vv.reshape(4, 4), edit_mode)
    dev.to_host(t, out)


# ----------------------------------------------------------------------------- brush
def brush_mask_box(shape, spacing, center, radius):
    """The voxel box a brush can touch, as the library computes it (brush_mask.rs:24-31):
    ((z0, z1), (y0, y1), (x0, x1)) inclusive, or None when it is empty."""
    dz, dy, dx = (int(s) for s in shape)
    sp, c = _dbl3(spacing, "spacing"), _dbl3(center, "center")
    box = (C.c_int64 * 6)()
    _lib.call("b2v_brush_mask_box", dz, dy, dx, C.c_void_p(sp.ctypes.data), C.c_void_p(c.ctypes.data), float(radius),
              box)
    if box[3] < box[0]:
        return None
    return (box[0], box[3]), (box[1], box[4]), (box[2], box[5])


def _brush(out: torch.Tensor, orig: torch.Tensor | None, origin, shape, sp: np.ndarray, c: np.ndarray, radius: float,
           edit_mode: int) -> None:
    """b2v_brush_mask on a dense buffer holding voxel `origin` of a `shape` volume at its first byte."""
    _dense(out, "out")
    if orig is not None:
        _dense(orig, "orig")
        if orig.shape != out.shape or orig.dtype != torch.uint8:
            raise ValueError("orig must be a uint8 tensor of out's shape")
    _, by, bx = out.shape
    with torch.cuda.device(out.device):
        _lib.call("b2v_brush_mask", _p(out), _p(orig), *shape, *origin, bx, by * bx, C.c_void_p(sp.ctypes.data),
                  C.c_void_p(c.ctypes.data), radius, edit_mode, _stream())


def brush_mask_device(out: torch.Tensor, orig: torch.Tensor | None, spacing, center, radius: float,
                      edit_mode: int) -> torch.Tensor:
    """brush_mask_rs on a dense uint8 [dz][dy][dx] device mask, in place; only the brush's box is
    visited. orig: None or a dense uint8 tensor of the same shape. Returns `out`."""
    if out.dtype != torch.uint8 or out.dim() != 3:
        raise TypeError("Invalid mask type for brush mask")
    _brush(out, orig, (0, 0, 0), tuple(out.shape), _dbl3(spacing, "spacing"), _dbl3(center, "center"), float(radius),
           _i32(edit_mode, "edit_mode"))
    return out


def brush_mask_rs(out, orig, spacing, center, radius, edit_mode) -> None:
    """invesalius_rs.brush_mask_rs: paint (mode 0: orig > 0, or 255 without orig) or erase (mode 1)
    a sphere of `radius` mm about `center` (x, y, z mm) into `out` in place. Only the sphere's box
    of `out` (and of `orig`) travels to the device and back, so a stroke costs the same on any
    volume size."""
    _writeable_u8_3d(out, "Invalid mask type for brush mask")
    if orig is not None:
        if not isinstance(orig, np.ndarray) or orig.dtype != np.uint8 or orig.ndim != 3:
            raise TypeError("Invalid mask type for brush mask")
        if orig.shape != out.shape:
            raise ValueError(f"orig has shape {orig.shape}, out has {out.shape} (the crate panics past a smaller orig)")
    sp, c = _dbl3(spacing, "spacing"), _dbl3(center, "center")
    radius = float(radius)
    edit_mode = _i32(edit_mode, "edit_mode")
    if edit_mode not in (0, 1):
        return
    box = brush_mask_box(out.shape, sp, c, radius)
    if box is None:
        return
    (z0, z1), (y0, y1), (x0, x1) = box
    sl = (slice(z0, z1 + 1), slice(y0, y1 + 1), slice(x0, x1 + 1))
    ob = out[sl]
    t = dev.to_device(ob)
    to = dev.to_device(orig[sl], t.device) if orig is not None else None
    _brush(t, to, (z0, y0, x0), out.shape, sp, c, radius, edit_mode)
    dev.to_host(t, ob)
