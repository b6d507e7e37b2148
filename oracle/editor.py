"""CPU checker for the 3-D mask editor — TEST INFRASTRUCTURE ONLY.

ctypes wrappers of oracle/editor.c (built into oracle/liboracle.so) with the
crate's names and argument order (invesalius_rs.polygon2mask_rs, mask_cut, brush_mask_rs), so the
parity tests read like calls of the reference. PARITY UNPINNED: see editor.c's header and DESIGN.md §5.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import _estrides, _ptr, lib

_IMAGE_DTYPES = (np.dtype(np.int16), np.dtype(np.uint8), np.dtype(np.float64))


def polygon2mask_rs(shape, polygon):
    """polygon_mask_py.rs:7-27 -> polygon_mask.rs:4-79."""
    w, h = (int(s) for s in shape)
    p = np.asarray(polygon)
    if p.dtype != np.float64 or p.ndim != 2:
        raise TypeError("polygon: 2-D float64 array expected")
    pts = np.ascontiguousarray(p[:, :2])
    out = np.zeros((w, h), np.uint8)
    lib().orc_polygon2mask(C.c_int64(w), C.c_int64(h), _ptr(pts), C.c_int64(len(pts)), _ptr(out))
    return out.view(np.bool_)


def mask_cut(image, sx, sy, sz, max_depth, mask, m, mv, out, edit_mode):
    """mask_cut_py.rs:8-69 -> mask_cut.rs:7-62."""
    if image.dtype not in _IMAGE_DTYPES or image.ndim != 3 or out.dtype != np.uint8 or out.ndim != 3:
        raise TypeError("Invalid image or mask type")
    if mask.dtype != np.bool_ or mask.ndim != 2:
        raise TypeError("mask: 2-D bool array expected")
    mm = np.ascontiguousarray(m, dtype=np.float64).reshape(16)
    vv = np.ascontiguousarray(mv, dtype=np.float64).reshape(16)
    mk = mask.view(np.uint8)
    lib().orc_mask_cut(C.c_double(sx), C.c_double(sy), C.c_double(sz), C.c_double(max_depth), _ptr(mk), _estrides(mk),
                       *map(C.c_int64, mask.shape), _ptr(mm), _ptr(vv), _ptr(out), _estrides(out),
                       *map(C.c_int64, out.shape), C.c_int32(int(edit_mode)))


def brush_mask_rs(out, orig, spacing, center, radius, edit_mode):
    """brush_mask_py.rs:7-28 -> brush_mask.rs:5-71."""
    if out.dtype != np.uint8 or out.ndim != 3 or (orig is not None and (orig.dtype != np.uint8 or orig.ndim != 3)):
        raise TypeError("Invalid mask type for brush mask")
    assert orig is None or orig.shape == out.shape
    og = orig if orig is not None else out
    lib().orc_brush_mask(_ptr(out), _estrides(out), None if orig is None else _ptr(orig), _estrides(og),
                         *map(C.c_int64, out.shape), *map(C.c_double, spacing), *map(C.c_double, center),
                         C.c_double(radius), C.c_int32(int(edit_mode)))
