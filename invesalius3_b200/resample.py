"""Spline resampling on the device: scipy.ndimage.zoom and shift, and the InVesalius functions built on them.

  zoom(input, zoom, output, order, mode, cval, ...)   scipy.ndimage.zoom, numpy in / numpy out
  resize_slice(im_array, resolution_percentage)       imagedata_utils.py:109-118 (order 2)
  resize_image_array(image, resolution_percentage, as_mmap)   imagedata_utils.py:121-129 (order 2); called
      twice by SurfaceManager.AddNewActor for the "Low" and "Medium" surface qualities (surface.py:1352-1353)
  shift(input, shift, output, order, mode, cval, prefilter)   scipy.ndimage.shift, numpy in / numpy out
  fix_gantry_tilt(matrix, spacing, tilt)              imagedata_utils.FixGantryTilt (:143-154), in place; called
      by the DICOM import (control.py:1331, :1334)
  make_orthogonal(matrix, old_spacing, new_spacing)   plugins/change_spacing/main.py:11-18

Under them, zoom_device, shift_device and fix_gantry_tilt_device work on device tensors. The built subset is
spline order 0-3, mode 'constant' or 'mirror', prefilter=True, grid_mode=False, and int16, uint8, float32 and
float64 arrays of 2 or 3 dimensions; anything else raises NotImplementedError. Within it the result equals
SciPy's bit for bit, including the 'constant' mode edge cases where a coordinate lies just outside the input
and SciPy writes cval.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import tempfile

import numpy as np
import torch

from . import _lib
from . import device as dev
from .device import _dense, _p, _stream

_CODE = {torch.int16: _lib.I16, torch.uint8: _lib.U8, torch.float32: _lib.F32, torch.float64: _lib.F64}
_NP = {np.dtype(np.int16): torch.int16, np.dtype(np.uint8): torch.uint8, np.dtype(np.float32): torch.float32,
       np.dtype(np.float64): torch.float64}
_MODES = {"constant": _lib.ZOOM_CONSTANT, "mirror": _lib.ZOOM_MIRROR}


def _per_axis(value, ndim: int) -> tuple[float, ...]:
    """A zoom factor or shift: one number for every axis, or one per axis."""
    if np.ndim(value) == 0:
        return (float(value),) * ndim
    v = tuple(float(x) for x in value)
    if len(v) != ndim:
        raise RuntimeError("sequence argument must have length equal to input rank")   # SciPy's message
    return v


def _check_built(name: str, t_dtype, out_dtype, ndim: int, order: int, mode: str) -> None:
    if ndim not in (2, 3):
        raise NotImplementedError(f"{name}: 2-D or 3-D input only")
    if t_dtype not in _CODE or out_dtype not in _CODE:
        raise NotImplementedError(f"{name}: dtypes int16, uint8, float32, float64 only ({t_dtype} -> {out_dtype})")
    if order not in (0, 1, 2, 3):
        raise NotImplementedError(f"{name}: spline order {order} not built (0-3)")
    if mode not in _MODES:
        raise NotImplementedError(f"{name}: mode {mode!r} not built ('constant', 'mirror')")


def _output(name: str, output, dtype, shape) -> np.ndarray:
    """The array that receives a result of `shape`: `output` itself if it is an array, else a new array of the
    dtype `output` names (None: `dtype`, the input's)."""
    if output is None:
        out_dtype = dtype
    elif isinstance(output, np.ndarray):
        if output.shape != shape:
            raise RuntimeError("output shape not correct")   # SciPy's message
        out_dtype = output.dtype
    else:
        out_dtype = np.dtype(output)
    if out_dtype not in _NP:
        raise NotImplementedError(f"{name}: output dtype {out_dtype} is not built (int16, uint8, float32, float64)")
    return output if isinstance(output, np.ndarray) else np.empty(shape, out_dtype)


def output_shape(shape, zoom) -> tuple[int, ...]:
    """SciPy's output shape: round(n * factor) per axis (Python's round, ties to even)."""
    return tuple(int(round(n * f)) for n, f in zip(shape, _per_axis(zoom, len(shape))))


def zoom_device(t: torch.Tensor, zoom, order: int, out_dtype: torch.dtype, cval: float = 0.0,
                mode: str = "constant") -> torch.Tensor:
    """scipy.ndimage.zoom(t, zoom, out_dtype, order, mode, cval) on a dense 2-D or 3-D device tensor of
    int16, uint8, float32 or float64; returns a new tensor of out_dtype. Where every factor is 1 the
    result is t cast to out_dtype, as SciPy returns its input unchanged."""
    _dense(t, "image")
    _check_built("zoom_device", t.dtype, out_dtype, t.dim(), order, mode)
    factors = _per_axis(zoom, t.dim())
    shape = output_shape(t.shape, factors)
    if all(f == 1 for f in factors):
        return t.to(out_dtype, copy=True)
    out = torch.empty(shape, dtype=out_dtype, device=t.device)
    if out.numel() == 0 or t.numel() == 0:
        return out
    dims3 = tuple(t.shape) if t.dim() == 3 else (1, *t.shape)
    out3 = shape if t.dim() == 3 else (1, *shape)
    ws = dev._workspace(_lib.load().b2v_zoom_workspace_bytes(*dims3, order), t.device)
    with torch.cuda.device(t.device):
        _lib.call("b2v_zoom", _p(t), _CODE[t.dtype], t.dim(), *dims3, *out3, order, _MODES[mode], float(cval), _p(out),
                  _CODE[out_dtype], _p(ws), _stream())
    return out


def zoom(input, zoom, output=None, order: int = 3, mode: str = "constant", cval: float = 0.0, prefilter: bool = True,
         grid_mode: bool = False):
    """scipy.ndimage.zoom for 2-D and 3-D numpy arrays (memmaps and strided views included). `output` is
    None (the input's dtype), a dtype, or an array of the output shape that receives the result."""
    a = np.asarray(input)
    if not prefilter:
        raise NotImplementedError("zoom: prefilter=False is not built")
    if grid_mode:
        raise NotImplementedError("zoom: grid_mode=True is not built")
    if a.dtype not in _NP:
        raise NotImplementedError(f"zoom: dtype {a.dtype} is not built (int16, uint8, float32, float64)")
    if a.ndim not in (2, 3):
        raise NotImplementedError("zoom: 2-D or 3-D input only")
    res = _output("zoom", output, a.dtype, output_shape(a.shape, zoom))
    if all(f == 1 for f in _per_axis(zoom, a.ndim)):
        res[...] = a
        return res
    if a.size == 0 or res.size == 0:
        return res
    t = dev.to_device(a)
    o = zoom_device(t, zoom, order, _NP[res.dtype], cval, mode)
    dev.to_host(o, res)
    return res


def shift_device(t: torch.Tensor, shift, order: int, out_dtype: torch.dtype, cval: float = 0.0,
                 mode: str = "constant") -> torch.Tensor:
    """scipy.ndimage.shift(t, shift, out_dtype, order, mode, cval) on a dense 2-D or 3-D device tensor of
    int16, uint8, float32 or float64; returns a new tensor of out_dtype and t's shape."""
    _dense(t, "image")
    _check_built("shift_device", t.dtype, out_dtype, t.dim(), order, mode)
    sh = (C.c_double * t.dim())(*_per_axis(shift, t.dim()))
    out = torch.empty(t.shape, dtype=out_dtype, device=t.device)
    if t.numel() == 0:
        return out
    dims3 = tuple(t.shape) if t.dim() == 3 else (1, *t.shape)
    ws = dev._workspace(_lib.load().b2v_shift_workspace_bytes(*dims3, order), t.device)
    with torch.cuda.device(t.device):
        _lib.call("b2v_shift", _p(t), _CODE[t.dtype], t.dim(), *dims3, sh, order, _MODES[mode], float(cval), _p(out),
                  _CODE[out_dtype], _p(ws), _stream())
    return out


def shift(input, shift, output=None, order: int = 3, mode: str = "constant", cval: float = 0.0,
          prefilter: bool = True):
    """scipy.ndimage.shift for 2-D and 3-D numpy arrays (memmaps and strided views included). `output` is
    None (the input's dtype), a dtype, or an array of the input's shape that receives the result."""
    a = np.asarray(input)
    if not prefilter:
        raise NotImplementedError("shift: prefilter=False is not built")
    if a.dtype not in _NP:
        raise NotImplementedError(f"shift: dtype {a.dtype} is not built (int16, uint8, float32, float64)")
    if a.ndim not in (2, 3):
        raise NotImplementedError("shift: 2-D or 3-D input only")
    res = _output("shift", output, a.dtype, a.shape)
    _check_built("shift", _NP[a.dtype], _NP[res.dtype], a.ndim, order, mode)
    _per_axis(shift, a.ndim)
    if a.size == 0:
        return res
    o = shift_device(dev.to_device(a), shift, order, _NP[res.dtype], cval, mode)
    dev.to_host(o, res)
    return res


def tilt_shifts(nz: int, spacing, tilt) -> np.ndarray:
    """The per-slice (y, x) shifts FixGantryTilt passes to scipy.ndimage.shift (imagedata_utils.py:143-154), in
    its float64 operations and order: offset = tan(radians(tilt)) * n * spacing[2], y shift -offset / spacing[1]."""
    angle = np.radians(tilt)
    spacing = spacing[0], spacing[1], spacing[2]
    gntan = math.tan(angle)
    shifts = np.zeros((nz, 2), np.float64)
    for n in range(nz):
        offset = gntan * n * spacing[2]
        shifts[n, 0] = -offset / spacing[1]
    return shifts


def fix_gantry_tilt_device(t: torch.Tensor, spacing, tilt, slab: int = 0) -> torch.Tensor:
    """imagedata_utils.FixGantryTilt in place on a dense int16 [z][y][x] device tensor: every slice shifted along
    y at order 3 in 'constant' mode with cval = matrix.min() of the volume as the sequential loop leaves it.
    slab: slices per prefilter pass (0: as many as fit 1 GiB of float64). Returns the per-slice cvals (int16)."""
    _dense(t, "matrix")
    if t.dim() != 3:
        raise ValueError("fix_gantry_tilt_device: 3-D volume expected")
    if t.dtype != torch.int16:
        raise NotImplementedError(f"fix_gantry_tilt_device: int16 only ({t.dtype})")
    nz, ny, nx = t.shape
    cvals = torch.empty(nz, dtype=torch.int16, device=t.device)
    if t.numel() == 0:
        return cvals
    shifts = tilt_shifts(nz, spacing, tilt)
    ws = dev._workspace(_lib.load().b2v_gantry_tilt_workspace_bytes(nz, ny, nx, int(slab)), t.device)
    with torch.cuda.device(t.device):
        _lib.call("b2v_gantry_tilt", _p(t), nz, ny, nx, C.c_void_p(shifts.ctypes.data), int(slab), _p(ws), _p(cvals),
                  _stream())
    return cvals


def fix_gantry_tilt(matrix, spacing, tilt) -> None:
    """imagedata_utils.FixGantryTilt(matrix, spacing, tilt): in place on an int16 [z][y][x] numpy array or
    np.memmap; the volume goes to the device once and comes back once."""
    if not isinstance(matrix, np.ndarray) or matrix.ndim != 3:
        # the reference's per-slice scipy.ndimage.shift(slice, (dy, 0)) needs 2-D slices
        raise RuntimeError("sequence argument must have length equal to input rank")
    if matrix.dtype != np.int16:
        raise NotImplementedError(f"fix_gantry_tilt: int16 only ({matrix.dtype})")
    if matrix.shape[0] == 0:
        return
    if matrix.size == 0:
        raise ValueError("zero-size array to reduction operation minimum which has no identity")   # NumPy's
    if not matrix.flags.writeable:
        raise ValueError("assignment destination is read-only")   # NumPy's
    t = dev.to_device(matrix)
    fix_gantry_tilt_device(t, spacing, tilt)
    dev.to_host(t, matrix)


def make_orthogonal(matrix, old_spacing, new_spacing):
    """plugins/change_spacing/main.py:make_orthogonal: zoom(matrix, old / new spacing per axis, reversed,
    output=matrix.dtype, mode='constant', cval=matrix.min()) at order 3, with the minimum taken on the device."""
    zooms = [i / j for (i, j) in zip(old_spacing, new_spacing)]
    a = np.asarray(matrix)
    if a.dtype not in (np.int16, np.uint8) or a.ndim != 3:
        raise NotImplementedError(f"make_orthogonal: 3-D int16 or uint8 only ({a.ndim}-D {a.dtype})")
    if a.size == 0:
        raise ValueError("zero-size array to reduction operation minimum which has no identity")   # NumPy's
    t = dev.to_device(a)
    cval = float(dev.minmax(t)[0].item())   # exact: every int16 and uint8 is a float32
    o = zoom_device(t, zooms[::-1], 3, t.dtype, cval, "constant")
    res = np.empty(tuple(o.shape), a.dtype)
    dev.to_host(o, res)
    return res


def resize_slice(im_array, resolution_percentage):
    """imagedata_utils.resize_slice: zoom(im_array, resolution_percentage, im_array.dtype, order=2)."""
    return zoom(im_array, resolution_percentage, im_array.dtype, order=2)


def resize_image_array(image, resolution_percentage, as_mmap=False):
    """imagedata_utils.resize_image_array: zoom(image, resolution_percentage, image.dtype, order=2), and
    with as_mmap a np.memmap over a new temporary file holding it."""
    out = zoom(image, resolution_percentage, image.dtype, order=2)
    if as_mmap:
        fd, fname = tempfile.mkstemp(suffix="_resized")
        out_mmap = np.memmap(fname, shape=out.shape, dtype=out.dtype, mode="w+")
        out_mmap[:] = out
        os.close(fd)
        return out_mmap
    return out
