"""Spline resampling on the device: scipy.ndimage.zoom and the two InVesalius functions built on it.

  zoom(input, zoom, output, order, mode, cval, ...)   scipy.ndimage.zoom, numpy in / numpy out
  resize_slice(im_array, resolution_percentage)       imagedata_utils.py:109-118 (order 2)
  resize_image_array(image, resolution_percentage, as_mmap)   imagedata_utils.py:121-129 (order 2); called
      twice by SurfaceManager.AddNewActor for the "Low" and "Medium" surface qualities (surface.py:1352-1353)

Under them, zoom_device works on device tensors. The built subset is spline order 0-3, mode 'constant' or
'mirror', prefilter=True, grid_mode=False, and int16, uint8, float32 and float64 arrays of 2 or 3
dimensions; anything else raises NotImplementedError. Within it the result equals SciPy's bit for bit,
including the 'constant' mode edge case where the last sample's coordinate rounds past the input's edge
and SciPy writes cval.
"""
from __future__ import annotations

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


def _factors(zoom, ndim: int) -> tuple[float, ...]:
    if np.ndim(zoom) == 0:
        return (float(zoom),) * ndim
    z = tuple(float(f) for f in zoom)
    if len(z) != ndim:
        raise RuntimeError("sequence argument must have length equal to input rank")   # SciPy's message
    return z


def output_shape(shape, zoom) -> tuple[int, ...]:
    """SciPy's output shape: round(n * factor) per axis (Python's round, ties to even)."""
    return tuple(int(round(n * f)) for n, f in zip(shape, _factors(zoom, len(shape))))


def zoom_device(t: torch.Tensor, zoom, order: int, out_dtype: torch.dtype, cval: float = 0.0,
                mode: str = "constant") -> torch.Tensor:
    """scipy.ndimage.zoom(t, zoom, out_dtype, order, mode, cval) on a dense 2-D or 3-D device tensor of
    int16, uint8, float32 or float64; returns a new tensor of out_dtype. Where every factor is 1 the
    result is t cast to out_dtype, as SciPy returns its input unchanged."""
    _dense(t, "image")
    if t.dim() not in (2, 3):
        raise NotImplementedError("zoom_device: 2-D or 3-D input only")
    if t.dtype not in _CODE or out_dtype not in _CODE:
        raise NotImplementedError(f"zoom_device: dtypes int16, uint8, float32, float64 only ({t.dtype} -> {out_dtype})")
    if order not in (0, 1, 2, 3):
        raise NotImplementedError(f"zoom_device: spline order {order} not built (0-3)")
    if mode not in _MODES:
        raise NotImplementedError(f"zoom_device: mode {mode!r} not built ('constant', 'mirror')")
    factors = _factors(zoom, t.dim())
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
    shape = output_shape(a.shape, zoom)
    res = None
    if output is None:
        out_dtype = a.dtype
    elif isinstance(output, np.ndarray):
        if output.shape != shape:
            raise RuntimeError("output shape not correct")   # SciPy's message
        res, out_dtype = output, output.dtype
    else:
        out_dtype = np.dtype(output)
    if out_dtype not in _NP:
        raise NotImplementedError(f"zoom: output dtype {out_dtype} is not built (int16, uint8, float32, float64)")
    if res is None:
        res = np.empty(shape, out_dtype)
    if all(f == 1 for f in _factors(zoom, a.ndim)):
        res[...] = a
        return res
    if a.size == 0 or res.size == 0:
        return res
    t = dev.to_device(a)
    o = zoom_device(t, zoom, order, _NP[out_dtype], cval, mode)
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
