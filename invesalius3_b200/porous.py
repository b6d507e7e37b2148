"""The porous-creation plugin's TPMS and Blobs scaffolds, and the float64 image_normalize, on the device.

  create_schwarzp(method, init_x, end_x, init_y, end_y, init_z, end_z, sx, sy, sz)   schwarzp.py:11-28
  create_blobs(sx, sy, sz, gaussian)                                                  schwarzp.py:31-34
  image_normalize(image, min_, max_, output_dtype)   imagedata_utils.py:580-587 (gui.py:28, 237)
  create_schwarzp_i16(..., min_, max_) / create_blobs_i16(..., min_, max_)   image_normalize(create_*(...)), the
      int16 matrix that the dialog's OnOk (gui.py:183-245) sends to "Create project from matrix"

numpy in, numpy out; the *_device forms return the CUDA tensor. Every result equals the plugin's bit for bit:

- create_schwarzp evaluates np.cos / np.sin on the 1-D np.ogrid axes only, then broadcasts float64 *, + and -.
  The axes and their six cos / sin tables are computed here with NumPy from the caller's arguments (single-point,
  reversed and equal-bounds axes come out exactly as NumPy makes them), and b2v_tpms_f64 combines the tables per
  voxel in NumPy's order. create_schwarzp_i16 never stores the float64 field: b2v_tpms_i16 evaluates it once for
  its min / max and once more for the int16 store, and only 2 B per voxel are downloaded.
- create_blobs draws np.random.random((sz, sy, sx)) on the host with the plugin's call, so the global RNG is
  consumed identically and one np.random.seed gives one scaffold. Reproducing the legacy MT19937 stream on the
  device would take a sequential twist or a GF(2) jump-ahead, so the draw and its upload stay on the host. The
  float64 gaussian_filter is filters._gaussian (three b2v_correlate1d passes), skipped where SciPy skips it
  (sigma <= 1e-15: a copy of the draw).
- image_normalize of a float64 image is (image - imin) * ((max_ - min_) / (imax - imin)) + min_ in float64, with
  NumPy's promotion of the bounds, stored with the C cast (b2v_image_normalize_f64_i16); min_ converted as NumPy
  converts it where the image is constant. float32 images go to voronoi.image_normalize.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from . import device as dev
from . import filters, voronoi
from .device import _p, _stream

SURFACES = _lib.TPMS_SURFACES


def _surface_code(method):
    for code, name in enumerate(SURFACES):
        if method == name:
            return code
    return None


def _axes(init_x, end_x, init_y, end_y, init_z, end_z, sx, sy, sz):
    """The plugin's np.ogrid axes (z, y, x), with NumPy's own argument errors."""
    return np.ogrid[init_z:end_z:complex(0, sz), init_y:end_y:complex(0, sy), init_x:end_x:complex(0, sx)]


def _tables(z, y, x) -> np.ndarray:
    """[cos_x | sin_x | cos_y | sin_y | cos_z | sin_z], NumPy's cos / sin of the axes as the plugin takes them."""
    parts = [np.cos(x), np.sin(x), np.cos(y), np.sin(y), np.cos(z), np.sin(z)]
    if any(p.dtype != np.float64 for p in parts):
        raise NotImplementedError("create_schwarzp: float64 axes only (Python int or float bounds)")
    return np.concatenate([p.ravel() for p in parts])


def _bounds(min_, max_):
    """(span, min_f, fill, fill_error) of image_normalize for a float64 image: float64(max_ - min_) and
    float64(min_), as NumPy promotes Python or NumPy scalars against float64, and min_ converted to int16 as
    `output[:] = min_` converts it. That conversion only happens on a constant image, so its error is returned,
    not raised."""
    for b in (min_, max_):
        if isinstance(b, np.generic):
            ok = isinstance(b, (np.integer, np.floating)) and b.dtype.itemsize <= 8
        else:
            ok = isinstance(b, (int, float))
        if not ok:
            raise NotImplementedError("image_normalize: Python or NumPy int / float bounds only")
    span, min_f = float(np.float64(max_ - min_)), float(np.float64(min_))
    fill = np.zeros((), np.int16)
    try:
        fill[...] = min_
    except (OverflowError, ValueError, TypeError) as e:
        return span, min_f, 0, e
    return span, min_f, int(fill), None


def _check_fill(ws: torch.Tensor, fill_error) -> None:
    """Raise the deferred conversion error of min_ if the image was constant ((imin, imax) lead the workspace)."""
    if fill_error is not None:
        lo, hi = ws[:16].view(torch.float64).tolist()
        if lo == hi:
            raise fill_error


def _download(t: torch.Tensor, dtype) -> np.ndarray:
    out = np.empty(tuple(t.shape), dtype)
    dev.to_host(t, out)
    return out


# ----------------------------------------------------------------------------- TPMS
def create_schwarzp_device(method, init_x, end_x, init_y, end_y, init_z, end_z, sx=256, sy=256, sz=256):
    """create_schwarzp's float64 (sz, sy, sx) field as a CUDA tensor; None for an unknown method."""
    z, y, x = _axes(init_x, end_x, init_y, end_y, init_z, end_z, sx, sy, sz)
    code = _surface_code(method)
    if code is None:
        return None
    tab = _tables(z, y, x)
    dev.require_cuda()
    shape = (z.size, y.size, x.size)
    out = torch.empty(shape, dtype=torch.float64, device="cuda")
    t = torch.from_numpy(tab).to(out.device)
    with torch.cuda.device(out.device):
        _lib.call("b2v_tpms_f64", _p(t), *shape, code, _p(out), _stream())
    return out


def create_schwarzp(method, init_x, end_x, init_y, end_y, init_z, end_z, sx=256, sy=256, sz=256):
    """schwarzp.create_schwarzp: float64 (sz, sy, sx), or None for an unknown method."""
    t = create_schwarzp_device(method, init_x, end_x, init_y, end_y, init_z, end_z, sx, sy, sz)
    return None if t is None else _download(t, np.float64)


def create_schwarzp_i16_device(method, init_x, end_x, init_y, end_y, init_z, end_z, sx=256, sy=256, sz=256,
                               min_=-1000, max_=1000):
    """image_normalize(create_schwarzp(...), min_, max_) as an int16 CUDA tensor, without the float64 field; None
    for an unknown method. An empty field raises NumPy's zero-size reduction ValueError."""
    z, y, x = _axes(init_x, end_x, init_y, end_y, init_z, end_z, sx, sy, sz)
    code = _surface_code(method)
    if code is None:
        return None
    tab = _tables(z, y, x)
    shape = (z.size, y.size, x.size)
    span, min_f, fill, fill_error = _bounds(min_, max_)
    if 0 in shape:
        np.empty(shape).min()   # NumPy's ValueError for a zero-size reduction
    dev.require_cuda()
    out = torch.empty(shape, dtype=torch.int16, device="cuda")
    t = torch.from_numpy(tab).to(out.device)
    ws = dev._workspace(_lib.load().b2v_tpms_i16_workspace_bytes(*shape), out.device)
    with torch.cuda.device(out.device):
        _lib.call("b2v_tpms_i16", _p(t), *shape, code, span, min_f, fill, _p(ws), _p(out), _stream())
    _check_fill(ws, fill_error)
    return out


def create_schwarzp_i16(method, init_x, end_x, init_y, end_y, init_z, end_z, sx=256, sy=256, sz=256, min_=-1000,
                        max_=1000):
    """image_normalize(create_schwarzp(...), min_, max_): the int16 matrix of the dialog's OnOk."""
    t = create_schwarzp_i16_device(method, init_x, end_x, init_y, end_y, init_z, end_z, sx, sy, sz, min_, max_)
    return None if t is None else _download(t, np.int16)


# ----------------------------------------------------------------------------- Blobs
def create_blobs_device(sx=256, sy=256, sz=256, gaussian=5) -> torch.Tensor:
    """schwarzp.create_blobs as a float64 (sz, sy, sx) CUDA tensor: the host draw, uploaded and blurred."""
    random_image = np.random.random((sz, sy, sx))
    sd = float(gaussian)
    dev.require_cuda()
    t = torch.from_numpy(random_image).to("cuda")
    if not sd > 1e-15 or t.numel() == 0:   # gaussian_filter copies the input
        return t
    return filters._gaussian(t, sd, torch.float64)


def create_blobs(sx=256, sy=256, sz=256, gaussian=5) -> np.ndarray:
    """schwarzp.create_blobs: float64 (sz, sy, sx)."""
    return _download(create_blobs_device(sx, sy, sz, gaussian), np.float64)


def create_blobs_i16_device(sx=256, sy=256, sz=256, gaussian=5, min_=-1000, max_=1000) -> torch.Tensor:
    """image_normalize(create_blobs(...), min_, max_) as an int16 CUDA tensor."""
    _bounds(min_, max_)   # bound type errors before the draw
    return image_normalize_device(create_blobs_device(sx, sy, sz, gaussian), min_, max_)


def create_blobs_i16(sx=256, sy=256, sz=256, gaussian=5, min_=-1000, max_=1000) -> np.ndarray:
    """image_normalize(create_blobs(...), min_, max_): the int16 matrix of the dialog's OnOk."""
    return _download(create_blobs_i16_device(sx, sy, sz, gaussian, min_, max_), np.int16)


# ----------------------------------------------------------------------------- image_normalize
def image_normalize_device(t: torch.Tensor, min_=0.0, max_=1.0) -> torch.Tensor:
    """image_normalize of a dense float64 CUDA tensor (any rank) into a new int16 tensor of its shape. An empty
    tensor raises NumPy's zero-size reduction ValueError."""
    dev._dense(t, "image")
    if t.dtype != torch.float64:
        raise TypeError("image_normalize_device: float64 tensor expected")
    span, min_f, fill, fill_error = _bounds(min_, max_)
    if t.numel() == 0:
        np.empty(0).min()   # NumPy's ValueError for a zero-size reduction
    out = torch.empty(t.shape, dtype=torch.int16, device=t.device)
    ws = dev._workspace(_lib.load().b2v_image_normalize_f64_workspace_bytes(t.numel()), t.device)
    with torch.cuda.device(t.device):
        _lib.call("b2v_image_normalize_f64_i16", _p(t), t.numel(), span, min_f, fill, _p(ws), _p(out), _stream())
    _check_fill(ws, fill_error)
    return out


def image_normalize(image, min_=0.0, max_=1.0, output_dtype=np.int16) -> np.ndarray:
    """imagedata_utils.image_normalize for a float32 or float64 image of any rank and an int16 output."""
    a = np.asarray(image)
    if a.dtype == np.float32:
        return voronoi.image_normalize(a, min_, max_, output_dtype)
    if a.dtype != np.float64 or np.dtype(output_dtype) != np.int16:
        raise NotImplementedError(f"image_normalize: float32 / float64 -> int16 only ({a.dtype} -> "
                                  f"{np.dtype(output_dtype)})")
    _bounds(min_, max_)
    if a.size == 0:
        a.min()   # NumPy's ValueError for a zero-size reduction
    return _download(image_normalize_device(dev.to_device(a), min_, max_), np.int16)
