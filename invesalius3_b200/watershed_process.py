"""do_watershed with the reference's signature (invesalius/data/watershed_process.py:19-60)
on the sm_90a kernels of libb2v.so (b2v_ws_*), plus the device-level pieces.

Cost model and labelling rule: include/b2v.h (b2v_ws_flood) and DESIGN.md section 6. The
LUT and the morphological gradient are bit-exact against NumPy / SciPy; the flood computes
the exact minimax cost field of the chosen algorithm and resolves label ties
deterministically (hops, then smaller label) where the reference follows its queue order.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from . import device as dev
from .device import _dense, _p, _stream, _workspace

ALGORITHMS = {"Watershed": 1, "Watershed IFT": 0}


def _sizes(mg_size, ndim=3):
    if np.isscalar(mg_size):
        return (int(mg_size),) * ndim
    s = tuple(int(v) for v in mg_size)
    if len(s) != ndim:
        raise RuntimeError("sequence argument must have length equal to input rank")  # SciPy's message
    return s


def lut_u16(image: torch.Tensor, ww, wl) -> torch.Tensor:
    """get_LUT_value(image, ww, wl).astype('uint16') (uint16 bits in an int16 tensor)."""
    _dense(image, "image")
    if image.dtype != torch.int16:
        raise TypeError("watershed: image must be int16")
    out = torch.empty_like(image)
    with torch.cuda.device(image.device):
        _lib.call("b2v_ws_lut_i16", _p(image), image.numel(), float(ww), float(wl), _p(out), _stream())
    return out


def shift_u16(image: torch.Tensor) -> torch.Tensor:
    """(image - image.min()).astype('uint16')."""
    _dense(image, "image")
    if image.dtype != torch.int16:
        raise TypeError("watershed: image must be int16")
    out = torch.empty_like(image)
    nz, ny, nx = image.shape
    ws = _workspace(_lib.load().b2v_ws_workspace_bytes(nz, ny, nx), image.device)
    with torch.cuda.device(image.device):
        _lib.call("b2v_ws_shift_i16", _p(image), image.numel(), _p(out), _p(ws), _stream())
    return out


def morphological_gradient_u16(pre: torch.Tensor, size) -> torch.Tensor:
    """scipy.ndimage.morphological_gradient(pre_uint16, size) on uint16 bits."""
    _dense(pre, "pre")
    sz, sy, sx = _sizes(size)
    out = torch.empty_like(pre)
    nz, ny, nx = pre.shape
    with torch.cuda.device(pre.device):
        _lib.call("b2v_ws_morph_gradient_u16", _p(pre), nz, ny, nx, sz, sy, sx, _p(out), _stream())
    return out


def flood(cost_u16: torch.Tensor, markers_i16: torch.Tensor, bstruct, algorithm: str, return_ambiguous: bool = False):
    """Marker flood; returns int16 labels (and, with return_ambiguous, the uint8 mask of the voxels
    whose label depends on the reference's queue order). Synchronises."""
    _dense(cost_u16, "cost"); _dense(markers_i16, "markers")
    if markers_i16.dtype != torch.int16 or markers_i16.shape != cost_u16.shape:
        raise TypeError("watershed: markers must be int16 with the image's shape")
    st = np.ascontiguousarray(bstruct, dtype=np.uint8)
    if st.ndim != 3:
        raise RuntimeError("structure and input must have equal rank")
    nz, ny, nx = cost_u16.shape
    labels = torch.empty_like(markers_i16)
    amb = torch.empty(markers_i16.shape, dtype=torch.uint8, device=cost_u16.device) if return_ambiguous else None
    ws = _workspace(_lib.load().b2v_ws_workspace_bytes(nz, ny, nx), cost_u16.device)
    rounds = C.c_int(0)
    with torch.cuda.device(cost_u16.device):
        _lib.call("b2v_ws_flood", _p(cost_u16), _p(markers_i16), nz, ny, nx, C.c_void_p(st.ctypes.data), *st.shape,
                  ALGORITHMS[algorithm], _p(labels), _p(amb), _p(ws), _stream(), C.byref(rounds))
    global LAST_ROUNDS
    LAST_ROUNDS = rounds.value
    return (labels, amb) if return_ambiguous else labels


LAST_ROUNDS = 0   # rounds of the last flood (diagnostics)


def watershed_device(image: torch.Tensor, markers: torch.Tensor, bstruct, algorithm, mg_size, use_ww_wl, wl, ww,
                     return_ambiguous: bool = False):
    """The array-level body of do_watershed on device tensors; returns int16 labels (with
    return_ambiguous: (labels, uint8 mask of order-dependent voxels))."""
    if algorithm not in ALGORITHMS:
        algorithm = "Watershed IFT"  # the reference's `else` branch
    pre = lut_u16(image, ww, wl) if use_ww_wl else shift_u16(image)
    if algorithm == "Watershed":
        pre = morphological_gradient_u16(pre, mg_size)
    mk = markers.to(torch.int16)
    if algorithm == "Watershed IFT" and not use_ww_wl:
        mk = mk.to(torch.int8).to(torch.int16)  # markers.astype('int8'), watershed_process.py:57
    return flood(pre, mk.contiguous(), bstruct, algorithm, return_ambiguous)


def do_watershed(image, markers, tfile, shape, bstruct, algorithm, mg_size, use_ww_wl, wl, ww, q) -> None:
    """Same protocol as the reference: the result goes into the uint8 memmap `tfile` of
    shape `shape`, then `q.put(1)`."""
    mask = np.memmap(tfile, shape=shape, dtype="uint8", mode="r+")
    image = np.asarray(image)
    if image.dtype != np.int16:
        raise TypeError("do_watershed: image must be int16")
    img = dev.to_device(image if image.ndim == 3 else image[None])
    mk_np = np.asarray(markers)
    mk = dev.to_device(np.ascontiguousarray(mk_np if mk_np.ndim == 3 else mk_np[None]).astype(np.int16))
    st = np.asarray(bstruct)
    if st.ndim == 2:
        st = st[None]
    labels = watershed_device(img, mk, st, algorithm, mg_size if image.ndim == 3 else (1,) + _sizes(mg_size, 2),
                              use_ww_wl, wl, ww)
    res = labels.cpu().numpy().reshape(image.shape)
    mask[:] = res
    mask.flush()
    q.put(1)
