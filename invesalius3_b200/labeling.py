"""Connected components on the device, with the signatures InVesalius uses (SURVEY 8f-3):

  label(input, structure, output=np.uint32)     scipy.ndimage.label   mask.py:526-530, 549-552
  count_regions(image, number_regions)          invesalius_rs.count_regions   count_regions.rs:5-18
                                                (int16, int32, int64 or uint8 labels)
  get_largest_connected_component(image)        imagedata_utils.py:717-721
  fill_holes_auto(matrix, conn, size)           the body of Mask.fill_holes_auto (mask.py:519-562):
                                                labelling and filling without leaving the device

Labels are numbered like SciPy's (raster order of each component's first voxel), so everything
downstream (fill_holes_automatically's size table, argmax of bincount) sees the same numbers.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from . import device as dev
from .device import _dense, _p, _stream, _workspace


def _structure(structure, ndim):
    if structure is None:
        from scipy.ndimage import generate_binary_structure
        structure = generate_binary_structure(ndim, 1)
    st = np.ascontiguousarray(structure, dtype=np.uint8)
    if st.ndim != ndim:
        raise RuntimeError("structure and input must have equal rank")     # SciPy's message
    while st.ndim < 3:
        st = st[None]
    return st


def label_device(fg: torch.Tensor, structure) -> tuple[torch.Tensor, int]:
    """fg: uint8 / bool device tensor [nz][ny][nx], non-zero = feature. Returns (labels as an int32
    tensor holding the uint32 label image, number of labels)."""
    if fg.dtype == torch.bool:
        fg = fg.to(torch.uint8)
    _dense(fg, "input")
    if fg.dtype != torch.uint8 or fg.dim() != 3:
        raise TypeError("label: 3-D uint8 / bool tensor expected")
    st = _structure(structure, 3)
    nz, ny, nx = fg.shape
    labels = torch.empty(fg.shape, dtype=torch.int32, device=fg.device)
    ws = _workspace(_lib.load().b2v_label_workspace_bytes(fg.numel()), fg.device)
    n = C.c_int64(0)
    with torch.cuda.device(fg.device):
        _lib.call("b2v_label", _p(fg), nz, ny, nx, C.c_void_p(st.ctypes.data), *st.shape, _p(labels), _p(ws), _stream(),
                  C.byref(n))
    return labels, int(n.value)


def label(input, structure=None, output=np.uint32):
    """scipy.ndimage.label for 2-D / 3-D inputs: (labels, num_features)."""
    a = np.asarray(input)
    if a.ndim not in (2, 3):
        raise NotImplementedError("label: 2-D or 3-D input")
    st = _structure(structure, a.ndim)
    a3 = a if a.ndim == 3 else a[None]
    fg = dev.to_device(np.ascontiguousarray(a3 != 0).view(np.uint8))
    lab, n = label_device(fg, st)
    res = np.empty(a3.shape, np.uint32)
    dev.to_host(lab, res.view(np.int32))
    return res.reshape(a.shape).astype(output, copy=False), n


# label images count_regions takes: the crate's int16 / int32 / int64 (nd.label returns int32) and uint8
_LABEL_DT = {torch.int16: _lib.I16, torch.uint8: _lib.U8, torch.int32: _lib.I32, torch.int64: _lib.I64}


def _label_code(t: torch.Tensor) -> int:
    _dense(t, "image")
    try:
        return _LABEL_DT[t.dtype]
    except KeyError:
        raise TypeError("count_regions: int16, int32, int64 or uint8 image expected") from None


def count_regions_device(t: torch.Tensor, number_regions: int) -> torch.Tensor:
    """count_regions on a dense device label image: an int32 tensor holding the uint32 region sizes.
    A value outside [0, number_regions] raises ValueError. Synchronises."""
    code = _label_code(t)
    out = torch.empty(t.shape, dtype=torch.int32, device=t.device)
    ws = _workspace(256 + 4 * (int(number_regions) + 1), t.device)
    with torch.cuda.device(t.device):
        _lib.call("b2v_count_regions", _p(t), code, t.numel(), int(number_regions), _p(out), _p(ws), _stream())
    return out


def region_sizes_device(t: torch.Tensor, number_regions: int) -> torch.Tensor:
    """The size table of count_regions: an int32 tensor [number_regions + 1] holding the uint32 number of
    voxels of each value. A value outside [0, number_regions] raises ValueError. Synchronises."""
    code = _label_code(t)
    sizes = torch.empty(int(number_regions) + 1, dtype=torch.int32, device=t.device)
    ws = _workspace(256, t.device)
    with torch.cuda.device(t.device):
        _lib.call("b2v_region_sizes", _p(t), code, t.numel(), int(number_regions), _p(sizes), _p(ws), _stream())
    return sizes


def count_regions(image: np.ndarray, number_regions: int) -> np.ndarray:
    """invesalius_rs.count_regions (invesalius_rs/__init__.py:108-111): uint32 image of region sizes, for
    int16, int32, int64 or uint8 labels."""
    a = np.asarray(image)
    if a.dtype not in (np.int16, np.int32, np.int64, np.uint8) or a.ndim != 3:
        raise TypeError("count_regions: int16, int32, int64 or uint8 3-D image expected")
    out = count_regions_device(dev.to_device(a), number_regions)
    res = np.empty(a.shape, np.uint32)
    dev.to_host(out, res.view(np.int32))
    return res


def get_largest_connected_component(image: np.ndarray) -> np.ndarray:
    """imagedata_utils.py:717-721: labels == argmax(bincount(labels)[1:]) + 1 (ties: the smaller label)."""
    a = np.asarray(image)
    a3 = a if a.ndim == 3 else a[None]
    fg = dev.to_device(np.ascontiguousarray(a3 != 0).view(np.uint8))
    lab, n = label_device(fg, _structure(None, 3) if a.ndim == 3 else _structure(None, 2))
    assert n != 0
    sizes = torch.bincount(lab.reshape(-1), minlength=n + 1)[1:]
    best = int(torch.argmax(sizes).item()) + 1       # torch.argmax returns the first maximum, like NumPy's
    res = np.empty(a3.shape, np.uint8)
    dev.to_host((lab == best).to(torch.uint8), res)
    return res.reshape(a.shape).astype(bool)


def fill_holes_auto(matrix: np.ndarray, conn: int, size: int) -> bool:
    """Mask.fill_holes_auto, 3-D target (mask.py:523-537) on the mask body `matrix`
    (= mask.matrix[1:, 1:, 1:], rewritten in place): label the unselected voxels, fill the components
    of at most `size` voxels with 254. Returns whether anything qualified."""
    from scipy.ndimage import generate_binary_structure
    if matrix.dtype != np.uint8 or matrix.ndim != 3:
        raise TypeError("Invalid mask type")
    st = generate_binary_structure(3, {6: 1, 18: 2, 26: 3}[conn])
    m = dev.to_device(matrix)
    lab, n = label_device((~(m > 127)).to(torch.uint8), st)
    if n == 0:
        return False
    ret = dev.fill_holes_automatically(m, lab, n, int(size))
    if ret:
        dev.to_host(m, matrix)
    return ret
