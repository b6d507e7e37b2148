"""The data preparation of the 3-D volume rendering on the device (C ABI: b2v_raycast_flip_shift_i16,
b2v_vtk_convolve5x5_u16, b2v_histogram_i16). Its caller in InVesalius is Volume (invesalius/data/volume.py):

  LoadVolume          :575-634  vtkImageFlip about the origin on axis 1, GetScalarRange, vtkImageShiftScale to
                                unsigned short with shift abs(min), then ApplyConvolution
  ApplyConvolution    :538-563  one vtkImageConvolve (SetKernel5x5) per entry of the preset's convolutionFilters
  __load_preset       :295-306  ApplyConvolution again on the shifted volume, on every preset change
  CalculateHistogram  :723-735  vtkImageAccumulate over the int16 image, for the transfer-function widget

RaycastingVolume is what the call site holds: the int16 matrix goes up once, only the shifted uint16 volume stays
resident, and each preset change convolves it on the device and brings back one uint16 array for VTK. The
rendering itself (mappers, colour and opacity tables, shading, the cut plane) stays with VTK. The weights come
from the caller, as volume.py computes them ([i / 60.0 for i in Kernels[name]]). Every result equals the
sequential restatement bit for bit; the contract, with VTK's boundary rule restated and unverified, is in the
header of oracle/raycasting.c.

int16 volumes only; other dtypes raise NotImplementedError. A kernel that is not 25 finite, non-negative weights
with 65535 * sum < 65536 raises ValueError.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from . import device as dev
from .device import _dense, _p, _stream


def _i16_volume(t: torch.Tensor, caller: str) -> None:
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{caller}: a torch tensor expected")
    if t.dtype != torch.int16:
        raise NotImplementedError(f"{caller}: int16 volumes only, not {t.dtype}")
    if t.dim() != 3 or t.numel() == 0:
        raise ValueError(f"{caller}: a non-empty 3-D volume expected")
    _dense(t, "t")


def _weights(weights):
    w = np.ascontiguousarray(weights, dtype=np.float64).reshape(-1)
    if w.size != 25:
        raise ValueError(f"convolve5x5: a 5x5 kernel has 25 weights, not {w.size}")
    return w, w.ctypes.data_as(C.POINTER(C.c_double))


def _flip_shift(t: torch.Tensor):
    mm = dev.minmax(t)
    u = torch.empty(t.shape, dtype=torch.uint16, device=t.device)
    with torch.cuda.device(t.device):
        _lib.call("b2v_raycast_flip_shift_i16", _p(t), *t.shape, _p(mm), _p(u), _stream())
    lo, hi = mm.cpu().tolist()
    return u, (float(lo), float(hi))


def flip_shift_device(t: torch.Tensor):
    """(u, (min, max)) of a resident int16 volume [dz][dy][dx]: u uint16 [dz][dy][dx] = the volume flipped along y
    plus abs(min) (LoadVolume's vtkImageFlip and vtkImageShiftScale), and the scalar range as floats (Volume.scale).
    The range stays on the device until the shift has been launched; reading it synchronises."""
    _i16_volume(t, "flip_shift")
    return _flip_shift(t)


def convolve5x5_device(u: torch.Tensor, weights, out: torch.Tensor | None = None) -> torch.Tensor:
    """One vtkImageConvolve pass with SetKernel5x5(weights) over every slice of a resident uint16 volume, into
    `out` (a new tensor when None; never u itself)."""
    if not isinstance(u, torch.Tensor) or u.dtype != torch.uint16 or u.dim() != 3 or u.numel() == 0:
        raise TypeError("convolve5x5: a non-empty 3-D uint16 tensor expected")
    _dense(u, "u")
    w, wp = _weights(weights)
    if out is None:
        out = torch.empty_like(u)
    _dense(out, "out")
    if out.shape != u.shape or out.dtype != u.dtype or out.device != u.device:
        raise ValueError("convolve5x5: out must match u")
    with torch.cuda.device(u.device):
        _lib.call("b2v_vtk_convolve5x5_u16", _p(u), *u.shape, wp, _p(out), _stream())
    return out


def _accumulate(t: torch.Tensor, lo: int, hi: int) -> torch.Tensor:
    """counts[k] = #(t == lo + k) for k < hi - lo: np.histogram's counts (b2v_histogram_i16) with the voxels equal
    to hi taken off the last bin (a one-bin histogram at hi counts them)."""
    r = hi - lo
    counts = torch.empty(r, dtype=torch.int64, device=t.device)
    if r == 0:
        return counts
    top = torch.empty(1, dtype=torch.int64, device=t.device)
    with torch.cuda.device(t.device):
        _lib.call("b2v_histogram_i16", _p(t), t.numel(), lo, r, _p(counts), _stream())
        _lib.call("b2v_histogram_i16", _p(t), t.numel(), hi, 1, _p(top), _stream())
        counts[-1:] -= top
    return counts


def accumulate_histogram_device(t: torch.Tensor):
    """CalculateHistogram on a resident int16 volume: (counts int64 device tensor [r], min, max) with
    r = int(max - min) and counts[k] = #(t == min + k); voxels equal to max are not counted, and a constant
    volume gives no bins. Synchronises (r sizes the output)."""
    _i16_volume(t, "accumulate_histogram")
    lo, hi = (int(v) for v in dev.minmax(t).cpu().tolist())
    return _accumulate(t, lo, hi), float(lo), float(hi)


class RaycastingVolume:
    """The volume rendering's arrays for one Slice.matrix (int16 [dz][dy][dx], memmaps and strided views
    accepted) and its spacing (sx, sy, sz). The matrix is uploaded once; only the shifted uint16 volume stays on
    the device, with one pair of ping-pong buffers for convolution chains, so calls run one at a time.

    .scale               (min, max) of the matrix, floats (Volume.scale)
    .extent / .spacing / .origin   how VTK is to wrap the returned arrays: the flipped image keeps the extent
                         (0, dx-1, 0, dy-1, 0, dz-1) and the spacing, its origin is (0, -(dy-1) sy, 0)
    .imagedata()         the shifted uint16 volume on the host (Volume.imagedata.GetOutput())
    .convolved(kernels)  ApplyConvolution of that volume: one pass per 25-weight kernel, in list order
    .histogram()         CalculateHistogram: (counts int64 [r], init, end), computed at load
    """

    def __init__(self, matrix, spacing, device=None):
        a = np.asarray(matrix)
        if a.dtype != np.int16:
            raise NotImplementedError(f"RaycastingVolume: int16 volumes only, not {a.dtype}")
        if a.ndim != 3 or a.size == 0:
            raise ValueError("RaycastingVolume: a non-empty 3-D volume expected")
        sx, sy, sz = (float(s) for s in spacing)
        dz, dy, dx = a.shape
        self.shape = a.shape
        self.spacing = (sx, sy, sz)
        self.extent = (0, dx - 1, 0, dy - 1, 0, dz - 1)
        self.origin = (0.0, -(dy - 1) * sy, 0.0)
        t = dev.to_device(a, device)
        self._u, self.scale = _flip_shift(t)
        counts = _accumulate(t, int(self.scale[0]), int(self.scale[1]))
        del t
        self._counts = counts.cpu().numpy()
        self._pp: list[torch.Tensor] = []

    def _download(self, t: torch.Tensor) -> np.ndarray:
        out = np.empty(self.shape, np.uint16)
        dev.to_host(t, out)
        return out

    def imagedata(self) -> np.ndarray:
        return self._download(self._u)

    def convolved(self, kernels) -> np.ndarray:
        """The shifted volume after one vtkImageConvolve pass per kernel (each 25 weights, row-major), in list
        order; no kernels gives imagedata(). The resident volume is never modified."""
        src = self._u
        for i, w in enumerate(kernels):
            if len(self._pp) <= min(i, 1):
                self._pp.append(torch.empty_like(self._u))
            src = convolve5x5_device(src, w, self._pp[i % 2])
        return self._download(src)

    def histogram(self):
        return self._counts.copy(), self.scale[0], self.scale[1]
