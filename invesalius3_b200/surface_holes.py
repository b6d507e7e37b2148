"""Surface hole filling (vtkFillHolesFilter) on arrays, restated on the device (C ABI: b2v_holes_*). Its
callers in InVesalius:

  polydata_utils.ApplySmoothFilter ("Smooth surface")   HoleSize 1000, after the smoother
  surface_process.join_process_surface ("Fill holes")   HoleSize 300
  FillSurfaceHole                                       HoleSize 500
  markers/surface_geometry                              after the smoother

fill_holes(vertices, faces, hole_size) takes numpy arrays and returns the faces; fill_holes_device does the
same on device tensors (the output of mesh.marching_cubes or the smoother never leaves HBM) and also reports
the boundary lines and every traced loop. The points never change: the faces are the input's, in their
order, followed by the new triangles. The default hole size is VTK's. The result equals the sequential filter
bit for bit (the contract, restated and unverified against VTK, is in DESIGN.md §3).

vertices: float32 [V,3]; faces: int32 / int64 [T,3], or [T,4] with a leading 3. The hole size is clamped to
[0, FLT_MAX] as SetHoleSize does; NaN and a face id outside [0, V) raise ValueError.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from .device import _mesh_arrays, _mesh_tensors, _p, _stream, _workspace, require_cuda

# a loop's status, as HoleFilling.status reports it
FILLED, FAILED, TOO_LARGE = 0, 1, 2


@dataclass
class HoleFilling:
    """One run of the filter. faces: the input's dtype and form, [T + N, 3 or 4], the input faces first;
    lines: the number of boundary lines; per traced loop, in the order of its first line: first_line and
    points (int64), radius (float64, the bounding sphere's) and status (int8: FILLED, FAILED when no ear
    qualifies or the loop has fewer than 3 points, TOO_LARGE when the radius exceeds the hole size). All
    tensors are on the input's device."""
    faces: torch.Tensor
    lines: int
    first_line: torch.Tensor
    points: torch.Tensor
    radius: torch.Tensor
    status: torch.Tensor


def _hole_size(hole_size) -> float:
    h = float(hole_size)
    if math.isnan(h):
        raise ValueError("fill_holes: the hole size is NaN")
    return min(max(h, 0.0), float(np.finfo(np.float32).max))


def fill_holes_device(vertices: torch.Tensor, faces: torch.Tensor, hole_size: float = 1.0) -> HoleFilling:
    """vtkFillHolesFilter on device tensors. Synchronises: the counts come back to the host."""
    cols = _mesh_tensors(vertices, faces, "fill_holes")
    h = _hole_size(hole_size)
    nv, nt, dev = vertices.shape[0], faces.shape[0], vertices.device
    lib = _lib.load()
    ws = _workspace(lib.b2v_holes_workspace_bytes(nv, nt), dev)
    counts = (C.c_int64 * 3)()
    i64 = int(faces.dtype == torch.int64)
    with torch.cuda.device(dev):
        _lib.call("b2v_holes_count", _p(vertices), nv, _p(faces), nt, cols, i64, h, _p(ws), _stream(), counts)
        nl, nloop, ntri = counts[0], counts[1], counts[2]
        out = torch.empty((nt + ntri, cols), dtype=faces.dtype, device=dev)
        first = torch.empty(nloop, dtype=torch.int64, device=dev)
        points = torch.empty(nloop, dtype=torch.int64, device=dev)
        radius = torch.empty(nloop, dtype=torch.float64, device=dev)
        status = torch.empty(nloop, dtype=torch.int8, device=dev)
        _lib.call("b2v_holes_emit", _p(faces), nv, nt, cols, i64, counts, _p(ws), _p(out), _p(first), _p(points),
                  _p(radius), _p(status), _stream())
    return HoleFilling(out, nl, first, points, radius, status)


def fill_holes(vertices: np.ndarray, faces: np.ndarray, hole_size: float = 1.0) -> np.ndarray:
    """vtkFillHolesFilter on numpy arrays: the faces, in the input's dtype and form, the input faces first."""
    _mesh_arrays(vertices, faces)
    _hole_size(hole_size)
    require_cuda()
    r = fill_holes_device(torch.from_numpy(np.ascontiguousarray(vertices)).cuda(),
                          torch.from_numpy(np.ascontiguousarray(faces)).cuda(), hole_size)
    return r.faces.cpu().numpy()
