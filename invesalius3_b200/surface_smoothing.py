"""Laplacian surface smoothing (vtkSmoothPolyDataFilter) on arrays, restated on the device (C ABI:
b2v_smooth_*). Its callers in InVesalius:

  polydata_utils.ApplySmoothFilter ("Smooth surface")   iterations=20, relaxation_factor=0.4,
                                                        feature_angle=80, boundary_smoothing=False
  surface.decimate_polydata                             iterations=15, VTK's defaults otherwise
  markers/surface_geometry                              a caller-set iteration count and relaxation,
                                                        boundary_smoothing=False

smooth_polydata(vertices, faces, ...) takes numpy arrays and returns the moved float32 vertices; the faces
and the point ids do not change, so point data carries over as it is. smooth_polydata_device does the same
on device tensors (the output of mesh.marching_cubes never leaves HBM) and also returns the point types and
the number of iterations done. The defaults are VTK's. The result equals VTK's sequential, in-place sweep in
ascending point id bit for bit (the contract, restated and unverified against VTK, is in DESIGN.md §3).

vertices: float32 [V,3]; faces: int32 / int64 [T,3], or [T,4] with a leading 3. As in VTK, the angles are
clamped to [0, 180] degrees and the convergence to [0, 1]. Non-float32 vertices, a face id outside [0, V)
and a negative iteration count raise ValueError.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from .device import _face_form, _p, _stream, _workspace, require_cuda

# VTK's vertex codes, as point_types reports them
SIMPLE, FIXED, FEATURE_EDGE, BOUNDARY_EDGE = 0, 1, 2, 3


@dataclass
class Smoothing:
    """One run of the filter. vertices float32 [V,3]; point_types int8 [V] (VTK's codes above);
    iterations: the iterations done (fewer than asked when the convergence test stopped the sweep);
    levels: the dependency levels of one iteration; steps: levels x iterations, the length of the device's
    schedule."""
    vertices: torch.Tensor
    point_types: torch.Tensor
    iterations: int
    levels: int
    steps: int


def _cosine(angle: float) -> float:
    return math.cos(min(max(float(angle), 0.0), 180.0) * (math.pi / 180.0))


def _check(vertices, faces, iterations):
    if vertices.dtype not in (torch.float32, np.float32):
        raise ValueError("vertices: float32 expected")
    if faces.dtype not in (torch.int32, torch.int64, np.int32, np.int64):
        raise ValueError("faces: int32 or int64 expected")
    if len(vertices.shape) != 2 or vertices.shape[1] != 3:
        raise ValueError("vertices: [V,3] expected")
    if int(iterations) < 0:
        raise ValueError("smoothing: the number of iterations must be >= 0")
    return _face_form(tuple(faces.shape))


def smooth_polydata_device(vertices: torch.Tensor, faces: torch.Tensor, iterations: int = 20,
                           relaxation_factor: float = 0.01, feature_angle: float = 45.0, edge_angle: float = 15.0,
                           feature_edge_smoothing: bool = False, boundary_smoothing: bool = True,
                           convergence: float = 0.0) -> Smoothing:
    """vtkSmoothPolyDataFilter on device tensors. Synchronises: the iteration count comes back to the host."""
    if not isinstance(vertices, torch.Tensor) or not isinstance(faces, torch.Tensor):
        raise TypeError("smoothing: torch tensors expected")
    cols = _check(vertices, faces, iterations)
    for t, name in ((vertices, "vertices"), (faces, "faces")):
        if not t.is_cuda or not t.is_contiguous():
            raise ValueError(f"{name} must be a dense CUDA tensor")
    if faces.device != vertices.device:
        raise ValueError("vertices and faces must be on the same device")
    nv, nt, dev = vertices.shape[0], faces.shape[0], vertices.device
    lib = _lib.load()
    ws = _workspace(lib.b2v_smooth_workspace_bytes(nv, nt), dev)
    bounds = (C.c_double * 6)()
    counts = (C.c_int64 * 3)()
    out = torch.empty_like(vertices)
    with torch.cuda.device(dev):
        _lib.call("b2v_smooth_analyse", _p(vertices), nv, _p(faces), nt, cols, int(faces.dtype == torch.int64),
                  _cosine(feature_angle), _cosine(edge_angle), int(bool(feature_edge_smoothing)),
                  int(bool(boundary_smoothing)), _p(ws), _stream(), bounds, counts)
        levels = counts[1]
        dx, dy, dz = bounds[1] - bounds[0], bounds[3] - bounds[2], bounds[5] - bounds[4]
        conv = min(max(float(convergence), 0.0), 1.0) * math.sqrt(dx * dx + dy * dy + dz * dz)
        run = (C.c_int64 * 3)()
        _lib.call("b2v_smooth_run", _p(vertices), nv, nt, int(iterations), float(relaxation_factor), conv, _p(ws),
                  _p(out), _stream(), run)
        if nv:
            lay = (C.c_int64 * 6)()
            _lib.call("b2v_smooth_layout", nv, nt, lay)
            types = ws[lay[0]:lay[0] + nv].view(torch.int8).clone()
        else:
            types = torch.empty(0, dtype=torch.int8, device=dev)
    return Smoothing(out, types, run[0], levels, run[1])


def smooth_polydata(vertices: np.ndarray, faces: np.ndarray, iterations: int = 20, relaxation_factor: float = 0.01,
                    feature_angle: float = 45.0, edge_angle: float = 15.0, feature_edge_smoothing: bool = False,
                    boundary_smoothing: bool = True, convergence: float = 0.0) -> np.ndarray:
    """vtkSmoothPolyDataFilter on numpy arrays: the moved vertices, float32 [V,3], in input point order."""
    if not isinstance(vertices, np.ndarray) or not isinstance(faces, np.ndarray):
        raise TypeError("smoothing: numpy arrays expected")
    _check(vertices, faces, iterations)
    require_cuda()
    r = smooth_polydata_device(torch.from_numpy(np.ascontiguousarray(vertices)).cuda(),
                               torch.from_numpy(np.ascontiguousarray(faces)).cuda(), iterations, relaxation_factor,
                               feature_angle, edge_angle, feature_edge_smoothing, boundary_smoothing, convergence)
    return r.vertices.cpu().numpy()


# polydata_utils.ApplySmoothFilter: the smoother with these settings, then vtkFillHolesFilter at HoleSize 1000
_APPLY_SMOOTH = dict(feature_angle=80.0, feature_edge_smoothing=False, boundary_smoothing=False)
_APPLY_SMOOTH_HOLE_SIZE = 1000.0


def apply_smooth_filter_device(vertices: torch.Tensor, faces: torch.Tensor, iterations: int,
                               relaxation_factor: float) -> tuple[torch.Tensor, torch.Tensor]:
    """ApplySmoothFilter ("Smooth surface") on device tensors: (smoothed vertices, faces with the holes of
    radius <= 1000 filled, in the input's dtype and form). Synchronises."""
    from .surface_holes import fill_holes_device
    s = smooth_polydata_device(vertices, faces, iterations, relaxation_factor, **_APPLY_SMOOTH)
    return s.vertices, fill_holes_device(s.vertices, faces, _APPLY_SMOOTH_HOLE_SIZE).faces


def apply_smooth_filter(vertices: np.ndarray, faces: np.ndarray, iterations: int,
                        relaxation_factor: float) -> tuple[np.ndarray, np.ndarray]:
    """ApplySmoothFilter ("Smooth surface") on numpy arrays: (float32 [V,3] vertices, faces)."""
    if not isinstance(vertices, np.ndarray) or not isinstance(faces, np.ndarray):
        raise TypeError("smoothing: numpy arrays expected")
    _check(vertices, faces, iterations)
    require_cuda()
    v, f = apply_smooth_filter_device(torch.from_numpy(np.ascontiguousarray(vertices)).cuda(),
                                      torch.from_numpy(np.ascontiguousarray(faces)).cuda(), iterations,
                                      relaxation_factor)
    return v.cpu().numpy(), f.cpu().numpy()
