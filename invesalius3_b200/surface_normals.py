"""Surface normals (vtkPolyDataNormals) and volume and area (vtkMassProperties) on arrays, restated on the
device (C ABI: b2v_normals_*, b2v_mass_properties). Their callers in InVesalius:

  surface_process.join_process_surface       feature angle 80, auto-orientation, cell normals
  surface_process (context-aware smoothing)  VTK's defaults (30 degrees) plus cell normals
  surface.CreateSurfaceFromPolydata, OnLoadSurfaceDict, surface export, viewer_volume
                                             feature angle 80, auto-orientation
  brainmesh_handler                          feature angle 160
  surface_process / surface.py / polydata_utils.CalculateSurfaceVolume, CalculateSurfaceArea
                                             the volume and area of the surface panel

Consistent ordering, splitting and non-manifold traversal are always on, as every caller sets them. The
defaults are VTK's. compute_normals_device and mass_properties_device take device tensors, so the output of
mesh.marching_cubes, the smoother or fill_holes_device never leaves HBM. The result equals the sequential
filter bit for bit (the contract, restated and unverified against VTK, is in DESIGN.md §3).

vertices: float32 [V,3]; faces: int32 / int64 [T,3], or [T,4] with a leading 3. The feature angle is clamped
to [0, 180] as SetFeatureAngle does; NaN and a face id outside [0, V) raise ValueError.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from .device import _mesh_arrays, _mesh_tensors, _p, _stream, _workspace, require_cuda


@dataclass
class Normals:
    """One run of the filter. points: float32 [V + new_points, 3], the input's points first and then the
    copies made by splitting; faces: the input's dtype and form, each cell in its final order on the split
    points; point_normals float32 [V + new_points, 3]; cell_normals float32 [T, 3]; flips: cells reversed;
    new_points; regions: traversals run; waves: the most waves one traversal took. Tensors are on the
    input's device."""
    points: torch.Tensor
    faces: torch.Tensor
    point_normals: torch.Tensor
    cell_normals: torch.Tensor
    flips: int
    new_points: int
    regions: int
    waves: int


def _angle(feature_angle) -> float:
    a = float(feature_angle)
    if math.isnan(a):
        raise ValueError("compute_normals: the feature angle is NaN")
    return a


def compute_normals_device(vertices: torch.Tensor, faces: torch.Tensor, feature_angle: float = 30.0,
                           auto_orient: bool = False) -> Normals:
    """vtkPolyDataNormals on device tensors. Synchronises: the counts come back to the host."""
    cols = _mesh_tensors(vertices, faces, "compute_normals")
    a = _angle(feature_angle)
    nv, nt, dev = vertices.shape[0], faces.shape[0], vertices.device
    lib = _lib.load()
    ws = _workspace(lib.b2v_normals_workspace_bytes(nv, nt), dev)
    counts = (C.c_int64 * 4)()
    i64 = int(faces.dtype == torch.int64)
    with torch.cuda.device(dev):
        _lib.call("b2v_normals_count", _p(vertices), nv, _p(faces), nt, cols, i64, a, int(bool(auto_orient)),
                  _p(ws), _stream(), counts)
        n = nv + counts[2]
        pts = torch.empty((n, 3), dtype=torch.float32, device=dev)
        pn = torch.empty((n, 3), dtype=torch.float32, device=dev)
        out = torch.empty((nt, cols), dtype=faces.dtype, device=dev)
        cn = torch.empty((nt, 3), dtype=torch.float32, device=dev)
        _lib.call("b2v_normals_emit", _p(vertices), nv, nt, cols, i64, counts, _p(ws), _p(pts), _p(out), _p(pn),
                  _p(cn), _stream())
    return Normals(pts, out, pn, cn, counts[1], counts[2], counts[0], counts[3])


def compute_normals(vertices: np.ndarray, faces: np.ndarray, feature_angle: float = 30.0,
                    auto_orient: bool = False):
    """vtkPolyDataNormals on numpy arrays: (points, faces, point_normals, cell_normals, flips, new_points)."""
    _mesh_arrays(vertices, faces)
    _angle(feature_angle)
    require_cuda()
    r = compute_normals_device(torch.from_numpy(np.ascontiguousarray(vertices)).cuda(),
                               torch.from_numpy(np.ascontiguousarray(faces)).cuda(), feature_angle, auto_orient)
    return (r.points.cpu().numpy(), r.faces.cpu().numpy(), r.point_normals.cpu().numpy(),
            r.cell_normals.cpu().numpy(), r.flips, r.new_points)


def mass_properties_device(vertices: torch.Tensor, faces: torch.Tensor) -> tuple[float, float]:
    """vtkMassProperties on device tensors: (volume, area). Synchronises."""
    cols = _mesh_tensors(vertices, faces, "mass_properties")
    nv, nt, dev = vertices.shape[0], faces.shape[0], vertices.device
    lib = _lib.load()
    ws = _workspace(lib.b2v_normals_workspace_bytes(nv, nt), dev)
    out = (C.c_double * 2)()
    with torch.cuda.device(dev):
        _lib.call("b2v_mass_properties", _p(vertices), nv, _p(faces), nt, cols, int(faces.dtype == torch.int64),
                  _p(ws), _stream(), out)
    return out[0], out[1]


def mass_properties(vertices: np.ndarray, faces: np.ndarray) -> tuple[float, float]:
    """vtkMassProperties on numpy arrays: (volume, area), as CalculateSurfaceVolume / CalculateSurfaceArea."""
    _mesh_arrays(vertices, faces)
    require_cuda()
    return mass_properties_device(torch.from_numpy(np.ascontiguousarray(vertices)).cuda(),
                                  torch.from_numpy(np.ascontiguousarray(faces)).cuda())
