"""Remove non-visible faces (plugins/remove_non_visible_faces/remove_non_visible_faces.py:19-119) on arrays,
with no OpenGL context and no display (C ABI: b2v_visibility_*):

  remove_non_visible_faces(vertices, faces, positions, remove_visible)          numpy in, numpy out
  remove_non_visible_faces_device(vertices, faces, positions, remove_visible)   device tensors

The surface is depth-rendered at 800x800 from a camera along each of `positions` (only the direction
counts), a vertex is visible when some view sees it, and the faces with a selected vertex (a visible one,
or an invisible one with remove_visible=True) are kept in input order and cleaned as vtkCleanPolyData
does: exactly coincident points merged (the first use wins), vertices numbered in order of first use,
faces that degenerate after the merge dropped. No face selected gives an empty mesh.

vertices: float32 [V,3]; faces: int32 / int64 [T,3], or [T,4] with a leading 3 (the Mesh form). The
result has faces of the same dtype and form. The output of mesh.marching_cubes can be passed straight
to the device entry, so the surface never leaves HBM.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from .device import _as_form, _mesh_arrays, _mesh_tensors, _p, _stream, _workspace, require_cuda

DEFAULT_POSITIONS = ((1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1))
MAX_VIEWS = 64


def _positions(positions) -> np.ndarray:
    try:
        p = np.asarray(positions, dtype=np.float64)
    except (TypeError, ValueError):
        raise TypeError("positions: a sequence of 3-component directions expected") from None
    if p.ndim != 2 or p.shape[1] != 3 or not 1 <= len(p) <= MAX_VIEWS:
        raise ValueError(f"positions: 1..{MAX_VIEWS} directions of 3 components expected")
    if not np.isfinite(p).all():
        raise ValueError("positions: every direction must be finite")
    if (p == 0).all(axis=1).any():
        raise ValueError("positions: a zero vector gives no view direction")
    return np.ascontiguousarray(p)


def remove_non_visible_faces_device(vertices: torch.Tensor, faces: torch.Tensor, positions=DEFAULT_POSITIONS,
                                    remove_visible: bool = False, _debug: dict | None = None):
    """(vertices float32 [V',3], faces [T',3|4]) device tensors. Synchronises twice: the vertex bounds and
    the output counts come back to the host. _debug, if a dict, receives the bounds, the camera records,
    and views into the workspace of the depth buffers, the per-vertex visibility and the number of
    triangles the cooperative (large-triangle) path drew."""
    cols = _mesh_tensors(vertices, faces, "remove_non_visible_faces_device")
    p = _positions(positions)
    nv, nt, nviews = vertices.shape[0], faces.shape[0], len(p)
    dev = vertices.device
    if nv == 0:
        if nt:
            raise ValueError("faces: index out of range (there are no vertices)")
        return vertices.new_empty((0, 3)), faces.new_empty((0, cols))
    lib = _lib.load()
    ws = _workspace(lib.b2v_visibility_workspace_bytes(nv, nt, nviews), dev)
    bounds = (C.c_double * 6)()
    cams = np.zeros((nviews, _lib.VIS_CAMERA_DOUBLES), np.float64)
    dptr = C.POINTER(C.c_double)
    nvo, nto = C.c_int64(0), C.c_int64(0)
    i64 = int(faces.dtype == torch.int64)
    with torch.cuda.device(dev):
        _lib.call("b2v_visibility_bounds", _p(vertices), nv, _p(ws), _stream(), bounds)
        _lib.call("b2v_visibility_cameras", bounds, p.ctypes.data_as(dptr), nviews, cams.ctypes.data_as(dptr))
        _lib.call("b2v_visibility_count", _p(vertices), nv, _p(faces), nt, cols, i64, cams.ctypes.data_as(dptr),
                  nviews, int(bool(remove_visible)), _p(ws), _stream(), C.byref(nvo), C.byref(nto))
        vout = torch.empty((nvo.value, 3), dtype=torch.float32, device=dev)
        fout = torch.empty((nto.value, 3), dtype=torch.int32, device=dev)
        if nvo.value or nto.value:
            _lib.call("b2v_visibility_emit", _p(vertices), nv, _p(faces), nt, cols, i64, nviews,
                      int(bool(remove_visible)), _p(ws), _p(vout), _p(fout), _stream())
    if _debug is not None:
        lay = (C.c_int64 * 3)()
        _lib.call("b2v_visibility_layout", nv, nt, nviews, lay)
        _debug["bounds"] = np.array(bounds[:], np.float64)
        _debug["cameras"] = cams
        _debug["zbuf"] = ws[lay[0]:lay[0] + nviews * 800 * 800 * 8].view(torch.float64).view(nviews, 800, 800)
        _debug["visible"] = ws[lay[1]:lay[1] + nv].view(torch.bool)
        _debug["big_triangles"] = ws[lay[2]:lay[2] + 8].view(torch.int64)
    return vout, _as_form(fout, faces.dtype, cols)


def remove_non_visible_faces(vertices, faces, positions=DEFAULT_POSITIONS, remove_visible: bool = False):
    """The plugin's remove_non_visible_faces(polydata, positions, remove_visible) on arrays: returns
    (vertices float32 [V',3], faces) with faces in the input's dtype and form."""
    cols = _mesh_arrays(vertices, faces)
    _positions(positions)
    if not np.isfinite(vertices).all():
        raise ValueError("vertices must be finite")
    if len(faces) == 0:
        return np.zeros((0, 3), np.float32), np.zeros((0, cols), faces.dtype)
    require_cuda()
    v = torch.from_numpy(np.ascontiguousarray(vertices)).cuda()
    f = torch.from_numpy(np.ascontiguousarray(faces)).cuda()
    vo, fo = remove_non_visible_faces_device(v, f, positions, remove_visible)
    return vo.cpu().numpy(), fo.cpu().numpy()
