"""Clean and triangulate surfaces on the device (C ABI: b2v_clean_*, b2v_triangle_filter_*):

  clean_polydata(points, polys, strips=None)             vtkCleanPolyData at InVesalius's settings, numpy
  clean_polydata_device(points, polys, strips=None)      the same on device tensors
  triangle_filter(points, polys=None, strips=None)       vtkTriangleFilter on polys and strips, numpy
  triangle_filter_device(points, polys=None, strips=None)

The clean merges exactly coincident points (float ==, -0 equals +0, a NaN point merges with no other),
numbers the points in order of first use over the polys' then the strips' corners, drops unused points,
removes consecutive repeated points from each cell (and a poly's last point when it repeats its first), and
turns short cells into lower ones: polys of 2 points into lines and of 1 into verts; strips of 3 points into
polys, of 2 into lines, of 1 into verts. The triangle filter copies triangles, splits a strip of n points
into n - 2 triangles with vtkTriangleStrip's alternating winding, and clips a polygon of more than 3 points
with vtkPolygon's ear cut (a polygon it cannot finish gives fewer than n - 2 triangles). The rules are stated in full in the
header of the C checker, clean.c; parity with VTK itself is unpinned.

points: float32 [V,3]. polys and strips each take one of
  - faces int32 / int64 [T,3], or [T,4] with a leading 3 (the form mesh.marching_cubes, compute_normals_device
    and the other device tools return);
  - VTK 9's (offsets, connectivity) pair, from vtk_to_numpy(cells.GetOffsetsArray()) and
    vtk_to_numpy(cells.GetConnectivityArray()).
Results come back in the same forms: polys as faces of the input's dtype and columns when the input polys
were faces and every output poly is a triangle, otherwise as (offsets int64, connectivity) pairs; verts,
lines and strips always as pairs. cell_ids (int64) gives the input cell of every output cell, the polys
numbered before the strips, and the output cells in the order verts, lines, polys, strips (the triangle
filter: its triangles in order).

Verts or lines as input raise NotImplementedError. Malformed offsets and point ids outside [0, V) raise ValueError.
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple

import numpy as np
import torch

from . import _lib
from .device import _dense, _p, _stream, _workspace, require_cuda

_INTS = (torch.int32, torch.int64)


class Cleaned(NamedTuple):
    points: object      # float32 [V',3]
    point_ids: object   # int64 [V']: the input point of each output point
    verts: object       # (offsets, connectivity)
    lines: object       # (offsets, connectivity)
    polys: object       # faces [T,3|4], or (offsets, connectivity)
    strips: object      # (offsets, connectivity)
    cell_ids: object    # int64: the input cell of every output cell (verts, lines, polys, strips)


class Triangles(NamedTuple):
    faces: object       # [T,3|4]
    cell_ids: object    # int64 [T]


class _Cells(NamedTuple):
    conn: torch.Tensor
    offs: torch.Tensor | None
    n: int
    nconn: int
    form: int           # 0: offsets + connectivity; 3 or 4: faces
    i64: int

    def args(self):
        return (_p(self.conn), _p(self.offs), self.n, self.nconn, self.form, self.i64)


def _no_cells(dev) -> _Cells:
    return _Cells(torch.zeros(0, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int64, device=dev),
                  0, 0, 0, 1)


def _cells(x, name: str, dev) -> _Cells:
    if x is None:
        return _no_cells(dev)
    if isinstance(x, (tuple, list)):
        if len(x) != 2:
            raise ValueError(f"{name}: an (offsets, connectivity) pair expected")
        offs, conn = x
        for t, what in ((offs, "offsets"), (conn, "connectivity")):
            if not isinstance(t, torch.Tensor) or t.dtype not in _INTS:
                raise TypeError(f"{name}: {what} must be an int32 or int64 tensor")
            if t.dim() != 1:
                raise ValueError(f"{name}: {what} must be 1-D")
            if t.device != dev:
                raise ValueError(f"{name}: {what} must be on the points' device")
        if offs.numel() == 0:
            if conn.numel():
                raise ValueError(f"{name}: malformed offsets (a connectivity without offsets)")
            return _no_cells(dev)
        offs = offs.to(torch.int64).contiguous()
        conn = conn.contiguous()
        return _Cells(conn, offs, offs.numel() - 1, conn.numel(), 0, int(conn.dtype == torch.int64))
    if not isinstance(x, torch.Tensor):
        raise TypeError(f"{name}: faces [T,3|4] or an (offsets, connectivity) pair expected")
    if x.dtype not in _INTS:
        raise TypeError(f"{name}: int32 or int64 faces expected")
    if x.dim() != 2 or x.shape[1] not in (3, 4):
        raise ValueError(f"{name}: faces [T,3] or [T,4] (leading 3) expected")
    if x.device != dev:
        raise ValueError(f"{name}: faces must be on the points' device")
    _dense(x, name)
    return _Cells(x, None, x.shape[0], 3 * x.shape[0], int(x.shape[1]), int(x.dtype == torch.int64))


def _points(points, caller: str) -> None:
    if not isinstance(points, torch.Tensor):
        raise TypeError(f"{caller}: torch tensors expected")
    if points.dtype != torch.float32 or points.dim() != 2 or points.shape[1] != 3:
        raise ValueError("points: float32 [V,3] expected")
    _dense(points, "points")
    if not points.is_cuda:
        raise ValueError(f"{caller}: points must be a CUDA tensor")


def _refuse(verts, lines) -> None:
    if verts is not None or lines is not None:
        raise NotImplementedError("verts and lines as input are not supported: InVesalius's surfaces have none")


def _out_dtype(p: _Cells, s: _Cells, polys, strips) -> torch.dtype:
    if polys is not None:
        return torch.int64 if p.i64 else torch.int32
    if strips is not None:
        return torch.int64 if s.i64 else torch.int32
    return torch.int64


def _as_faces(tri: torch.Tensor, dtype: torch.dtype, cols: int) -> torch.Tensor:
    f = tri.to(dtype)
    if cols == 4:
        f = torch.cat((torch.full((f.shape[0], 1), 3, dtype=dtype, device=f.device), f), 1)
    return f


def _pair(offs: torch.Tensor, conn: torch.Tensor, dtype: torch.dtype):
    return offs, conn.to(dtype)


def clean_polydata_device(points: torch.Tensor, polys=None, strips=None, *, verts=None, lines=None) -> Cleaned:
    """vtkCleanPolyData on device tensors (see the module's docstring). Synchronises twice: the input check
    and the output counts come back to the host."""
    _refuse(verts, lines)
    _points(points, "clean_polydata_device")
    dev = points.device
    p, s = _cells(polys, "polys", dev), _cells(strips, "strips", dev)
    nv, G, Cn = points.shape[0], p.n + s.n, p.nconn + s.nconn
    lib = _lib.load()
    ws = _workspace(lib.b2v_clean_workspace_bytes(nv, G, Cn), dev)
    cnt = (C.c_int64 * 7)()
    e64 = dict(dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        _lib.call("b2v_clean_count", _p(points), nv, *p.args(), *s.args(), _p(ws), _stream(), cnt)
        npts, nvc, nlc, npc, npk, nsc, nsk = (int(x) for x in cnt)
        pts = torch.empty((npts, 3), dtype=torch.float32, device=dev)
        pid = torch.empty(npts, **e64)
        vconn, lconn = torch.empty(nvc, **e64), torch.empty(2 * nlc, **e64)
        poffs, pconn = torch.empty(npc + 1, **e64), torch.empty(npk, **e64)
        soffs, sconn = torch.empty(nsc + 1, **e64), torch.empty(nsk, **e64)
        cell_ids = torch.empty(nvc + nlc + npc + nsc, **e64)
        _lib.call("b2v_clean_emit", _p(points), nv, *p.args(), *s.args(), _p(ws), _p(pts), _p(pid), _p(vconn),
                  _p(lconn), _p(poffs), _p(pconn), _p(soffs), _p(sconn), _p(cell_ids), _stream())
    dt = _out_dtype(p, s, polys, strips)
    if p.form and npk == 3 * npc:   # faces in, and every poly is still a triangle
        out_polys = _as_faces(pconn.view(npc, 3), dt, p.form)
    else:
        out_polys = _pair(poffs, pconn, dt)
    return Cleaned(pts, pid, _pair(torch.arange(nvc + 1, **e64), vconn, dt),
                   _pair(torch.arange(0, 2 * nlc + 1, 2, **e64), lconn, dt), out_polys, _pair(soffs, sconn, dt),
                   cell_ids)


def triangle_filter_device(points: torch.Tensor, polys=None, strips=None, *, verts=None, lines=None) -> Triangles:
    """vtkTriangleFilter on device tensors (see the module's docstring). Synchronises twice."""
    _refuse(verts, lines)
    _points(points, "triangle_filter_device")
    dev = points.device
    p, s = _cells(polys, "polys", dev), _cells(strips, "strips", dev)
    nv = points.shape[0]
    lib = _lib.load()
    ws = _workspace(lib.b2v_triangle_filter_workspace_bytes(p.n + s.n, p.nconn), dev)
    cnt = (C.c_int64 * 1)()
    with torch.cuda.device(dev):
        _lib.call("b2v_triangle_filter_count", _p(points), nv, *p.args(), *s.args(), _p(ws), _stream(), cnt)
        nt = int(cnt[0])
        tris = torch.empty((nt, 3), dtype=torch.int64, device=dev)
        cell_ids = torch.empty(nt, dtype=torch.int64, device=dev)
        if nt:
            _lib.call("b2v_triangle_filter_emit", _p(points), nv, *p.args(), *s.args(), _p(ws), _p(tris),
                      _p(cell_ids), _stream())
    return Triangles(_as_faces(tris, _out_dtype(p, s, polys, strips), p.form if p.form else 3), cell_ids)


# ----------------------------------------------------------------------------- numpy entries
def _to_dev(x, name: str):
    if x is None:
        return None
    if isinstance(x, (tuple, list)):
        if len(x) != 2:
            raise ValueError(f"{name}: an (offsets, connectivity) pair expected")
        return tuple(_to_dev(a, name) for a in x)
    if not isinstance(x, np.ndarray) or x.dtype not in (np.int32, np.int64):
        raise TypeError(f"{name}: int32 or int64 numpy arrays expected")
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _to_np(x):
    if isinstance(x, tuple):
        return tuple(_to_np(a) for a in x)
    return x.cpu().numpy()


def _points_np(points) -> torch.Tensor:
    if not isinstance(points, np.ndarray) or points.dtype != np.float32 or points.ndim != 2 or points.shape[1] != 3:
        raise TypeError("points: a float32 numpy array [V,3] expected")
    require_cuda()
    return torch.from_numpy(np.ascontiguousarray(points)).cuda()


def clean_polydata(points, polys=None, strips=None, *, verts=None, lines=None) -> Cleaned:
    """vtkCleanPolyData on numpy arrays (see the module's docstring)."""
    _refuse(verts, lines)
    r = clean_polydata_device(_points_np(points), _to_dev(polys, "polys"), _to_dev(strips, "strips"))
    return Cleaned(*(_to_np(x) for x in r))


def triangle_filter(points, polys=None, strips=None, *, verts=None, lines=None) -> Triangles:
    """vtkTriangleFilter on numpy arrays (see the module's docstring)."""
    _refuse(verts, lines)
    r = triangle_filter_device(_points_np(points), _to_dev(polys, "polys"), _to_dev(strips, "strips"))
    return Triangles(*(_to_np(x) for x in r))
