"""The geodesic ("curved") surface measurement of the 3-D viewer on the device (C ABI: b2v_geodesic_*,
b2v_closest_points). Its caller in InVesalius is GeodesicMeasure._draw_line (measures.py:1202-1273), run on every
click and every drag of a point by CurvedMeasureInteractorStyle (styles_3d.py:647-771): for each pair of
consecutive picks, vtkPointLocator::FindClosestPoint snaps both picks to the surface, vtkDijkstraGraphGeodesicPath
finds the shortest edge path between the two points, and the polyline's length is summed.

GeodesicSurface builds the point -> cell links once, so dragging one point recomputes only the paths. The
functions taking device tensors leave the surface in HBM (the output of mesh.marching_cubes, the smoother or
surface_normals.compute_normals_device). The distances equal the sequential Dijkstra bit for bit; where two
neighbours at the same distance lead equally short (an ambiguous step, left to VTK's heap order) the path takes
the smaller point id and says so. The contract, restated and unverified against VTK, is in DESIGN.md §3.

vertices: float32 or float64 [V,3]; faces: int32 / int64 [T,3], or [T,4] with a leading 3; picks: float64-able
[P,3]. Inputs are never modified. A face id outside [0, V) raises ValueError.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np
import torch

from . import _lib
from .device import _dense, _face_form, _p, _stream, _workspace, require_cuda


@dataclass
class GeodesicPath:
    """The body of _draw_line without the tube and the actor. ids: one int64 tensor per segment, its points from
    the end pick's point back to the start pick's (one point when they coincide or the end is unreached); points:
    float32 [N, 3], the segments appended in order (vtkAppendPolyData); lengths: per segment; total: the
    measurement, summed step by step across the segments as measures.py sums it; ambiguous: per segment, whether
    a step of it was decided by the smaller id; unreached: per segment, whether the end is in another connected
    part of the surface. No segments when there are fewer than two picks or no cells."""
    ids: list = field(default_factory=list)
    points: torch.Tensor | np.ndarray | None = None
    lengths: list = field(default_factory=list)
    total: float = 0.0
    ambiguous: list = field(default_factory=list)
    unreached: list = field(default_factory=list)


def _verts(vertices, caller: str) -> int:
    if not isinstance(vertices, torch.Tensor):
        raise TypeError(f"{caller}: torch tensors expected")
    if vertices.dtype not in (torch.float32, torch.float64):
        raise TypeError("vertices: float32 or float64 expected")
    if vertices.dim() != 2 or vertices.shape[1] != 3:
        raise ValueError("vertices: [V,3] expected")
    _dense(vertices, "vertices")
    return int(vertices.dtype == torch.float64)


def _picks(picks, device) -> torch.Tensor:
    p = torch.as_tensor(picks, dtype=torch.float64).to(device).reshape(-1, 3).contiguous()
    return p


def closest_points_device(vertices: torch.Tensor, picks) -> torch.Tensor:
    """vtkPointLocator::FindClosestPoint for every pick: int64 [P] point ids on the device (ties to the smaller
    id). Does not synchronise."""
    f64 = _verts(vertices, "closest_points")
    nv = vertices.shape[0]
    if nv == 0:
        raise ValueError("closest_points: no points")
    p = _picks(picks, vertices.device)
    ids = torch.empty(p.shape[0], dtype=torch.int64, device=vertices.device)
    scratch = torch.empty(p.shape[0], dtype=torch.float64, device=vertices.device)
    with torch.cuda.device(vertices.device):
        _lib.call("b2v_closest_points", _p(vertices), nv, f64, _p(p), p.shape[0], _p(scratch), _p(ids), _stream())
    return ids


class GeodesicSurface:
    """A surface ready for geodesic measurements: the links are built once, here. Holds one workspace, so its
    calls run one at a time."""

    def __init__(self, vertices: torch.Tensor, faces: torch.Tensor):
        self.f64 = _verts(vertices, "GeodesicSurface")
        if not isinstance(faces, torch.Tensor):
            raise TypeError("GeodesicSurface: torch tensors expected")
        if faces.dtype not in (torch.int32, torch.int64):
            raise TypeError("faces: int32 or int64 expected")
        cols = _face_form(tuple(faces.shape))
        _dense(faces, "faces")
        if faces.device != vertices.device:
            raise ValueError("vertices and faces must be on the same device")
        self.vertices, self.nv, self.nt = vertices, vertices.shape[0], faces.shape[0]
        if self.nt > 0 and self.nv == 0:
            raise ValueError("GeodesicSurface: faces without vertices")
        self.rounds = self.buckets = 0
        self._ws = None
        if self.nt == 0:
            return
        lib = _lib.load()
        self._ws = _workspace(lib.b2v_geodesic_workspace_bytes(self.nv, self.nt), vertices.device)
        with torch.cuda.device(vertices.device):
            _lib.call("b2v_geodesic_links", _p(vertices), self.nv, self.f64, _p(faces), self.nt, cols,
                      int(faces.dtype == torch.int64), _p(self._ws), _stream())

    def closest_points(self, picks) -> torch.Tensor:
        return closest_points_device(self.vertices, picks)

    def _distances(self, start: int, end: int, out) -> None:
        if not 0 <= start < self.nv or not -1 <= end < self.nv:
            raise ValueError("geodesic: start / end outside [0, V)")
        stats = (C.c_int64 * 2)()
        with torch.cuda.device(self.vertices.device):
            _lib.call("b2v_geodesic_distances", _p(self.vertices), self.nv, self.f64, self.nt, _p(self._ws), start,
                      end, _p(out), _stream(), stats)
        self.rounds, self.buckets = stats[0], stats[1]

    def distances(self, start: int, end: int | None = None) -> torch.Tensor:
        """Float64 [V] edge-path distances from `start` (+inf where unreached), VTK's GetCumulativeWeights. With
        `end`, the computation stops early and only the points with d <= d[end] are final. Synchronises; the
        rounds and buckets it took are left in .rounds and .buckets."""
        if self.nt == 0:
            raise ValueError("geodesic: the surface has no cells")
        out = torch.empty(self.nv, dtype=torch.float64, device=self.vertices.device)
        self._distances(int(start), -1 if end is None else int(end), out)
        return out

    def path(self, picks) -> GeodesicPath:
        """_draw_line's measurement for the picks. Synchronises once per segment."""
        p = _picks(picks, self.vertices.device)
        r = GeodesicPath(points=torch.zeros((0, 3), dtype=torch.float32, device=self.vertices.device))
        if p.shape[0] < 2 or self.nt == 0:
            return r
        snap = self.closest_points(p).cpu().tolist()
        ids_buf = torch.empty(self.nv, dtype=torch.int64, device=self.vertices.device)
        pts_buf = torch.empty((self.nv, 3), dtype=torch.float32, device=self.vertices.device)
        counts, lengths = (C.c_int64 * 3)(), (C.c_double * 2)()
        pts = []
        for s, e in zip(snap[:-1], snap[1:]):
            self._distances(s, e, None)
            with torch.cuda.device(self.vertices.device):
                _lib.call("b2v_geodesic_trace", _p(self.vertices), self.nv, self.f64, self.nt, _p(self._ws), s, e,
                          r.total, _p(ids_buf), _p(pts_buf), _stream(), counts, lengths)
            n = counts[0]
            r.ids.append(ids_buf[:n].clone())
            pts.append(pts_buf[:n].clone())
            r.lengths.append(lengths[0])
            r.total = lengths[1]
            r.ambiguous.append(counts[1] > 0)
            r.unreached.append(bool(counts[2]))
        r.points = torch.cat(pts)
        return r


def geodesic_distances_device(vertices: torch.Tensor, faces: torch.Tensor, start: int,
                              end: int | None = None) -> torch.Tensor:
    """GeodesicSurface(vertices, faces).distances(start, end)."""
    return GeodesicSurface(vertices, faces).distances(start, end)


def geodesic_path_device(vertices: torch.Tensor, faces: torch.Tensor, picks) -> GeodesicPath:
    """GeodesicSurface(vertices, faces).path(picks)."""
    return GeodesicSurface(vertices, faces).path(picks)


def geodesic_path(vertices: np.ndarray, faces: np.ndarray, picks) -> GeodesicPath:
    """geodesic_path_device on numpy arrays: the ids, points and flags come back as numpy arrays."""
    if not isinstance(vertices, np.ndarray) or vertices.dtype not in (np.float32, np.float64):
        raise TypeError("vertices: a float32 or float64 numpy array expected")
    if not isinstance(faces, np.ndarray) or faces.dtype not in (np.int32, np.int64):
        raise TypeError("faces: an int32 or int64 numpy array expected")
    require_cuda()
    r = geodesic_path_device(torch.from_numpy(np.ascontiguousarray(vertices)).cuda(),
                             torch.from_numpy(np.ascontiguousarray(faces)).cuda(), picks)
    return GeodesicPath([i.cpu().numpy() for i in r.ids], r.points.cpu().numpy(), list(r.lengths), r.total,
                        list(r.ambiguous), list(r.unreached))
