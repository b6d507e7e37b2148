"""The surface panel's connectivity tools (polydata_utils.py:206-278, surface.py:319-411) on arrays, through
vtkPolyDataConnectivityFilter's semantics restated on the device (C ABI: b2v_conn_*):

  select_largest_part(vertices, faces, compact=False)            "Select largest surface"
  split_disconnected_parts(vertices, faces, compact=False)       "Split all disconnected surfaces"
  join_seeds_parts(vertices, faces, seeds, compact=False)        "Select regions of interest..."

numpy in, numpy out; the *_device variants take and return device tensors, and connectivity_device returns
the filter's state. Regions are numbered in the order of their lowest face; points are numbered in VTK's
wave order (PointMap). By default a result has VTK's form: EVERY point the traversal numbered (with
seeds: every point reached), in PointMap order, and the selected faces in ascending input order with
their corners through PointMap. The points of region r are the contiguous range
[point_offsets[r], point_offsets[r + 1]), so compact=True keeps only those and subtracts the offset.

Every result is (vertices float32 [N,3], faces, point_ids int32 [N], cell_ids int32 [C]): the input ids of
its points and faces, so that normals or other attributes follow with one gather. vertices: float32
[V,3]; faces: int32 / int64 [T,3], or [T,4] with a leading 3; the faces come back in the input's dtype
and form. An empty mesh, or seeds that reach nothing, gives an empty mesh; a seed id >= V raises
ValueError (VTK leaves it undefined). The output of mesh.marching_cubes can be passed straight to the
device entries, so the surface never leaves HBM.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from .device import _as_form, _mesh_arrays, _mesh_tensors, _p, _stream, _workspace, require_cuda


@dataclass
class Connectivity:
    """State of one run of the filter, on the device.

    region int32 [T] (-1: not visited); sizes int64 [R]; point_map int32 [V] (-1: not numbered);
    point_ids int32 [N] (the inverse of point_map); point_offsets / cell_offsets int64 [R + 1];
    vertices float32 [N,3] in point_map order; faces int32 [C,3] and cell_ids int32 [C]: the visited
    faces grouped by region, ascending input id inside each, corners through point_map. largest is the
    first region of the highest size (-1 if none); depth the most waves one region needed."""
    region: torch.Tensor
    sizes: torch.Tensor
    point_map: torch.Tensor
    point_ids: torch.Tensor
    point_offsets: torch.Tensor
    cell_offsets: torch.Tensor
    vertices: torch.Tensor
    faces: torch.Tensor
    cell_ids: torch.Tensor
    largest: int
    depth: int


def _seeds(seeds) -> np.ndarray:
    try:
        s = np.asarray(seeds, dtype=np.int64).reshape(-1)
    except (TypeError, ValueError):
        raise TypeError("seeds: a sequence of point ids expected") from None
    return np.ascontiguousarray(s)


def connectivity_device(vertices: torch.Tensor, faces: torch.Tensor, seeds=None) -> Connectivity:
    """Runs the filter: every region (seeds=None) or the region grown from the point ids `seeds`.
    Synchronises: the counts come back to the host."""
    cols = _mesh_tensors(vertices, faces, "connectivity")
    nv, nt, dev = vertices.shape[0], faces.shape[0], vertices.device
    s = None if seeds is None else _seeds(seeds)
    ns = 0 if s is None else len(s)
    lib = _lib.load()
    ws = _workspace(lib.b2v_conn_workspace_bytes(nv, nt, ns), dev)
    counts = (C.c_int64 * 5)()
    with torch.cuda.device(dev):
        _lib.call("b2v_conn_count", _p(vertices), nv, _p(faces), nt, cols, int(faces.dtype == torch.int64),
                  int(s is not None), C.c_void_p(None if not ns else s.ctypes.data), ns, _p(ws), _stream(), counts)
        nr, npts, ncells = counts[0], counts[1], counts[2]
        vout = torch.empty((npts, 3), dtype=torch.float32, device=dev)
        pids = torch.empty(npts, dtype=torch.int32, device=dev)
        fout = torch.empty((ncells, 3), dtype=torch.int32, device=dev)
        cids = torch.empty(ncells, dtype=torch.int32, device=dev)
        poff = torch.empty(nr + 1, dtype=torch.int64, device=dev)
        coff = torch.empty(nr + 1, dtype=torch.int64, device=dev)
        _lib.call("b2v_conn_emit", _p(vertices), nv, nt, ns, counts, _p(ws), _p(vout), _p(pids), _p(fout), _p(cids),
                  _p(poff), _p(coff), _stream())
        if nt:
            lay = (C.c_int64 * 6)()
            _lib.call("b2v_conn_layout", nv, nt, ns, lay)
            region = ws[lay[0]:lay[0] + 4 * nt].view(torch.int32).clone()
            pmap = ws[lay[1]:lay[1] + 4 * nv].view(torch.int32).clone()
        else:
            region = torch.empty(0, dtype=torch.int32, device=dev)
            pmap = torch.full((nv,), -1, dtype=torch.int32, device=dev)
    return Connectivity(region, coff[1:] - coff[:-1], pmap, pids, poff, coff, vout, fout, cids, counts[4], counts[3])


def _slice(c: Connectivity, r: int | None, poff, coff, compact: bool):
    """Region r of c (None: every visited face, the one region of a seeded run; -1: nothing) as views of its
    arrays, which may be tensors or numpy arrays: (vertices, faces int32, point_ids, cell_ids). The VTK form
    shares the whole point set between regions; poff / coff: the region offsets on the host."""
    if r is None:
        f0, f1, p0, p1 = 0, c.faces.shape[0], 0, c.vertices.shape[0]
    elif r < 0:
        f0 = f1 = p0 = p1 = 0
    else:
        f0, f1, p0, p1 = coff[r], coff[r + 1], poff[r], poff[r + 1]
    faces = c.faces[f0:f1]
    if compact or (r is not None and r < 0):
        v, pids, faces = c.vertices[p0:p1], c.point_ids[p0:p1], faces - p0
    else:
        v, pids = c.vertices, c.point_ids
    return v, faces, pids, c.cell_ids[f0:f1]


def _part(c, r, poff, coff, dtype, cols, compact):
    v, f, p, i = _slice(c, r, poff, coff, compact)
    return v, _as_form(f.contiguous(), dtype, cols), p, i


def _host_part(h, r, poff, coff, dtype, cols, compact):
    v, f, p, i = _slice(h, r, poff, coff, compact)
    f = f.astype(dtype, copy=False)
    if cols == 4:
        f = np.concatenate((np.full((len(f), 1), 3, dtype), f), 1)
    return v, f, p, i


def _largest_offsets(c: Connectivity):
    r = c.largest
    if r < 0:
        return -1, [], []
    return 0, c.point_offsets[r:r + 2].tolist(), c.cell_offsets[r:r + 2].tolist()


def select_largest_part_device(vertices: torch.Tensor, faces: torch.Tensor, compact: bool = False):
    """polydata_utils.SelectLargestPart on device tensors: (vertices, faces, point_ids, cell_ids), the ids
    int32."""
    cols = _mesh_tensors(vertices, faces, "connectivity")
    c = connectivity_device(vertices, faces)
    return _part(c, *_largest_offsets(c), faces.dtype, cols, compact)


def split_disconnected_parts_device(vertices: torch.Tensor, faces: torch.Tensor, compact: bool = False):
    """polydata_utils.SplitDisconectedParts on device tensors: one (vertices, faces, point_ids, cell_ids) per
    region, in region order; one traversal serves them all. In the VTK form every part's vertices and
    point_ids are the same tensors."""
    cols = _mesh_tensors(vertices, faces, "connectivity")
    c = connectivity_device(vertices, faces)
    poff, coff = c.point_offsets.tolist(), c.cell_offsets.tolist()
    return [_part(c, r, poff, coff, faces.dtype, cols, compact) for r in range(len(coff) - 1)]


def join_seeds_parts_device(vertices: torch.Tensor, faces: torch.Tensor, seeds, compact: bool = False):
    """polydata_utils.JoinSeedsParts on device tensors: (vertices, faces, point_ids, cell_ids) of the faces
    reached from the point ids `seeds`."""
    cols = _mesh_tensors(vertices, faces, "connectivity")
    c = connectivity_device(vertices, faces, seeds)
    return _part(c, None, None, None, faces.dtype, cols, compact)


def _on_host(vertices, faces, seeds=None):
    """connectivity_device on numpy arrays, its result copied to the host once."""
    cols = _mesh_arrays(vertices, faces)
    require_cuda()
    c = connectivity_device(torch.from_numpy(np.ascontiguousarray(vertices)).cuda(),
                            torch.from_numpy(np.ascontiguousarray(faces)).cuda(), seeds)
    h = Connectivity(**{k: (x.cpu().numpy() if isinstance(x, torch.Tensor) else x) for k, x in vars(c).items()})
    return h, cols


def select_largest_part(vertices, faces, compact: bool = False):
    """SelectLargestPart(polydata) on arrays: (vertices float32 [N,3], faces, point_ids, cell_ids)."""
    h, cols = _on_host(vertices, faces)
    return _host_part(h, *_largest_offsets(h), faces.dtype, cols, compact)


def split_disconnected_parts(vertices, faces, compact: bool = False):
    """SplitDisconectedParts(polydata) on arrays: a list of (vertices, faces, point_ids, cell_ids). In the VTK
    form every part's vertices and point_ids are the same (read-only) arrays."""
    h, cols = _on_host(vertices, faces)
    h.vertices.flags.writeable = h.point_ids.flags.writeable = compact
    poff, coff = h.point_offsets.tolist(), h.cell_offsets.tolist()
    return [_host_part(h, r, poff, coff, faces.dtype, cols, compact) for r in range(len(coff) - 1)]


def join_seeds_parts(vertices, faces, seeds, compact: bool = False):
    """JoinSeedsParts(polydata, point_id_list) on arrays: (vertices, faces, point_ids, cell_ids)."""
    h, cols = _on_host(vertices, faces, seeds)
    return _host_part(h, None, None, None, faces.dtype, cols, compact)
