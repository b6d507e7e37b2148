"""Context-aware mesh smoothing with the reference's interface (SURVEY 8f-2):

  Mesh(vertices=, faces=, normals=) / Mesh(other=)     invesalius_rs/__init__.py:114-249 (array form)
  ca_smoothing(mesh, T, tmax, bmin, n_iters)           invesalius_rs/__init__.py:251-270
  context_aware_smoothing(vertices, faces, normals, T, tmax, bmin, n_iters)   the native entry (mesh_py.rs)

vertices float32 [V,3] are smoothed IN PLACE like the Rust function does; faces [M,4] (leading 3) of
any of the reference's integer types; normals float32 / float64 [M,3] per face.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from . import device as dev
from .device import _p, _stream, _workspace


def _n_iters(n_iters) -> int:
    """The reference's `n_iters: u32`: PyO3 raises OverflowError outside [0, 2**32)."""
    n = int(n_iters)
    if n < 0:
        raise OverflowError("can't convert negative int to unsigned")
    if n > 0xFFFFFFFF:
        raise OverflowError("out of range integral type conversion attempted")
    return n


def smooth_device(verts: torch.Tensor, faces4: torch.Tensor, normals: torch.Tensor, T, tmax, bmin, n_iters) -> None:
    """float32 [V,3] / int64 [M,4] / float32 [M,3] device tensors; verts is modified in place."""
    n_iters = _n_iters(n_iters)
    if verts.dtype != torch.float32 or faces4.dtype != torch.int64 or normals.dtype != torch.float32:
        raise TypeError("ca_smoothing: float32 vertices, int64 faces, float32 normals")
    if faces4.dim() != 2 or faces4.shape[1] != 4 or normals.shape != (faces4.shape[0], 3) or verts.dim() != 2 or verts.shape[1] != 3:
        raise TypeError("ca_smoothing: vertices [V,3], faces [M,4], normals [M,3]")
    for t_ in (verts, faces4, normals):
        dev._dense(t_, "mesh array")
    nv, nf = verts.shape[0], faces4.shape[0]
    if nv == 0 or nf == 0:
        return
    # the stable order of the face entries by vertex id (plumbing: any stable sort does)
    order = torch.sort(faces4.reshape(-1), stable=True).indices.contiguous()
    ws = _workspace(_lib.load().b2v_ca_smoothing_workspace_bytes(nv, nf), verts.device)
    with torch.cuda.device(verts.device):
        _lib.call("b2v_ca_smoothing", _p(verts), nv, _p(faces4), nf, _p(normals), _p(order), float(T), float(tmax), float(bmin),
                  n_iters, _p(ws), _stream())


def context_aware_smoothing(vertices, faces, normals, T, tmax, bmin, n_iters) -> None:
    if not isinstance(vertices, np.ndarray) or vertices.dtype != np.float32:
        raise TypeError("ca_smoothing: vertices must be a float32 array (the float64 variant is not built)")
    if not isinstance(faces, np.ndarray) or faces.dtype not in (np.int64, np.int32, np.uint64, np.uint32):
        raise TypeError("Invalid face type")
    if not isinstance(normals, np.ndarray) or normals.dtype not in (np.float32, np.float64):
        raise TypeError("Invalid normals type")
    if not vertices.flags.writeable:
        raise ValueError("vertices is read-only")
    n_iters = _n_iters(n_iters)
    v = torch.from_numpy(np.ascontiguousarray(vertices)).cuda()
    f = torch.from_numpy(np.ascontiguousarray(faces).astype(np.int64)).cuda()
    n = torch.from_numpy(np.ascontiguousarray(normals, dtype=np.float32)).cuda()   # as_(): float64 normals enter the float64 test exactly
    if normals.dtype == np.float64 and not np.array_equal(normals.astype(np.float32).astype(np.float64), normals):
        raise NotImplementedError("ca_smoothing: float64 normals that are not float32-representable are not built")
    smooth_device(v, f, n, T, tmax, bmin, n_iters)
    vertices[...] = v.cpu().numpy()


class Mesh:
    """Array form of invesalius_rs.Mesh (no VTK on this side: build it from arrays or from another Mesh)."""

    def __init__(self, pd=None, other=None, vertices=None, faces=None, normals=None):
        if pd is not None:
            raise NotImplementedError("Mesh(pd=vtkPolyData) needs VTK; pass vertices / faces / normals")
        if other is not None:
            if not isinstance(other, Mesh):
                raise TypeError("other must be a Mesh instance")
            self._vertices = np.ascontiguousarray(other.vertices.copy())
            self._faces = np.ascontiguousarray(other.faces.copy())
            self._normals = np.ascontiguousarray(other.normals.copy())
        elif vertices is not None and faces is not None and normals is not None:
            self._vertices = np.ascontiguousarray(vertices)
            self._faces = np.ascontiguousarray(faces)
            self._normals = np.ascontiguousarray(normals)
        else:
            raise ValueError("Must provide either pd, other, or (vertices, faces, normals)")

    vertices = property(lambda self: self._vertices)
    faces = property(lambda self: self._faces)
    normals = property(lambda self: self._normals)

    def ca_smoothing(self, T, tmax, bmin, n_iters):
        context_aware_smoothing(self._vertices, self._faces, self._normals, T, tmax, bmin, n_iters)


def ca_smoothing(mesh, T, tmax, bmin, n_iters):
    mesh.ca_smoothing(T, tmax, bmin, n_iters)
