"""Jump flooding and the porous-scaffold "Voronoi" generator on the device.

  jump_flooding(distance_map, map_owners, sites, normalize)   invesalius_rs.jump_flooding
      (floodfill_py.rs:262-276 -> floodfill.rs:298-507), numpy in place; imported by
      plugins/porous_creation/schwarzp.py:5
  create_voronoi(sx, sy, sz, number_sites, normalize, border)   schwarzp.py:37-52
  create_voronoi_non_random(sx, sy, sz, nsx, nsy, nsz, normalize, noise, border)   schwarzp.py:55-84
  image_normalize(image, min_, max_, output_dtype)   imagedata_utils.py:580-587, float32 -> int16
      (plugins/porous_creation/gui.py:28, 237)

Under them, jump_flooding_device and voronoi_borders_device work on device tensors. Every result equals
the reference's bit for bit: jump flooding restates the crate's float32 arithmetic and visiting order,
the scaffold borders are np.gradient's non-zero test on the integer owners, the float32 gaussian_filter
is filters._gaussian, and image_normalize is NumPy's float32 evaluation of its formula.

The generators draw their sites on the host with the plugin's NumPy calls in the plugin's order, so
the global RNG is consumed identically and one np.random.seed gives one scaffold.
"""
from __future__ import annotations

import operator

import numpy as np
import torch

from . import _lib
from . import device as dev
from . import filters
from .device import _dense, _p, _stream

GAUSSIAN_SIGMA = 1.5   # schwarzp.py:8
_GRADIENT_MSG = ("Shape of array too small to calculate a numerical gradient, at least (edge_order + 1) elements "
                 "are required.")   # NumPy's message


def _require(a, dtype, ndim: int, name: str) -> None:
    """The array checks of PyO3's extraction: a numpy array of exactly this dtype and rank, else TypeError."""
    if not isinstance(a, np.ndarray) or a.dtype != dtype or a.ndim != ndim:
        raise TypeError(f"{name}: {np.dtype(dtype)} {ndim}-D numpy array expected")


def jump_flooding_device(dist: torch.Tensor, owners: torch.Tensor, sites_t: torch.Tensor, normalize: bool) -> None:
    """invesalius_rs.jump_flooding on dense device tensors, in place: dist float32 and owners int32 of one
    3-D shape, sites_t int32 [n][>= 3] (z, y, x) rows on the same device."""
    _dense(dist, "distance_map"); _dense(owners, "map_owners"); _dense(sites_t, "sites")
    if dist.dtype != torch.float32 or dist.dim() != 3:
        raise TypeError("distance_map: float32 3-D tensor expected")
    if owners.dtype != torch.int32 or owners.dim() != 3:
        raise TypeError("map_owners: int32 3-D tensor expected")
    if sites_t.dtype != torch.int32 or sites_t.dim() != 2:
        raise TypeError("sites: int32 2-D tensor expected")
    n = sites_t.shape[0]
    if n == 0 or dist.numel() == 0:
        return
    if owners.shape != dist.shape:
        raise ValueError(f"jump_flooding: map_owners {tuple(owners.shape)} and distance_map {tuple(dist.shape)} differ")
    if sites_t.shape[1] < 3:
        raise ValueError("jump_flooding: sites need (z, y, x) columns")
    if owners.device != dist.device or sites_t.device != dist.device:
        raise ValueError("jump_flooding: tensors on different devices")
    s = sites_t[:, :3].contiguous()
    ws = dev._workspace(_lib.load().b2v_jump_flooding_workspace_bytes(*dist.shape, n), dist.device)
    with torch.cuda.device(dist.device):
        _lib.call("b2v_jump_flooding", _p(dist), _p(owners), *dist.shape, _p(s), n, int(bool(normalize)), _p(ws),
                  _stream())


def jump_flooding(distance_map, map_owners, sites, normalize) -> None:
    """invesalius_rs.jump_flooding(distance_map, map_owners, sites, normalize): writes both volumes in
    place (strided views included). Where the crate panics (volumes of different shapes, sites with fewer
    than 3 columns) this raises ValueError; with no sites or an empty volume it returns untouched."""
    _require(distance_map, np.float32, 3, "distance_map")
    _require(map_owners, np.int32, 3, "map_owners")
    _require(sites, np.int32, 2, "sites")
    if not isinstance(normalize, (bool, np.bool_)):
        raise TypeError("normalize: bool expected")
    if sites.shape[0] == 0 or distance_map.size == 0:
        return
    if map_owners.shape != distance_map.shape:
        raise ValueError(f"jump_flooding: map_owners {map_owners.shape} and distance_map {distance_map.shape} differ")
    if sites.shape[1] < 3:
        raise ValueError("jump_flooding: sites need (z, y, x) columns")
    if not distance_map.flags.writeable or not map_owners.flags.writeable:
        raise ValueError("output array is read-only")
    d = dev.to_device(distance_map)
    o = dev.to_device(map_owners, d.device)
    s = torch.from_numpy(np.ascontiguousarray(sites[:, :3])).to(d.device)
    jump_flooding_device(d, o, s, bool(normalize))
    dev.to_host(d, distance_map)
    dev.to_host(o, map_owners)


def voronoi_borders_device(owners: torch.Tensor) -> torch.Tensor:
    """float32 (owners' np.gradient magnitude > 0) of a dense int32 [sz][sy][sx] tensor: over y and x when
    sz == 1 (schwarzp.py:43-45), over all three axes otherwise (:47-48). Raises NumPy's ValueError where
    np.gradient would (a differentiated axis shorter than 2)."""
    _dense(owners, "map_owners")
    if owners.dtype != torch.int32 or owners.dim() != 3:
        raise TypeError("map_owners: int32 3-D tensor expected")
    planar = owners.shape[0] == 1
    if any(n < 2 for n in (owners.shape[1:] if planar else owners.shape)):
        raise ValueError(_GRADIENT_MSG)
    out = torch.empty(owners.shape, dtype=torch.float32, device=owners.device)
    with torch.cuda.device(owners.device):
        _lib.call("b2v_voronoi_borders", _p(owners), *owners.shape, int(planar), _p(out), _stream())
    return out


def _volume_shape(sx, sy, sz) -> tuple[int, int, int]:
    """(sz, sy, sx) with np.zeros' argument errors, raised before the sites are drawn as in the plugin."""
    shape = tuple(operator.index(n) for n in (sz, sy, sx))
    if any(n < 0 for n in shape):
        raise ValueError("negative dimensions are not allowed")
    return shape


def _scaffold(shape, sites: np.ndarray, normalize, border) -> np.ndarray:
    """The device tail of both generators: jump flooding from zeroed volumes, then the distances, or the
    owner borders blurred by the float32 gaussian_filter(sigma = 1.5)."""
    if border and any(n < 2 for n in (shape[1:] if shape[0] == 1 else shape)):
        raise ValueError(_GRADIENT_MSG)
    dev.require_cuda()
    dist = torch.zeros(shape, dtype=torch.float32, device="cuda")
    owners = torch.zeros(shape, dtype=torch.int32, device="cuda")
    jump_flooding_device(dist, owners, torch.from_numpy(np.ascontiguousarray(sites)).to(dist.device), normalize)
    out = filters._gaussian(voronoi_borders_device(owners), GAUSSIAN_SIGMA, torch.float32) if border else dist
    res = np.empty(shape, np.float32)
    dev.to_host(out, res)
    return res


def create_voronoi(sx=256, sy=256, sz=256, number_sites=1000, normalize=False, border=True) -> np.ndarray:
    """schwarzp.create_voronoi: number_sites uniformly random sites; float32 (sz, sy, sx)."""
    shape = _volume_shape(sx, sy, sz)
    sites = np.random.randint((0, 0, 0), (sz, sy, sx), (number_sites, 3), dtype=np.int32)
    return _scaffold(shape, sites, normalize, border)


def create_voronoi_non_random(sx=256, sy=256, sz=256, nsx=25, nsy=25, nsz=25, normalize=False, noise=False,
                              border=True) -> np.ndarray:
    """schwarzp.create_voronoi_non_random: one site per cell of an nsz x nsy x nsx lattice, at the cell
    centre (optionally moved by uniform noise in [-0.25, 0.25) cells), truncated to int32."""
    shape = _volume_shape(sx, sy, sz)
    zz, yy, xx = np.meshgrid(np.arange(nsz), np.arange(nsy), np.arange(nsx))   # default 'xy': site order matters
    sites = np.stack((zz.flatten() + 0.5, yy.flatten() + 0.5, xx.flatten() + 0.5), axis=1)
    if noise:
        sites += np.random.random(sites.shape) * 0.5 - 0.25
    sites[:, 0] *= sz / nsz
    sites[:, 1] *= sy / nsy
    sites[:, 2] *= sx / nsx
    return _scaffold(shape, np.array(sites, dtype=np.int32), normalize, border)


def image_normalize(image, min_=0.0, max_=1.0, output_dtype=np.int16) -> np.ndarray:
    """imagedata_utils.image_normalize for a float32 image, Python int or float bounds and an int16
    output: (image - min) * ((max_ - min_) / (max - min)) + min_ evaluated in float32, as NumPy promotes
    Python scalars against float32, and stored with the C cast; min_ everywhere when the image is
    constant. Anything else raises NotImplementedError."""
    a = np.asarray(image)
    if a.dtype != np.float32 or np.dtype(output_dtype) != np.int16:
        raise NotImplementedError(f"image_normalize: float32 -> int16 only ({a.dtype} -> {np.dtype(output_dtype)})")
    for b in (min_, max_):
        if isinstance(b, np.generic) or not isinstance(b, (int, float)):
            raise NotImplementedError("image_normalize: Python int or float bounds only (NumPy scalars promote "
                                      "differently)")
    out = np.empty(a.shape, np.int16)
    if a.size == 0:
        a.min()   # NumPy's ValueError for a zero-size reduction
    t = dev.to_device(a)
    lo, hi = (float(v) for v in torch.aminmax(t))
    fill = np.zeros((), np.int16)
    if lo == hi:
        fill[...] = min_   # NumPy's conversion of min_, errors included
    o = torch.empty(t.shape, dtype=torch.int16, device=t.device)
    with torch.cuda.device(t.device):
        _lib.call("b2v_image_normalize_f32_i16", _p(t), t.numel(), lo, hi, float(np.float32(max_ - min_)),
                  float(np.float32(min_)), int(fill), _p(o), _stream())
    dev.to_host(o, out)
    return out
