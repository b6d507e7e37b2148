"""CPU checker for the porous-scaffold Voronoi generator — TEST INFRASTRUCTURE ONLY.

jump_flooding: ctypes wrapper of oracle/voronoi.c (built into oracle/libvoronoi.so by oracle/voronoi.mk) with
the crate's name and argument order (invesalius_rs.jump_flooding, in place). create_voronoi,
create_voronoi_non_random and image_normalize restate plugins/porous_creation/schwarzp.py:37-84 and
imagedata_utils.py:580-587 in NumPy / SciPy: the checker's jump_flooding, then np.gradient,
scipy.ndimage.gaussian_filter and the image_normalize formula themselves. The random sites are drawn with
the same NumPy calls in the same order, so one np.random.seed gives one scaffold.
PARITY UNPINNED against the crate: see voronoi.c's header and DESIGN.md §5.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np
from scipy import ndimage as ndi

_HERE = Path(__file__).resolve().parent
_LIB = None
GAUSSIAN_SIGMA = 1.5


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        so, src = _HERE / "libvoronoi.so", _HERE / "voronoi.c"
        if not so.exists() or so.stat().st_mtime < src.stat().st_mtime:
            subprocess.run(["make", "-C", str(_HERE), "-f", "voronoi.mk"], check=True, capture_output=True)
        _LIB = C.CDLL(str(so))
    return _LIB


def jump_flooding(distance_map, map_owners, sites, normalize, nthreads=None):
    """floodfill_py.rs:262-276 -> floodfill.rs:298-507, in place (any strides: dense copies are written back)."""
    if distance_map.dtype != np.float32 or distance_map.ndim != 3:
        raise TypeError("distance_map: float32 3-D array expected")
    if map_owners.dtype != np.int32 or map_owners.ndim != 3:
        raise TypeError("map_owners: int32 3-D array expected")
    if sites.dtype != np.int32 or sites.ndim != 2:
        raise TypeError("sites: int32 2-D array expected")
    if sites.shape[0] == 0 or distance_map.size == 0:
        return
    if map_owners.shape != distance_map.shape or sites.shape[1] < 3:
        raise ValueError("jump_flooding: the crate panics on these shapes")
    d = np.ascontiguousarray(distance_map)
    o = np.ascontiguousarray(map_owners)
    s = np.ascontiguousarray(sites[:, :3])
    nthreads = nthreads or os.cpu_count() or 1
    lib().orc_jump_flooding(C.c_void_p(d.ctypes.data), C.c_void_p(o.ctypes.data), *map(C.c_int64, d.shape),
                            C.c_void_p(s.ctypes.data), C.c_int64(len(s)), C.c_int(int(bool(normalize))),
                            C.c_int(int(nthreads)))
    distance_map[...] = d
    map_owners[...] = o


def _scaffold(shape, sites, normalize, border):
    """The common tail of both generators: jump flooding from zeroed volumes, then either the distances
    or the blurred owner borders."""
    distances = np.zeros(shape, np.float32)
    owners = np.zeros(shape, np.int32)
    jump_flooding(distances, owners, sites, normalize)
    if not border:
        return distances
    if shape[0] == 1:
        grads = np.gradient(owners[0])
    else:
        grads = np.gradient(owners)
    mag = np.sqrt(sum(g * g for g in grads)).reshape(shape)
    return ndi.gaussian_filter((mag > 0).astype(np.float32), GAUSSIAN_SIGMA)


def create_voronoi(sx=256, sy=256, sz=256, number_sites=1000, normalize=False, border=True):
    """schwarzp.py:37-52."""
    sites = np.random.randint((0, 0, 0), (sz, sy, sx), (number_sites, 3), dtype=np.int32)
    return _scaffold((sz, sy, sx), sites, normalize, border)


def non_random_sites(sx, sy, sz, nsx, nsy, nsz, noise):
    """The jittered lattice of schwarzp.py:57-72: cell centres of an nsz x nsy x nsx grid (in meshgrid's
    default 'xy' order), optionally moved by uniform noise in [-0.25, 0.25), scaled to the volume and
    truncated to int32."""
    zz, yy, xx = np.meshgrid(np.arange(nsz), np.arange(nsy), np.arange(nsx))
    sites = np.stack((zz.flatten() + 0.5, yy.flatten() + 0.5, xx.flatten() + 0.5), axis=1)
    if noise:
        sites += np.random.random(sites.shape) * 0.5 - 0.25
    sites[:, 0] *= sz / nsz
    sites[:, 1] *= sy / nsy
    sites[:, 2] *= sx / nsx
    return np.array(sites, dtype=np.int32)


def create_voronoi_non_random(sx=256, sy=256, sz=256, nsx=25, nsy=25, nsz=25, normalize=False, noise=False,
                              border=True):
    """schwarzp.py:55-84."""
    return _scaffold((sz, sy, sx), non_random_sites(sx, sy, sz, nsx, nsy, nsz, noise), normalize, border)


def image_normalize(image, min_=0.0, max_=1.0, output_dtype=np.int16):
    """imagedata_utils.py:580-587."""
    out = np.empty(image.shape, output_dtype)
    lo, hi = image.min(), image.max()
    if lo == hi:
        out[:] = min_
    else:
        out[:] = (image - lo) * ((max_ - min_) / (hi - lo)) + min_
    return out
