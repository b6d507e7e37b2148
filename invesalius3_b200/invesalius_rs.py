"""Mirror of the reference's native package `invesalius_rs` (numpy in, numpy out).

Same names, argument order, in-place output convention and error behaviour as
`invesalius_rs/__init__.py:11-111` + the PyO3 layer (`src/*_py.rs`), so the callers in
`invesalius/data/{slice_,styles,mask}.py` can bind this module under the aliases they
already use (`import invesalius_rs as floodfill / mips`), see INTEGRATION.md.

Every function packs its (possibly strided, memmap-backed) arguments into dense device
tensors, runs the sm_90a kernels of libb2v.so and writes results back into the
caller's arrays. There is no CPU fallback.

Error mapping (reference -> here):
  PyO3 extraction TypeError / OverflowError  -> same exception types
  "Invalid image or output type" TypeError   -> same
  Rust panic (out-of-bounds seed, unrepresentable MIDA result, label > nlabels)
      pyo3_runtime.PanicException             -> ValueError (IndexError for seeds)
"""
from __future__ import annotations

import numpy as np

from . import device as dev
from ._lib import B2VError  # noqa: F401

_SUFFIX = {np.dtype(np.int16): "i16", np.dtype(np.uint8): "u8", np.dtype(np.float64): "f64"}
_RANGE = {"i16": (-32768, 32767), "u8": (0, 255)}


def _suffix(a, what="image"):
    if not isinstance(a, np.ndarray):
        raise TypeError(f"{what} must be a numpy array")
    try:
        return _SUFFIX[a.dtype]
    except KeyError:
        raise TypeError(f"Invalid {what} type: {a.dtype}") from None


def _extract(v, suf):
    """PyO3 `extract::<T>()`: integers must fit T; a float is only accepted for f64."""
    if suf == "f64":
        return float(v)
    if isinstance(v, (float, np.floating)):
        raise TypeError("'float' object cannot be interpreted as an integer")
    v = int(v)
    lo, hi = _RANGE[suf]
    if not lo <= v <= hi:
        raise OverflowError("out of range integral type conversion attempted")
    return v


def _need3(a, name):
    if a.ndim != 3:
        raise TypeError(f"{name} must be 3-dimensional")


def _seed_check(exc):
    if "outside the volume" in str(exc):
        raise IndexError(str(exc)) from None
    raise exc


# ------------------------------------------------------------------------------- flood fill
def floodfill_threshold(data, seeds, t0, t1, fill, strct, out):
    """invesalius_rs/__init__.py:21-40."""
    suf = _suffix(data, "data")
    _need3(data, "data")
    if not isinstance(out, np.ndarray) or out.dtype != np.uint8 or out.ndim != 3:
        raise TypeError("Invalid output type")
    if out.shape != data.shape:
        raise ValueError("data and out shapes differ")
    tuple_seeds = [tuple(s) for s in seeds]
    strct_u8 = np.ascontiguousarray(strct, dtype=np.uint8)
    if suf == "i16":
        t0, t1, fill = int(t0), int(t1), int(fill)
    elif suf == "f64":
        t0, t1, fill = float(t0), float(t1), float(fill)
    t0, t1 = _extract(t0, suf), _extract(t1, suf)
    fill = _extract(fill, "u8")
    if not out.flags.writeable:
        raise ValueError("out is read-only")
    aliased = np.shares_memory(data, out)
    d = dev.to_device(data)
    o = d if (aliased and suf == "u8") else dev.to_device(out)
    try:
        if aliased and suf == "u8":
            # data is out (styles.py:2932-2940): degenerates to the in-place walk
            dev.floodfill_threshold_inplace(d, tuple_seeds, t0, t1, fill, strct_u8)
        else:
            dev.floodfill_threshold(d, tuple_seeds, t0, t1, fill, strct_u8, o)
    except ValueError as e:
        _seed_check(e)
    dev.to_host(o, out)


def floodfill_threshold_inplace(data, seeds, t0, t1, fill, strct):
    """invesalius_rs/__init__.py:43-54."""
    suf = _suffix(data, "data")
    _need3(data, "data")
    tuple_seeds = [tuple(s) for s in seeds]
    strct_u8 = np.ascontiguousarray(strct, dtype=np.uint8)
    t0, t1, fill = _extract(t0, suf), _extract(t1, suf), _extract(fill, suf)
    if not data.flags.writeable:
        raise ValueError("data is read-only")
    d = dev.to_device(data)
    try:
        dev.floodfill_threshold_inplace(d, tuple_seeds, t0, t1, fill, strct_u8)
    except ValueError as e:
        _seed_check(e)
    dev.to_host(d, data)


def floodfill(data, i, j, k, v, fill, out):
    """floodfill_py.rs:87-135 (exported as-is by __init__.py:11)."""
    suf = _suffix(data, "data")
    _need3(data, "data")
    if not isinstance(out, np.ndarray) or out.dtype != np.uint8 or out.shape != data.shape:
        raise TypeError("Invalid output type")
    v, fill = _extract(v, suf), _extract(fill, "u8")
    for c in (i, j, k):
        if int(c) < 0:
            raise OverflowError("can't convert negative int to unsigned")
    d, o = dev.to_device(data), dev.to_device(out)
    try:
        dev.floodfill(d, int(i), int(j), int(k), v, fill, o)
    except ValueError as e:
        _seed_check(e)
    dev.to_host(o, out)


def fill_holes_automatically(mask, labels, nlabels, max_size) -> bool:
    """floodfill_py.rs:233-249; caller invesalius/data/mask.py:519-562."""
    if not isinstance(mask, np.ndarray) or mask.dtype != np.uint8:
        raise TypeError("Invalid mask type")
    if not isinstance(labels, np.ndarray) or labels.dtype != np.uint32:
        raise TypeError("labels must be a uint32 array")
    _need3(mask, "mask")
    if labels.shape != mask.shape:
        raise ValueError("mask and labels shapes differ")
    nlabels, max_size = int(nlabels), int(max_size)
    if not (0 <= nlabels < 2 ** 32 and 0 <= max_size < 2 ** 32):
        raise OverflowError("out of range integral type conversion attempted")
    m = dev.to_device(mask)
    lab = dev.to_device(labels)
    modified = dev.fill_holes_automatically(m, lab, nlabels, max_size)
    if modified:
        dev.to_host(m, mask)
    return modified


# ------------------------------------------------------------------------------- projections
def _need_2d_out(out, shape3, axis):
    want = [(shape3[1], shape3[2]), (shape3[0], shape3[2]), (shape3[0], shape3[1])][axis]
    if out.ndim != 2 or tuple(out.shape) != want:
        raise ValueError(f"out must have shape {want}")
    if not out.flags.writeable:
        raise ValueError("out is read-only")


def _axis(axis):
    axis = int(axis)
    if axis < 0:
        raise OverflowError("can't convert negative int to unsigned")
    return axis


def mida(image, axis, wl, ww, out):
    """invesalius_rs/__init__.py:91-95 (wl, ww pass through int(); mips_py.rs:161-202)."""
    from . import projection
    axis = _axis(axis)
    if not isinstance(image, np.ndarray) or not isinstance(out, np.ndarray):
        raise TypeError("Invalid image or output type")
    pair = (image.dtype, out.dtype)
    if pair not in ((np.int16, np.int16), (np.uint8, np.uint8), (np.float64, np.uint8)):
        raise TypeError("Invalid image or output type")
    _need3(image, "image")
    suf = _SUFFIX[image.dtype]
    wl, ww = _extract(int(wl), suf), _extract(int(ww), suf)
    if axis > 2:
        return  # mips.rs:128-132 treats any other axis like 2 only inside the match default
    _need_2d_out(out, image.shape, axis)
    res = projection.mida(dev.to_device(image), axis, wl, ww)
    dev.to_host(res[None], out[None])


def lmip(image, axis, tmin, tmax, out):
    """mips.rs:7-86; the call sites are slice_.py:892, 980, 1063 (`mips.lmip`)."""
    from . import projection
    axis = _axis(axis)
    suf = _suffix(image)
    if not isinstance(out, np.ndarray) or out.dtype != image.dtype:
        raise TypeError("Invalid image or output type")
    _need3(image, "image")
    tmin, tmax = _extract(tmin, suf), _extract(tmax, suf)
    if axis > 2:
        return  # mips.rs:84 `_ => ()`
    _need_2d_out(out, image.shape, axis)
    res = projection.lmip(dev.to_device(image), axis, tmin, tmax)
    dev.to_host(res[None], out[None])


def fast_countour_mip(image, n, axis, wl, ww, tmip, out):
    """invesalius_rs/__init__.py:98-101 -> mips_py.rs:204-253."""
    from . import projection
    axis, tmip = _axis(axis), _axis(tmip)
    if not isinstance(image, np.ndarray) or not isinstance(out, np.ndarray) or image.dtype != out.dtype \
            or image.dtype not in _SUFFIX:
        raise TypeError("Invalid image or output type")
    _need3(image, "image")
    suf = _SUFFIX[image.dtype]
    wl, ww = _extract(int(wl), suf), _extract(int(ww), suf)
    if axis > 2 or tmip > 2:
        raise ValueError("fast_countour_mip: axis and tmip must be 0, 1 or 2")
    _need_2d_out(out, image.shape, axis)
    if suf == "f64" and tmip == 2:
        raise NotImplementedError("fast_countour_mip: float64 contour-MIDA (float64 output) is not built on the device")
    res = projection.fast_countour_mip(dev.to_device(image), float(n), axis, wl, ww, tmip)
    dev.to_host(res[None], out[None])


def count_regions(image, number_regions):
    """invesalius_rs/__init__.py:108-111 -> count_regions.rs:5-18."""
    from . import labeling
    return labeling.count_regions(image, number_regions)


def _mesh_ops():
    from . import mesh_ops
    return mesh_ops


def ca_smoothing(mesh, T, tmax, bmin, n_iters):
    """invesalius_rs/__init__.py:251-270 (Mesh.ca_smoothing -> mesh.rs:27-395)."""
    mesh.ca_smoothing(T, tmax, bmin, n_iters)


def convolve_non_zero(volume, kernel, cval):
    """invesalius_rs/__init__.py -> transforms_py.rs:52-93 (Slice.calc_mask_area, slice_.py:2319)."""
    from . import filters
    return filters.convolve_non_zero(volume, kernel, cval)


ORIENTATIONS = {"AXIAL": 0, "CORONAL": 1, "SAGITAL": 2}


def apply_view_matrix_transform(volume, spacing, m, n, orientation, minterpol, cval, out):
    """invesalius_rs/__init__.py:84 -> transforms_py.rs:96-148: resample `volume` through the 4x4
    view matrix into the slab `out` (callers: slice_.py:865, 949, 1036, 1980, 2038). The volume is
    shipped to the device whole (the rotation gathers from anywhere in it); `out` is written in place."""
    import ctypes as C
    from . import _lib
    if not isinstance(volume, np.ndarray) or not isinstance(out, np.ndarray) or volume.dtype != out.dtype \
            or volume.dtype not in _SUFFIX:
        raise TypeError("Invalid volume or output type")
    _need3(volume, "volume")
    _need3(out, "out")
    suf = _SUFFIX[volume.dtype]
    cval = _extract(cval if suf == "f64" else int(cval), suf)
    n = int(n)
    if n < 0:
        raise OverflowError("can't convert negative int to unsigned")
    sp = np.ascontiguousarray([float(v) for v in spacing], dtype=np.float64)
    mm = np.ascontiguousarray(m, dtype=np.float64)
    if sp.shape != (3,) or mm.shape != (4, 4):
        raise TypeError("spacing must have 3 entries and m must be 4x4")
    if not out.flags.writeable:
        raise ValueError("out is read-only")
    d = dev.to_device(volume)
    import torch
    o = torch.empty(out.shape, dtype=d.dtype, device=d.device)
    ws = dev._workspace(256, d.device)
    with torch.cuda.device(d.device):
        _lib.call("b2v_apply_view_matrix_transform", dev._p(d), dev.dtype_code(d), *volume.shape,
                  C.c_void_p(sp.ctypes.data), C.c_void_p(mm.ctypes.data), n, ORIENTATIONS.get(orientation, 3), int(minterpol),
                  float(cval), dev._p(o), *out.shape, dev._p(ws), dev._stream())
    dev.to_host(o, out)


# ---- the rest of the crate's surface (invesalius_rs/__init__.py:273-300) ---------------------------
# The functions above replace the hot path. Everything else the reference imports from
# `invesalius_rs` under its other aliases (`import invesalius_rs as transforms / cy_mesh / ...`:
# interpolation, apply_view_matrix_transform, convolve_non_zero, mask_cut, polygon2mask_rs,
# brush_mask_rs, Mesh, ca_smoothing, count_regions, jump_flooding, floodfill_voronoi,
# floodfill_auto_threshold) is forwarded, on first use, to the compiled crate installed beside this
# package — so binding this module under every alias keeps the rest of InVesalius working. Without
# the crate the attribute error says which name is missing and why.
FORWARDED = (
    "trilin_interpolate_py", "nearest_neighbour_interp", "tricub_interpolate_py", "tricub_interpolate2_py",
    "lanczos_interpolate_py", "floodfill_auto_threshold", "floodfill_voronoi", "jump_flooding",
    "mask_cut", "polygon2mask_rs", "brush_mask_rs", "_native",
)

__all__ = ["floodfill", "floodfill_threshold", "floodfill_threshold_inplace", "fill_holes_automatically", "mida", "lmip",
           "fast_countour_mip", "apply_view_matrix_transform", "count_regions", "convolve_non_zero", "Mesh", "ca_smoothing", *[n for n in FORWARDED if not n.startswith("_")]]

_crate = None


def _load_crate():
    global _crate
    if _crate is None:
        import importlib
        try:
            mod = importlib.import_module("invesalius_rs")     # the reference's own package (top level)
        except ImportError as e:
            raise ImportError("the compiled invesalius_rs crate is not installed: only the hot path "
                              f"({', '.join(__all__[:12])}) is provided by invesalius3_b200") from e
        if mod is globals().get("__spec__") or getattr(mod, "__file__", None) == __file__:
            raise ImportError("invesalius_rs resolves to this shim; install the reference crate under its own name")
        _crate = mod
    return _crate


def __getattr__(name):
    if name == "Mesh":                       # array-based Mesh of mesh_ops (no VTK needed on this side)
        return _mesh_ops().Mesh
    if name in FORWARDED:
        try:
            return getattr(_load_crate(), name)
        except ImportError as e:
            raise AttributeError(f"invesalius3_b200.invesalius_rs.{name}: {e}") from e
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
