"""CPU oracle for the InVesalius hot path — TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
may import this package. It restates the reference semantics (Rust crate `invesalius_rs`,
NumPy statements in `invesalius/data/slice_.py`, SciPy/skimage callees of
`watershed_process.py`, classic marching cubes for `surface_process.py`) on the CPU.
The function names and argument order follow the reference's Python boundary
(`invesalius_rs/__init__.py`), so parity tests read like the reference's own tests.

Pinning status is listed in oracle/oracle.c's header and DESIGN.md.
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
_LIB = None


def lib() -> C.CDLL:
    """liboracle.so, the one library of every C checker, loaded once per process. make decides whether it is
    stale, so the rebuild follows oracle/Makefile's prerequisites exactly and does nothing when it is not."""
    global _LIB
    if _LIB is None:
        subprocess.run(["make", "-C", str(_HERE)], check=True, capture_output=True)
        _LIB = C.CDLL(str(_HERE / "liboracle.so"))
    return _LIB


def _estrides(a: np.ndarray):
    assert all(s % a.itemsize == 0 for s in a.strides)
    return (C.c_int64 * a.ndim)(*[s // a.itemsize for s in a.strides])


def _ptr(a: np.ndarray | None):
    return C.c_void_p(None if a is None else a.ctypes.data)


def _faces3(faces) -> np.ndarray:
    """Contiguous int64 [T,3] of int32 / int64 faces [T,3] or [T,4] with a leading 3 in every row."""
    f = np.asarray(faces)
    if f.dtype not in (np.int32, np.int64):
        raise TypeError("faces: int32 or int64 expected")
    if f.ndim != 2 or f.shape[1] not in (3, 4):
        raise ValueError("faces: [T,3] or [T,4] expected")
    if f.shape[1] == 4:
        if len(f) and (f[:, 0] != 3).any():
            raise ValueError("faces: the [T,4] form needs a leading 3 in every row")
        f = f[:, 1:]
    return np.ascontiguousarray(f, dtype=np.int64)


_SUFFIX = {np.dtype(np.int16): "i16", np.dtype(np.uint8): "u8", np.dtype(np.float64): "f64"}
_CT = {"i16": C.c_int16, "u8": C.c_uint8, "f64": C.c_double}
_RANGE = {"i16": (-32768, 32767), "u8": (0, 255)}


def _suffix(a: np.ndarray, what="image") -> str:
    try:
        return _SUFFIX[a.dtype]
    except KeyError:
        raise TypeError(f"Invalid {what} type: {a.dtype}") from None


def _extract(v, suf: str):
    """PyO3 `extract::<T>()`: ints must fit T (OverflowError); floats only for f64."""
    if suf == "f64":
        return float(v)
    if isinstance(v, (float, np.floating)):
        raise TypeError("'float' object cannot be interpreted as an integer")
    v = int(v)
    lo, hi = _RANGE[suf]
    if not lo <= v <= hi:
        raise OverflowError("out of range integral type conversion attempted")
    return v


# --------------------------------------------------------------------------- threshold
def threshold(image: np.ndarray, lo, hi, mask: np.ndarray, preserve_markers: bool) -> None:
    """mask[...] = 255*[lo<=image<=hi] (markers 1/2/253/254 kept when preserve_markers).
    invesalius/data/slice_.py:1238-1246, :1731-1737."""
    assert image.dtype == np.int16 and mask.dtype == np.uint8 and image.shape == mask.shape
    dz, dy, dx = image.shape
    lib().orc_threshold_i16(_ptr(image), _estrides(image), C.c_int64(dz), C.c_int64(dy), C.c_int64(dx),
                            C.c_double(lo), C.c_double(hi), _ptr(mask), _estrides(mask), int(preserve_markers))


def do_threshold_to_a_slice_numpy(slice_matrix, mask, threshold_range):
    """The reference statements verbatim (slice_.py:1731-1737) — used as the CPU baseline."""
    thresh_min, thresh_max = threshold_range
    m = ((slice_matrix >= thresh_min) & (slice_matrix <= thresh_max)) * 255
    m[mask == 1] = 1
    m[mask == 2] = 2
    m[mask == 253] = 253
    m[mask == 254] = 254
    return m.astype("uint8")


def set_mask_threshold_numpy(matrix, mask_matrix, threshold_range):
    """Whole-volume branch of Slice.SetMaskThreshold verbatim (slice_.py:1240-1246)."""
    thresh_min, thresh_max = threshold_range
    for n, slice_ in enumerate(matrix):
        m = np.ones(slice_.shape, mask_matrix.dtype)
        m[slice_ < thresh_min] = 0
        m[slice_ > thresh_max] = 0
        m[m == 1] = 255
        mask_matrix[n + 1, 1:, 1:] = m
        mask_matrix[n + 1, 0, 0] = 1


def do_threshold_to_all_slices_numpy(matrix, mask_matrix, threshold_range):
    """Slice.do_threshold_to_all_slices verbatim (slice_.py:1762-1767)."""
    for n in range(1, mask_matrix.shape[0]):
        if mask_matrix[n, 0, 0] == 0:
            m = mask_matrix[n, 1:, 1:]
            mask_matrix[n, 1:, 1:] = do_threshold_to_a_slice_numpy(matrix[n - 1], m, threshold_range)
            mask_matrix[n, 0, 0] = 1


# --------------------------------------------------------------------------- flood fill
def _seeds(seeds):
    s = np.ascontiguousarray(np.array([tuple(int(c) for c in p) for p in seeds], dtype=np.int64).reshape(-1, 3))
    if (s < 0).any():
        raise OverflowError("can't convert negative int to unsigned")
    return s


def floodfill_threshold(data, seeds, t0, t1, fill, strct, out):
    """invesalius_rs/__init__.py:21-40 -> floodfill_py.rs:137-185 -> floodfill.rs:96-166."""
    suf = _suffix(data)
    if out.dtype != np.uint8:
        raise TypeError("Invalid output type")
    strct_u8 = np.ascontiguousarray(strct, dtype=np.uint8)
    if suf in ("i16",):
        t0, t1, fill = int(t0), int(t1), int(fill)
    elif suf == "f64":
        t0, t1, fill = float(t0), float(t1), float(fill)
    t0, t1 = _extract(t0, suf), _extract(t1, suf)
    # NB: for float64 data the reference wrapper has just turned `fill` into a float, which
    # the PyO3 signature `fill: u8` then rejects -> the f64 branch always raises TypeError.
    fill = _extract(fill, "u8")
    _floodfill_threshold_core(data, seeds, t0, t1, fill, strct_u8, out)


def _floodfill_threshold_core(data, seeds, t0, t1, fill, strct_u8, out):
    """generic_floodfill_threshold itself (floodfill.rs:96-166), past the Python/PyO3 coercions."""
    suf = _suffix(data)
    s = _seeds(seeds)
    fn = getattr(lib(), f"orc_floodfill_threshold_{suf}")
    ct = _CT[suf]
    rc = fn(_ptr(data), _estrides(data), *map(C.c_int64, data.shape), _ptr(s), C.c_int64(len(s)), ct(t0), ct(t1),
            C.c_uint8(fill), _ptr(strct_u8), *map(C.c_int64, strct_u8.shape), _ptr(out), _estrides(out))
    if rc:
        raise IndexError("seed out of bounds (Rust panic in floodfill.rs:122)")


def floodfill_threshold_inplace(data, seeds, t0, t1, fill, strct):
    """invesalius_rs/__init__.py:43-54 -> floodfill_py.rs:187-231 -> floodfill.rs:168-237."""
    suf = _suffix(data)
    strct_u8 = np.ascontiguousarray(strct, dtype=np.uint8)
    t0, t1, fill = _extract(t0, suf), _extract(t1, suf), _extract(fill, suf)
    s = _seeds(seeds)
    fn = getattr(lib(), f"orc_floodfill_threshold_inplace_{suf}")
    ct = _CT[suf]
    rc = fn(_ptr(data), _estrides(data), *map(C.c_int64, data.shape), _ptr(s), C.c_int64(len(s)), ct(t0), ct(t1),
            ct(fill), _ptr(strct_u8), *map(C.c_int64, strct_u8.shape))
    if rc:
        raise IndexError("seed out of bounds (Rust panic in floodfill.rs:194)")


def floodfill(data, i, j, k, v, fill, out):
    """floodfill_py.rs:87-135 -> floodfill.rs:5-49; (i, j, k) = (x, y, z)."""
    suf = _suffix(data)
    if out.dtype != np.uint8:
        raise TypeError("Invalid output type")
    v, fill = _extract(v, suf), _extract(fill, "u8")
    fn = getattr(lib(), f"orc_floodfill_{suf}")
    rc = fn(_ptr(data), _estrides(data), *map(C.c_int64, data.shape), C.c_int64(i), C.c_int64(j), C.c_int64(k),
            _CT[suf](v), C.c_uint8(fill), _ptr(out), _estrides(out))
    if rc:
        raise IndexError("seed out of bounds (Rust panic in floodfill.rs:21)")


def fill_holes_automatically(mask, labels, nlabels, max_size) -> bool:
    """floodfill_py.rs:233-249 -> floodfill.rs:51-94."""
    if mask.dtype != np.uint8:
        raise TypeError("Invalid mask type")
    if labels.dtype != np.uint32:
        raise TypeError("labels must be uint32")
    rc = lib().orc_fill_holes_automatically(_ptr(mask), _estrides(mask), _ptr(labels), _estrides(labels),
                                            *map(C.c_int64, mask.shape), C.c_uint32(nlabels), C.c_uint32(max_size))
    if rc < 0:
        raise IndexError("label > nlabels (Rust panic in floodfill.rs:62)")
    return bool(rc)


# --------------------------------------------------------------------------- projections
def mip(image, axis, kind):
    """NumPy reductions used by Slice.get_image_slice (slice_.py:881-886)."""
    return {"max": image.max, "min": image.min, "mean": image.mean}[kind](axis)


_MIDA_OUT = {"i16": np.int16, "u8": np.uint8, "f64": np.uint8}


def mida(image, axis, wl, ww, out):
    """invesalius_rs/__init__.py:91-95 -> mips_py.rs:161-202 -> mips.rs:102-168."""
    suf = _SUFFIX.get(image.dtype)
    if suf is None or out.dtype != _MIDA_OUT[suf]:
        raise TypeError("Invalid image or output type")
    wl, ww = _extract(int(wl), suf), _extract(int(ww), suf)
    fn = getattr(lib(), f"orc_mida_{suf}")
    rc = fn(_ptr(image), _estrides(image), *map(C.c_int64, image.shape), int(axis), C.c_float(wl), C.c_float(ww),
            _ptr(out), _estrides(out))
    if rc:
        raise ValueError("MIDA result not representable (Rust panic at mips.rs:166)")


def lmip(image, axis, tmin, tmax, out):
    """mips.rs:7-86 (called as mips.lmip by slice_.py:892 but not exported by the crate)."""
    suf = _suffix(image)
    if out.dtype != image.dtype:
        raise TypeError("Invalid image or output type")
    tmin, tmax = _extract(tmin, suf), _extract(tmax, suf)
    fn = getattr(lib(), f"orc_lmip_{suf}")
    ct = _CT[suf]
    fn(_ptr(image), _estrides(image), *map(C.c_int64, image.shape), int(axis), ct(tmin), ct(tmax), _ptr(out),
       _estrides(out))


def fcm_volume(image, n, axis):
    """The T-typed temp volume of fast_countour_mip_internal (mips.rs:235-242)."""
    suf = _suffix(image)
    tmp = np.zeros(image.shape, dtype=image.dtype)
    fn = getattr(lib(), f"orc_fcm_{suf}")
    rc = fn(_ptr(image), _estrides(image), *map(C.c_int64, image.shape), C.c_float(n), int(axis), _ptr(tmp))
    if rc:
        raise ValueError("contour intensity not representable (Rust panic at mips.rs:241)")
    return tmp


def fast_countour_mip(image, n, axis, wl, ww, tmip, out):
    """invesalius_rs/__init__.py:98-101 -> mips_py.rs:204-253 -> mips.rs:215-279."""
    suf = _SUFFIX.get(image.dtype)
    if suf is None or out.dtype != image.dtype:
        raise TypeError("Invalid image or output type")
    wl, ww = _extract(int(wl), suf), _extract(int(ww), suf)
    tmp = fcm_volume(image, n, axis)
    if tmip == 0:
        out[...] = tmp.max(axis)
    elif tmip == 1:
        lmip(tmp, axis, 700, 3033, out)  # NumCast::from(700) panics for u8 -> _extract raises
    elif tmip == 2:
        if suf == "f64":
            # mida_internal::<f64, f64>: output cast is f32 -> f64
            o8 = np.zeros(out.shape, dtype=np.float64)
            _mida_f64_f64(tmp, axis, wl, ww, o8)
            out[...] = o8
        else:
            mida(tmp, axis, wl, ww, out)


def _mida_f64_f64(image, axis, wl, ww, out):
    raise NotImplementedError("f64 contour-MIDA is outside the GPU core's dtype set")


# --------------------------------------------------------------------------- mesh smoothing
def ca_smoothing(vertices, faces, normals, T, tmax, bmin, n_iters, return_weights=False):
    """invesalius_rs.context_aware_smoothing (mesh_py.rs -> mesh.rs:27-395) on float32 vertices [V,3]
    (modified in place), int64 faces [M,4] (leading 3) and float32 face normals [M,3]. Checked by the NumPy
    restatement of tests/ca_smoothing_model.py; parity with the crate unpinned. IndexError: an entry of
    columns 1..3 outside the vertex array (the crate panics); the leading column may hold any value."""
    if vertices.dtype != np.float32 or faces.dtype != np.int64 or normals.dtype != np.float32:
        raise TypeError("ca_smoothing checker: float32 vertices, int64 faces, float32 normals")
    assert vertices.flags.c_contiguous and faces.flags.c_contiguous and normals.flags.c_contiguous and faces.shape[1] == 4
    w = np.zeros(len(vertices), np.float64)
    rc = lib().orc_ca_smoothing(_ptr(vertices), C.c_int64(len(vertices)), _ptr(faces), C.c_int64(len(faces)), _ptr(normals),
                                C.c_double(T), C.c_double(tmax), C.c_double(bmin), C.c_uint32(int(n_iters)), _ptr(w))
    if rc:
        raise IndexError("face entry (columns 1..3) outside the vertex array")
    return w if return_weights else None


# --------------------------------------------------------------------------- transforms
ORIENT = {"AXIAL": 0, "CORONAL": 1, "SAGITAL": 2}


def apply_view_matrix_transform(volume, spacing, m, n, orientation, minterpol, cval, out):
    """invesalius_rs/__init__.py:84 -> transforms_py.rs:96-148 -> transforms.rs:9-55 ->
    interpolation.rs (nearest 0, trilinear 1, tricubic 2, Lanczos-4 otherwise). PARITY UNPINNED
    (no reference test): restated in oracle/transforms.c."""
    rc = apply_view_matrix_transform_rc(volume, spacing, m, n, orientation, minterpol, cval, out)
    if rc == 4:
        raise ValueError("Lanczos-4 tap outside the volume after the one-step wrap: index out of bounds "
                         "(Rust panic in ndarray indexing, interpolation.rs:34)")
    if rc:
        raise ValueError("interpolated value not representable in the output type (Rust panic in interpolation.rs)")


def apply_view_matrix_transform_rc(volume, spacing, m, n, orientation, minterpol, cval, out):
    """apply_view_matrix_transform returning the checker's code instead of raising: 0, 3 (a cast
    panics) or 4 (a Lanczos-4 tap outside the volume); `out` is written in every case, 0 where a
    sample panics."""
    suf = _SUFFIX.get(volume.dtype)
    if suf is None or out.dtype != volume.dtype or volume.ndim != 3 or out.ndim != 3:
        raise TypeError("Invalid volume or output type")
    cval = _extract(cval if suf == "f64" else int(cval), suf)
    mm = np.ascontiguousarray(m, dtype=np.float64).reshape(16)
    sp = np.ascontiguousarray(spacing, dtype=np.float64)
    fn = getattr(lib(), f"orc_avmt_{suf}")
    rc = fn(_ptr(volume), _estrides(volume), *map(C.c_int64, volume.shape), _ptr(sp), _ptr(mm), C.c_int64(int(n)),
            ORIENT.get(orientation, 3), int(minterpol), _CT[suf](cval), _ptr(out), _estrides(out), *map(C.c_int64, out.shape))
    return rc


# --------------------------------------------------------------------------- marching cubes
def marching_cubes(volume, iso, spacing=(1.0, 1.0, 1.0), origin_index=(0, 0, 0), flip_y=True):
    """Canonical marching cubes (parity unpinned: stands in for vtkContourFilter,
    surface_process.py:172-186). volume: dense int16/uint8 [nz][ny][nx];
    spacing = (sx, sy, sz); origin_index = (ox, oy, oz) added to the (x, y, z) indices.
    Returns (vertices float32 [V,3], triangles int64 [T,3])."""
    v = np.ascontiguousarray(volume)
    dt = {np.dtype(np.int16): 0, np.dtype(np.uint8): 1}[v.dtype]
    nz, ny, nx = v.shape
    nv, nt = C.c_int64(0), C.c_int64(0)
    args = [_ptr(v), dt, C.c_int64(nz), C.c_int64(ny), C.c_int64(nx), C.c_double(iso), C.c_float(spacing[0]),
            C.c_float(spacing[1]), C.c_float(spacing[2]), C.c_int64(origin_index[0]), C.c_int64(origin_index[1]),
            C.c_int64(origin_index[2]), int(bool(flip_y))]
    lib().orc_marching_cubes(*args, None, None, C.byref(nv), C.byref(nt))
    verts = np.zeros((nv.value, 3), np.float32)
    tris = np.zeros((nt.value, 3), np.int64)
    lib().orc_marching_cubes(*args, _ptr(verts), _ptr(tris), C.byref(nv), C.byref(nt))
    return verts, tris
