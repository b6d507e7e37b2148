"""The "Region growing" tool (invesalius/data/styles.py:2991-3251) and Slice.calc_image_density
(slice_.py:2284-2297) on the device.

  get_LUT_value_255(data, window, level)                    imagedata_utils.py:540-552
  do_rg_confidence(image, mask, p, bstruct, iters, mult, ...)   styles.py:3220-3251 (3-D) and :3091-3101 (2-D)
  region_grow_3d(image, p, bstruct, method, ...)            the growth part of do_3d_seg, styles.py:3157-3203
  calc_image_density(matrix, mask_body)                     slice_.py:2288-2297

The numpy functions take the reference's arguments (the tool's config attributes become keyword
arguments) and return what it computes; the caller keeps its mask write-back and undo history.
RegionGrower keeps the image resident between clicks, so a click moves only its out_mask. Under
them is a device-tensor layer (lut255_device, masked_moments_device, confidence_grow_device).

np.std and np.mean of the selection are bit-identical to NumPy's: the device sums in NumPy's
pairwise order. Each confidence iteration selects the 3x3x3 box about the seed plus every voxel
already grown (out == 1): that is the reference's bool_mask, since out_mask only ever gains 1s.
out_mask is not cleared between iterations, so voxels already at 1 are walls for the next flood
(floodfill.rs:154): from the second iteration on, growth starts only at the seed's still-unfilled
neighbours. The reference behaves so and this module reproduces it.

Deviations, where the reference fails: a seed outside the volume raises IndexError (negative
coordinates OverflowError) before any work; an empty selection raises ValueError (NumPy would
give NaN thresholds); float thresholds on a uint8 image are truncated with int() as on int16 (the
crate's wrapper raises TypeError); a float64 image grows (the crate's wrapper passes fill as a
float and raises TypeError).
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple

import numpy as np
import torch

from . import _lib
from . import device as dev
from .device import _dense, _p, _stream
from .invesalius_rs import _SUFFIX, _extract

_MODES = {"eq": _lib.SEL_EQ, "gt127": _lib.SEL_GT127}


class Moments(NamedTuple):
    """count, min, max, mean and std of a selection (NaN statistics when count is 0)."""
    count: int
    min: float
    max: float
    mean: float
    std: float


# ----------------------------------------------------------------------------- device layer
def lut255_device(t: torch.Tensor, window, level, out: torch.Tensor | None = None) -> torch.Tensor:
    """get_LUT_value_255 on a dense int16 / uint8 / float64 tensor; the result has its dtype."""
    _dense(t, "image")
    code = dev.dtype_code(t)
    if out is None:
        out = torch.empty_like(t)
    _dense(out, "out")
    if out.dtype != t.dtype or out.shape != t.shape:
        raise TypeError("lut255_device: out must have the image's dtype and shape")
    with torch.cuda.device(t.device):
        _lib.call("b2v_lut255", _p(t), code, t.numel(), float(window), float(level), _p(out), _stream())
    return out


def _workspace(shape, device) -> torch.Tensor:
    return dev._workspace(_lib.load().b2v_masked_moments_workspace_bytes(*shape), device)


def masked_moments_device(image_t: torch.Tensor, sel_t: torch.Tensor | None, mode: str = "gt127", value: int = 0,
                          box=None, workspace: torch.Tensor | None = None) -> Moments:
    """Moments of image_t over the voxels where sel_t == value (mode "eq") or sel_t > 127 (mode
    "gt127"), OR inside box = (z0, y0, x0, z1, y1, x1) (inclusive, clipped to the volume). sel_t: a
    dense uint8 tensor of the image's shape, or None. Synchronises."""
    _dense(image_t, "image")
    if image_t.dim() != 3:
        raise TypeError("masked_moments_device: 3-D image expected")
    code = dev.dtype_code(image_t)
    if sel_t is not None:
        _dense(sel_t, "sel")
        if sel_t.dtype != torch.uint8 or sel_t.shape != image_t.shape:
            raise TypeError("masked_moments_device: sel must be uint8 with the image's shape")
    if mode not in _MODES:
        raise ValueError(f"masked_moments_device: mode must be one of {sorted(_MODES)}")
    bx = None if box is None else (C.c_int64 * 6)(*(int(v) for v in box))
    if workspace is None:
        workspace = _workspace(image_t.shape, image_t.device)
    st = _lib.Moments()
    with torch.cuda.device(image_t.device):
        _lib.call("b2v_masked_moments", _p(image_t), code, *image_t.shape, _p(sel_t), _MODES[mode], int(value), bx,
                  C.byref(st), _p(workspace), _stream())
    return Moments(int(st.count), st.min, st.max, st.mean, st.std)


def _seed(p, shape) -> tuple[int, int, int]:
    x, y, z = (int(c) for c in p)
    if min(x, y, z) < 0:
        raise OverflowError("can't convert negative int to unsigned")
    if z >= shape[0] or y >= shape[1] or x >= shape[2]:
        raise IndexError(f"seed {(x, y, z)} (x, y, z) is outside the volume {tuple(shape)} (z, y, x)")
    return x, y, z


def _flood_thresholds(t0, t1, dtype):
    """The flood's thresholds as the crate's wrapper converts them: int() and a range check for
    int16 / uint8 (OverflowError out of range), float() for float64."""
    suf = _SUFFIX[np.dtype(dtype)]
    if suf == "f64":
        return float(t0), float(t1)
    return _extract(int(t0), suf), _extract(int(t1), suf)


def confidence_grow_device(image_t: torch.Tensor, p, bstruct, iters: int, mult, out_t: torch.Tensor | None = None,
                           thresholds: list | None = None, workspace: torch.Tensor | None = None) -> torch.Tensor:
    """do_rg_confidence's loop on a resident image (already through the LUT if the tool uses WW/WL):
    `iters` times, the mean and std over the seed's box and the grown voxels give
    t0, t1 = mean -/+ std * mult, and the flood from p = (x, y, z) grows out_t (zeroed first) with 1s.
    `thresholds`, if given, receives each iteration's (t0, t1) as numpy float64."""
    _dense(image_t, "image")
    if image_t.dim() != 3:
        raise TypeError("confidence_grow_device: 3-D image expected")
    x, y, z = _seed(p, image_t.shape)
    if out_t is None:
        out_t = torch.zeros(image_t.shape, dtype=torch.uint8, device=image_t.device)
    else:
        _dense(out_t, "out")
        if out_t.dtype != torch.uint8 or out_t.shape != image_t.shape:
            raise TypeError("confidence_grow_device: out must be uint8 with the image's shape")
        out_t.zero_()
    if workspace is None:
        workspace = _workspace(image_t.shape, image_t.device)
    box = (z - 1, y - 1, x - 1, z + 1, y + 1, x + 1)
    np_dt = torch.empty(0, dtype=image_t.dtype).numpy().dtype
    for _ in range(int(iters)):
        m = masked_moments_device(image_t, out_t, "eq", 1, box, workspace)
        if m.count == 0:
            raise ValueError("confidence_grow_device: empty selection")
        var, mean = np.float64(m.std), np.float64(m.mean)
        t0 = mean - var * mult
        t1 = mean + var * mult
        if thresholds is not None:
            thresholds.append((t0, t1))
        c0, c1 = _flood_thresholds(t0, t1, np_dt)
        dev.floodfill_threshold(image_t, [(x, y, z)], c0, c1, 1, bstruct, out_t)
    return out_t


# ----------------------------------------------------------------------------- resident image
class RegionGrower:
    """One image on the device for many clicks of the region growing tool. The LUT image of the
    last (ww, wl) is cached; a click moves only its out_mask (and a mask for image_density)."""

    def __init__(self, matrix: np.ndarray, device=None):
        if not isinstance(matrix, np.ndarray) or matrix.dtype not in _SUFFIX or matrix.ndim != 3:
            raise TypeError("RegionGrower: a 3-D int16, uint8 or float64 image expected")
        self.dtype = matrix.dtype
        self.shape = matrix.shape
        self.image = dev.to_device(matrix, device)
        self._lut_key = None
        self._lut = None
        self._ws = None

    def _workspace(self) -> torch.Tensor:
        if self._ws is None:
            self._ws = _workspace(self.shape, self.image.device)
        return self._ws

    def lut(self, ww, wl) -> torch.Tensor:
        """The resident image through get_LUT_value_255(., ww, wl), cached for the last (ww, wl)."""
        key = (ww, wl)
        if self._lut_key != key:
            self._lut = lut255_device(self.image, ww, wl, self._lut)
            self._lut_key = key
        return self._lut

    def _value(self, t: torch.Tensor, p):
        x, y, z = p
        return t[z, y, x].cpu().numpy()[()]            # a numpy scalar of the image's dtype

    def confidence(self, p, bstruct, confid_iters=3, confid_mult=2.5, use_ww_wl=False, ww=None, wl=None,
                   thresholds: list | None = None) -> np.ndarray:
        """do_rg_confidence: the uint8 out_mask (0 / 1) of the image's shape."""
        _seed(p, self.shape)
        img = self.lut(ww, wl) if use_ww_wl else self.image
        out = confidence_grow_device(img, p, bstruct, confid_iters, confid_mult, thresholds=thresholds,
                                     workspace=self._workspace())
        return dev.to_numpy(out)

    def grow(self, p, bstruct, method, *, t0=None, t1=None, dev_min=25, dev_max=25, use_ww_wl=True, ww=None, wl=None,
             confid_iters=3, confid_mult=2.5) -> np.ndarray | None:
        """region_grow_3d on the resident image."""
        if method == "confidence":
            return self.confidence(p, bstruct, confid_iters, confid_mult, use_ww_wl, ww, wl)
        x, y, z = _seed(p, self.shape)
        if method == "threshold":
            img = self.image
            if t0 is None or t1 is None:
                raise ValueError("region_grow_3d: the threshold method needs t0 and t1")
        elif method == "dynamic":
            img = self.lut(ww, wl) if use_ww_wl else self.image
            v = self._value(img, (x, y, z))
            with np.errstate(over="ignore"):          # int16 / uint8 scalar arithmetic wraps, as in NumPy
                t0 = v - dev_min
                t1 = v + dev_max
        else:
            raise ValueError(f"region_grow_3d: unknown method {method!r}")
        v = self._value(img, (x, y, z))
        if v < t0 or v > t1:
            return None
        c0, c1 = _flood_thresholds(t0, t1, self.dtype)
        out = torch.zeros(self.shape, dtype=torch.uint8, device=self.image.device)
        dev.floodfill_threshold(img, [(x, y, z)], c0, c1, 1, bstruct, out)
        return dev.to_numpy(out)

    def image_density(self, mask_body: np.ndarray):
        """calc_image_density: (min, max, mean, std) of the image where mask_body > 127, or
        (0, 0, 0, 0) when no voxel is selected. mask_body: uint8 of the image's shape (the
        mask.matrix[1:, 1:, 1:] view is fine)."""
        if not isinstance(mask_body, np.ndarray) or mask_body.dtype != np.uint8 or mask_body.shape != self.shape:
            raise TypeError("calc_image_density: a uint8 mask of the image's shape expected")
        sel = dev.to_device(mask_body, self.image.device)
        m = masked_moments_device(self.image, sel, "gt127", workspace=self._workspace())
        if m.count == 0:
            return 0, 0, 0, 0
        t = self.dtype.type
        return t(m.min), t(m.max), np.float64(m.mean), np.float64(m.std)


# ----------------------------------------------------------------------------- numpy API
def get_LUT_value_255(data: np.ndarray, window, level) -> np.ndarray:
    """imagedata_utils.get_LUT_value_255: a new array of data's shape and dtype (int16, uint8 or
    float64)."""
    if not isinstance(data, np.ndarray) or data.dtype not in _SUFFIX:
        raise TypeError("get_LUT_value_255: an int16, uint8 or float64 array expected")
    t = dev.to_device(data.reshape(-1) if data.flags.c_contiguous else np.ascontiguousarray(data).reshape(-1))
    return dev.to_numpy(lut255_device(t, window, level)).reshape(data.shape)


def do_rg_confidence(image: np.ndarray, mask, p, bstruct, confid_iters, confid_mult, use_ww_wl=False, ww=None,
                     wl=None) -> np.ndarray:
    """FloodFillSegmentInteractorStyle.do_rg_confidence with the config as arguments: the uint8
    out_mask. `mask` only gives the shape (None: the image's); p = (x, y, z). The 2-D tool passes
    (1, dy, dx) arrays and a (1, 3, 3) structure."""
    if mask is not None and tuple(np.shape(mask)) != tuple(image.shape):
        raise ValueError("do_rg_confidence: mask and image shapes differ")
    return RegionGrower(image).confidence(p, bstruct, confid_iters, confid_mult, use_ww_wl, ww, wl)


def region_grow_3d(image: np.ndarray, p, bstruct, method, *, t0=None, t1=None, dev_min=25, dev_max=25, use_ww_wl=True,
                   ww=None, wl=None, confid_iters=3, confid_mult=2.5) -> np.ndarray | None:
    """The growth part of do_3d_seg: the uint8 out_mask of `method` ("threshold", "dynamic" or
    "confidence") from p = (x, y, z), or None where the reference returns early (the seed's
    value outside [t0, t1])."""
    return RegionGrower(image).grow(p, bstruct, method, t0=t0, t1=t1, dev_min=dev_min, dev_max=dev_max,
                                    use_ww_wl=use_ww_wl, ww=ww, wl=wl, confid_iters=confid_iters,
                                    confid_mult=confid_mult)


def calc_image_density(matrix: np.ndarray, mask_body: np.ndarray):
    """Slice.calc_image_density after its do_threshold_to_all_slices: (min, max, mean, std) of
    matrix[mask_body > 127] with NumPy's scalar types, or (0, 0, 0, 0)."""
    return RegionGrower(matrix).image_density(mask_body)
