"""CPU checker for `do_watershed` (invesalius/data/watershed_process.py:19-60) — TEST
INFRASTRUCTURE ONLY.

  get_LUT_value            the reference's NumPy statements verbatim (imagedata_utils.py:555-564)
  morphological_gradient   scipy.ndimage (the true callee; SciPy 1.18.1 here, 1.14.0 pinned upstream)
  watershed_ift            scipy.ndimage (the true callee)
  watershed (skimage)      restated in oracle/watershed.c (scikit-image absent) — parity unpinned
"""
from __future__ import annotations

import ctypes as C

import numpy as np
from scipy import ndimage

from . import _ptr, lib


def get_LUT_value(data: np.ndarray, window: int, level: int) -> np.ndarray:
    shape = data.shape
    data_ = data.ravel()
    data = np.piecewise(
        data_,
        [data_ <= (level - 0.5 - (window - 1) / 2), data_ > (level - 0.5 + (window - 1) / 2)],
        [0, window, lambda data_: ((data_ - (level - 0.5)) / (window - 1) + 0.5) * (window)],
    )
    data.shape = shape
    return data


def watershed_skimage(image_u16: np.ndarray, markers_i16: np.ndarray, bstruct) -> np.ndarray:
    img = np.ascontiguousarray(image_u16, dtype=np.uint16)
    mk = np.ascontiguousarray(markers_i16, dtype=np.int16)
    st = np.ascontiguousarray(bstruct, dtype=np.uint8)
    if img.ndim == 2:
        img, mk, st = img[None], mk[None], st[None]
    out = np.zeros(img.shape, np.int16)
    lib().orc_watershed_skimage(_ptr(img), _ptr(mk), *map(C.c_int64, img.shape), _ptr(st), *map(C.c_int64, st.shape),
                                _ptr(out))
    return out.reshape(np.shape(image_u16))


def preprocess(image, use_ww_wl, wl, ww):
    """The uint16 cost image both algorithms start from (watershed_process.py:36,42,50,55)."""
    if use_ww_wl:
        return get_LUT_value(image, ww, wl).astype("uint16")
    return (image - image.min()).astype("uint16")


def do_watershed_array(image, markers, bstruct, algorithm, mg_size, use_ww_wl, wl, ww) -> np.ndarray:
    """do_watershed without the memmap/queue plumbing: returns tmp_mask."""
    pre = preprocess(image, use_ww_wl, wl, ww)
    if algorithm == "Watershed":
        grad = ndimage.morphological_gradient(pre, mg_size)
        return watershed_skimage(grad, markers.astype("int16"), bstruct)
    mk = markers.astype("int16") if use_ww_wl else markers.astype("int8")
    return ndimage.watershed_ift(pre, mk, bstruct)


MULTI = np.iinfo(np.int32).min


def order_independence_model(image_u16, markers_i16, bstruct, mode):
    """(cost uint32, label set int32) of oracle/watershed.c::orc_ws_model: set == label where
    the reference's answer cannot depend on its queue order, MULTI where it can, 0 unreachable.
    mode 0 = scipy.ndimage.watershed_ift, mode 1 = skimage.segmentation.watershed."""
    img = np.ascontiguousarray(image_u16, dtype=np.uint16)
    mk = np.ascontiguousarray(markers_i16, dtype=np.int16)
    st = np.ascontiguousarray(bstruct, dtype=np.uint8)
    if img.ndim == 2:
        img, mk, st = img[None], mk[None], st[None]
    cost = np.zeros(img.shape, np.uint32)
    sets = np.zeros(img.shape, np.int32)
    lib().orc_ws_model(_ptr(img), _ptr(mk), *map(C.c_int64, img.shape), _ptr(st), *map(C.c_int64, st.shape),
                       C.c_int(mode), _ptr(cost), _ptr(sets))
    return cost.reshape(np.shape(image_u16)), sets.reshape(np.shape(image_u16))


def ift_scipy_restated(image_u16, markers_i16, bstruct, quirk=True):
    """oracle/watershed.c::orc_ift_scipy — pointer-faithful restatement of SciPy's watershed_ift
    (quirk=True) or the algorithm as intended (quirk=False). Returns (labels int16, number of
    sole-element events)."""
    img = np.ascontiguousarray(image_u16, dtype=np.uint16)
    mk = np.ascontiguousarray(markers_i16, dtype=np.int16)
    st = np.ascontiguousarray(bstruct, dtype=np.uint8)
    if img.ndim == 2:
        img, mk, st = img[None], mk[None], st[None]
    out = np.zeros(img.shape, np.int16)
    sole = C.c_int64(0)
    lib().orc_ift_scipy(_ptr(img), _ptr(mk), *map(C.c_int64, img.shape), _ptr(st), *map(C.c_int64, st.shape),
                        C.c_int(1 if quirk else 0), _ptr(out), C.byref(sole))
    return out.reshape(np.shape(image_u16)), sole.value


def ws_labels(image_u16, markers_i16, bstruct, mode, return_hops=False):
    """oracle/watershed.c::orc_ws_labels — the device flood's complete labelling rule (b2v_ws_flood,
    DESIGN.md section 6) in O(N): labels (int16: fewest hops along cost-optimal edges, then the
    smaller label; 0 unreached) and the ambiguous mask (uint8: two different labels reach the voxel
    along cost-optimal edges); with return_hops also the hop counts (uint32, 0xffffffff unreached).
    Any structuring element; mode 0 = watershed_ift's cost and flat-array neighbourhood, mode 1 =
    skimage's cost, proper bounds."""
    img = np.ascontiguousarray(image_u16, dtype=np.uint16)
    mk = np.ascontiguousarray(markers_i16, dtype=np.int16)
    st = np.ascontiguousarray(bstruct, dtype=np.uint8)
    if img.ndim == 2:
        img, mk, st = img[None], mk[None], st[None]
    if img.shape != mk.shape or st.ndim != 3:
        raise ValueError("ws_labels: image and markers must share a 3-D shape, with a 3-D structure")
    labels = np.empty(img.shape, np.int16)
    amb = np.empty(img.shape, np.uint8)
    hops = np.empty(img.shape, np.uint32) if return_hops else None
    rc = lib().orc_ws_labels(_ptr(img), _ptr(mk), *map(C.c_int64, img.shape), _ptr(st), *map(C.c_int64, st.shape),
                             C.c_int(mode), _ptr(labels), _ptr(amb), _ptr(hops) if return_hops else None)
    if rc != 0:
        raise MemoryError("ws_labels: out of memory")
    shape = np.shape(image_u16)
    out = (labels.reshape(shape), amb.reshape(shape))
    return out + (hops.reshape(shape),) if return_hops else out
