"""A device-resident working set for one user action (threshold -> region grow -> surface).

The numpy-in / numpy-out functions of `slice_ops`, `invesalius_rs` and `surface_process` are what
the reference's call sites bind to, one call at a time — and each call ships its arrays over PCIe
again: the image twice, the grown mask there and back (805 MB in, 324 MB out for the 512^3 action:
32 ms per action against 1.28 ms of kernels on one H100 80GB HBM3 at a 400 W power limit). The three calls of one action read the same
image and hand each other their results, so `VolumeSession` keeps them in HBM:

    with VolumeSession(matrix) as s:                       # the int16 image goes up ONCE
        s.set_mask_threshold(mask.matrix, (tmin, tmax))    # Slice.SetMaskThreshold      slice_.py:1238-1246
        s.floodfill_threshold(seeds, t0, t1, 254, bstruct, out_mask)          # styles.py:3183-3202
        verts, faces = s.contour([127], spacing)           # create_surface_piece's contour step

Same semantics and error behaviour as the one-shot functions (they share the checks); results
still land in the caller's host arrays (memmaps included). `out` of the flood is taken to be the
freshly zeroed array the reference allocates (`np.zeros_like(mask)`, styles.py:3183) unless
`out_has_content=True`, in which case it is uploaded first like the one-shot call does.
"""
from __future__ import annotations

import numpy as np
import torch

from . import device as dev
from . import invesalius_rs as rs
from .slice_ops import _check_image
from .surface_process import _contour_device


class VolumeSession:
    def __init__(self, matrix: np.ndarray):
        _check_image(matrix, 3)
        self.shape = matrix.shape
        self.image = dev.to_device(matrix)        # int16 [dz][dy][dx], dense
        self.mask = None                          # last threshold mask (uint8, device)
        self.out = None                           # last grown mask (uint8, device)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False

    def close(self):
        self.image = self.mask = self.out = None

    # ---- Slice.SetMaskThreshold, whole-volume branch (slice_.py:1238-1246)
    def set_mask_threshold(self, mask_matrix: np.ndarray | None, threshold_range) -> torch.Tensor:
        """Thresholds the resident image; with `mask_matrix` (the padded Mask memmap, shape
        (dz+1, dy+1, dx+1)) the result is also written there and the axial flags set, as the
        reference does. Returns the device mask."""
        dz, dy, dx = self.shape
        tmin, tmax = threshold_range
        self.mask = dev.threshold(self.image, tmin, tmax, out=self.mask)
        if mask_matrix is not None:
            if mask_matrix.shape != (dz + 1, dy + 1, dx + 1) or mask_matrix.dtype != np.uint8:
                raise ValueError("mask_matrix must be uint8 of shape (dz+1, dy+1, dx+1)")
            dev.to_host(self.mask, mask_matrix[1:, 1:, 1:])
            mask_matrix[1:, 0, 0] = 1
        return self.mask

    # ---- invesalius_rs.floodfill_threshold on the resident image (floodfill_py.rs:137-183)
    def floodfill_threshold(self, seeds, t0, t1, fill, strct, out: np.ndarray | None, out_has_content: bool = False):
        """Region grow from `seeds` through t0 <= image <= t1. `out` (host uint8, same shape) receives
        the result; its previous content is only consulted (out != fill) when out_has_content."""
        t0, t1 = rs._extract(int(t0), "i16"), rs._extract(int(t1), "i16")
        fill = rs._extract(fill, "u8")
        if out is not None:
            if not isinstance(out, np.ndarray) or out.dtype != np.uint8 or out.ndim != 3:
                raise TypeError("Invalid output type")
            if out.shape != self.shape:
                raise ValueError("data and out shapes differ")
            if not out.flags.writeable:
                raise ValueError("out is read-only")
        if out is not None and out_has_content:
            self.out = dev.to_device(out)
        elif self.out is None or self.out.shape != self.image.shape:
            self.out = torch.zeros(self.shape, dtype=torch.uint8, device=self.image.device)
        else:
            self.out.zero_()
        try:
            dev.floodfill_threshold(self.image, [tuple(s) for s in seeds], t0, t1, fill,
                                    np.ascontiguousarray(strct, dtype=np.uint8), self.out)
        except ValueError as e:
            rs._seed_check(e)
        if out is not None:
            dev.to_host(self.out, out)
        return self.out

    # ---- the contour step of create_surface_piece (surface_process.py:156-186) on a resident mask
    def contour(self, isovalues=(127,), spacing=(1.0, 1.0, 1.0), z0: int = 0, flip_y: bool = True, source: str = "out",
                index_dtype=np.int32):
        """Iso-surface of the grown mask (source="out"), the threshold mask ("mask") or the image
        ("image": the Default algorithm's tmin / tmax contours). Returns numpy (vertices, faces)."""
        t = {"out": self.out, "mask": self.mask, "image": self.image}[source]
        if t is None:
            raise ValueError(f"contour: no resident {source!r} yet")
        return _contour_device(t, [float(v) for v in np.atleast_1d(isovalues)], spacing, z0, flip_y, (0, 0, 0), index_dtype)
