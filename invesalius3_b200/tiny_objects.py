"""The "Remove tiny objects" plugin on the device (plugins/remove_tiny_objects/gui.py).

The plugin labels the mask body (`nd.label(mask.matrix[1:, 1:, 1:])`: 6-connected, every non-zero voxel a
feature, the edit markers 1, 2, 253 and 254 included), turns the labels into an image of region sizes
(`count_regions`), shows `(counts <= min_size) * 255` as a preview on every change of the spin control, and
on "Remove" sets `m[preview > 127] = 1` in the body. TinyObjects keeps the labels and their size table
(one uint32 per label) on the device while the dialog is open, so each preview is one launch and one
download, and a removal one upload, one launch and one download.

Quirks kept from the plugin, which the results reproduce:
- Label 0, the background, has a size too. Where it holds no more than min_size voxels it is previewed
  and "removed" (its voxels set to 1) like any other region.
- An empty body has num_labels == 0, and counts() is the number of voxels everywhere.
- A removed voxel holds 1, which is non-zero: labelled again (refresh, the plugin's on_modified_mask), it
  still belongs to its region, so the regions and their sizes do not change.
- min_size is compared with the uint32 sizes exactly, as NumPy 2 compares a uint32 array with a Python
  int: a negative min_size previews nothing, one of 2**32 or more previews everything.

The labeller takes bodies of fewer than 2**31 voxels; the preview and removal kernels index in 64 bits.
"""
from __future__ import annotations

import operator

import numpy as np
import torch

from . import _lib
from . import device as dev
from . import labeling
from .device import _p, _stream


def _min_size(min_size) -> int:
    """An int (NumPy integers included) clamped to [-1, 2**32], where the uint32 comparison's answer no
    longer changes."""
    return max(-1, min(operator.index(min_size), 2 ** 32))


def _padded_mask(mask_matrix, what: str = "mask_matrix") -> np.ndarray:
    if not isinstance(mask_matrix, np.ndarray) or mask_matrix.dtype != np.uint8 or mask_matrix.ndim != 3:
        raise TypeError(f"{what}: the padded 3-D uint8 mask matrix expected")
    if min(mask_matrix.shape) < 2:
        raise ValueError(f"{what}: the mask body is empty (shape {mask_matrix.shape})")
    return mask_matrix


class TinyObjects:
    """Device state of one open "Remove tiny objects" dialog over `mask_matrix`, the padded
    [dz + 1][dy + 1][dx + 1] uint8 mask (memmaps included).

    labels: int32 device tensor [dz][dy][dx] holding the uint32 labels of nd.label(body).
    sizes: int32 device tensor [num_labels + 1] holding the uint32 number of voxels of each label."""

    def __init__(self, mask_matrix):
        self.refresh(mask_matrix)

    def refresh(self, mask_matrix) -> None:
        """Label the body again (the plugin's on_modified_mask) and rebuild the size table."""
        m = _padded_mask(mask_matrix)
        body = dev.to_device(m[1:, 1:, 1:])
        self.labels, self.num_labels = labeling.label_device(body, None)
        del body
        self.sizes = labeling.region_sizes_device(self.labels, self.num_labels)
        self.shape = tuple(m.shape)

    @property
    def body_shape(self) -> tuple[int, int, int]:
        return tuple(self.labels.shape)

    def counts(self) -> np.ndarray:
        """count_regions(labels, num_labels): the uint32 image of each voxel's region size."""
        out = labeling.count_regions_device(self.labels, self.num_labels)
        res = np.empty(self.body_shape, np.uint32)
        dev.to_host(out, res.view(np.int32))
        return res

    def preview_device(self, min_size, out: torch.Tensor | None = None) -> torch.Tensor:
        """(counts <= min_size) * 255 as a dense uint8 device tensor of the body's shape. Does not synchronise."""
        ms = _min_size(min_size)
        if out is None:
            out = torch.empty(self.body_shape, dtype=torch.uint8, device=self.labels.device)
        dev._dense(out, "out")
        if out.dtype != torch.uint8 or tuple(out.shape) != self.body_shape or out.device != self.labels.device:
            raise ValueError("preview_device: out must be uint8 with the body's shape, on the labels' device")
        with torch.cuda.device(out.device):
            _lib.call("b2v_tiny_objects_preview", _p(self.labels), self.labels.numel(), _p(self.sizes),
                      self.sizes.numel(), ms, _p(out), _stream())
        return out

    def preview(self, min_size, out: np.ndarray | None = None) -> np.ndarray:
        """The plugin's `preview_matrix[:] = (counts <= min_size) * 255`, written into `out` (the uint8
        body-shaped preview memmap) or a new array. Returns it."""
        if out is None:
            out = np.empty(self.body_shape, np.uint8)
        elif not isinstance(out, np.ndarray) or out.dtype != np.uint8 or tuple(out.shape) != self.body_shape:
            raise ValueError(f"preview: out must be a uint8 array of shape {self.body_shape}")
        dev.to_host(self.preview_device(min_size), out)
        return out

    def _upload_mask(self, mask_matrix) -> torch.Tensor:
        m = _padded_mask(mask_matrix)
        if tuple(m.shape) != self.shape:
            raise ValueError(f"mask_matrix has shape {m.shape}, the labels were built for {self.shape}")
        return dev.to_device(m)

    def remove(self, mask_matrix, min_size) -> None:
        """Set the body voxels of every region of at most min_size voxels to 1, in `mask_matrix` (the mask as
        it is now, of the shape the labels were built for), as the plugin's preview and OnRemove do together.
        The flag planes are not changed."""
        ms = _min_size(min_size)
        t = self._upload_mask(mask_matrix)
        dz, dy, dx = self.body_shape
        with torch.cuda.device(t.device):
            _lib.call("b2v_tiny_objects_remove", _p(self.labels), dz, dy, dx, _p(self.sizes), self.sizes.numel(), ms,
                      _p(t), _stream())
        dev.to_host(t, mask_matrix)

    def apply_preview(self, mask_matrix, preview_matrix) -> None:
        """The plugin's OnRemove, literally: `mask_matrix[1:, 1:, 1:][preview_matrix > 127] = 1`."""
        p = np.asarray(preview_matrix)
        if p.dtype != np.uint8 or tuple(p.shape) != self.body_shape:
            raise ValueError(f"apply_preview: preview_matrix must be uint8 of shape {self.body_shape}")
        t = self._upload_mask(mask_matrix)
        pv = dev.to_device(p)
        dz, dy, dx = self.body_shape
        with torch.cuda.device(t.device):
            _lib.call("b2v_tiny_objects_apply_preview", _p(pv), dz, dy, dx, _p(t), _stream())
        dev.to_host(t, mask_matrix)
