"""Device-resident API: the hot path on torch CUDA tensors.

PyTorch is used for device memory, streams and (in dist.py) torch.distributed only;
every computation is a kernel of libb2v.so reached through the C ABI (include/b2v.h).
All functions enqueue on torch's current stream and do not synchronise unless stated.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

_DT = {torch.int16: _lib.I16, torch.uint8: _lib.U8, torch.float64: _lib.F64}
_NP2T = {np.dtype(np.int16): torch.int16, np.dtype(np.uint8): torch.uint8, np.dtype(np.float64): torch.float64,
         np.dtype(np.uint32): torch.int32, np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32,
         np.dtype(np.int64): torch.int64}
_KIND = {"max": _lib.MIP_MAX, "min": _lib.MIP_MIN, "mean": _lib.MIP_MEAN}


def require_cuda() -> None:
    if not torch.cuda.is_available():
        raise RuntimeError("invesalius3_b200 needs a CUDA device (sm_90a, H100); there is no CPU fallback")


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t: torch.Tensor | None) -> C.c_void_p:
    return C.c_void_p(0 if t is None else t.data_ptr())


def _dense(t: torch.Tensor, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be dense C-order; pack strided views with to_device()")
    return t


def dtype_code(t: torch.Tensor) -> int:
    try:
        return _DT[t.dtype]
    except KeyError:
        raise TypeError(f"Invalid image type: {t.dtype}") from None


def _workspace(nbytes: int, device) -> torch.Tensor | None:
    return torch.empty(int(nbytes), dtype=torch.uint8, device=device) if nbytes > 0 else None


# ----------------------------------------------------------------------------- triangle meshes
# vertices float32 [V,3]; faces int32 / int64 [T,3], or [T,4] with a leading 3 (the Mesh form)
def _face_form(shape) -> int:
    if len(shape) != 2 or shape[1] not in (3, 4):
        raise ValueError("faces: [T,3] or [T,4] (leading 3) expected")
    return int(shape[1])


def _mesh_tensors(vertices, faces, caller: str) -> int:
    """Checks a mesh given as dense CUDA tensors on one device; returns the face form (3 or 4 columns)."""
    if not isinstance(vertices, torch.Tensor) or not isinstance(faces, torch.Tensor):
        raise TypeError(f"{caller}: torch tensors expected")
    if vertices.dtype != torch.float32:
        raise TypeError("vertices: float32 expected")
    if faces.dtype not in (torch.int32, torch.int64):
        raise TypeError("faces: int32 or int64 expected")
    if vertices.dim() != 2 or vertices.shape[1] != 3:
        raise ValueError("vertices: [V,3] expected")
    cols = _face_form(tuple(faces.shape))
    _dense(vertices, "vertices")
    _dense(faces, "faces")
    if faces.device != vertices.device:
        raise ValueError("vertices and faces must be on the same device")
    return cols


def _mesh_arrays(vertices, faces) -> int:
    """Checks a mesh given as numpy arrays; returns the face form (3 or 4 columns)."""
    if not isinstance(vertices, np.ndarray) or vertices.dtype != np.float32:
        raise TypeError("vertices: a float32 numpy array expected")
    if not isinstance(faces, np.ndarray) or faces.dtype not in (np.int32, np.int64):
        raise TypeError("faces: an int32 or int64 numpy array expected")
    if vertices.ndim != 2 or vertices.shape[1] != 3:
        raise ValueError("vertices: [V,3] expected")
    return _face_form(faces.shape)


def _as_form(f32: torch.Tensor, dtype: torch.dtype, cols: int) -> torch.Tensor:
    """int32 [T,3] device faces in the given dtype and form."""
    f = f32 if dtype == torch.int32 else f32.to(dtype)
    if cols == 4:
        f = torch.cat((torch.full((f.shape[0], 1), 3, dtype=dtype, device=f.device), f), 1)
    return f


# ----------------------------------------------------------------------------- transfers
def _box_pitches(a: np.ndarray):
    """(row_pitch, plane_pitch) in bytes if `a` (3-D) is an x-contiguous box view."""
    if a.ndim != 3 or a.size == 0:
        return None
    sz, sy, sx = a.strides
    if sx != a.itemsize or sy < a.shape[2] * a.itemsize or sz <= 0 or sy <= 0:
        return None
    if sz % sy != 0 or sz // sy < a.shape[1]:
        if a.shape[0] == 1:
            return sy, sy * a.shape[1]
        return None
    return sy, sz


def to_device(a: np.ndarray, device=None) -> torch.Tensor:
    """Host array (any strides, memmap views included) -> dense device tensor.

    x-contiguous 3-D box views such as `mask.matrix[1:, 1:, 1:]` are packed by the DMA
    engine (b2v_copy3d_h2d) straight from the view; anything else is made contiguous on
    the host first."""
    require_cuda()
    device = torch.device("cuda" if device is None else device)
    tdt = _NP2T.get(a.dtype)
    if tdt is None:
        raise TypeError(f"unsupported dtype {a.dtype}")
    t = torch.empty(a.shape, dtype=tdt, device=device)
    if a.size == 0:
        return t
    pit = None if a.flags.c_contiguous else _box_pitches(a)
    with torch.cuda.device(device):
        if a.flags.c_contiguous:
            # one flat copy: the DMA engine is measurably slower on 3-D copies with short rows
            _lib.call("b2v_copy3d_h2d", _p(t), C.c_void_p(a.ctypes.data), 1, 1, a.size, a.itemsize,
                      a.size * a.itemsize, a.size * a.itemsize, _stream())
        elif pit is not None:
            dz, dy, dx = a.shape
            _lib.call("b2v_copy3d_h2d", _p(t), C.c_void_p(a.ctypes.data), dz, dy, dx, a.itemsize, pit[0], pit[1],
                      _stream())
        else:
            c = np.ascontiguousarray(a)
            _lib.call("b2v_copy3d_h2d", _p(t), C.c_void_p(c.ctypes.data), 1, 1, c.size, c.itemsize,
                      c.size * c.itemsize, c.size * c.itemsize, _stream())
            torch.cuda.current_stream().synchronize()  # `c` may be a temporary
    return t


def h2d_async(dst: torch.Tensor, a: np.ndarray) -> None:
    """Enqueue host box view -> dense device tensor on the current stream, no synchronise
    (the caller keeps `a` alive and untouched until the stream is synchronised)."""
    pit = _box_pitches(a)
    if pit is None or tuple(dst.shape) != tuple(a.shape) or not dst.is_contiguous():
        raise ValueError("h2d_async needs an x-contiguous 3-D box view and a dense destination")
    dz, dy, dx = a.shape
    with torch.cuda.device(dst.device):
        _lib.call("b2v_copy3d_h2d", _p(dst), C.c_void_p(a.ctypes.data), dz, dy, dx, a.itemsize, pit[0], pit[1],
                  _stream())


def d2h_async(src: torch.Tensor, out: np.ndarray) -> None:
    """Enqueue dense device tensor -> host box view on the current stream, no synchronise."""
    pit = _box_pitches(out)
    if pit is None or tuple(src.shape) != tuple(out.shape) or not src.is_contiguous():
        raise ValueError("d2h_async needs an x-contiguous 3-D box view and a dense source")
    if not out.flags.writeable:
        raise ValueError("output array is read-only")
    dz, dy, dx = out.shape
    with torch.cuda.device(src.device):
        _lib.call("b2v_copy3d_d2h", C.c_void_p(out.ctypes.data), _p(src), dz, dy, dx, out.itemsize, pit[0], pit[1],
                  _stream())


class _PinnedPool:
    """Recycled page-locked host blocks for result arrays. `tensor.cpu()` into fresh pageable
    memory is slowed by page faults and staged copies; a DMA into pinned memory runs at PCIe
    rate, but cudaHostAlloc is slow, so blocks are pooled: a block returns
    to the pool when the numpy array handed to the caller (and every view of it) is gone."""

    def __init__(self):
        import os
        self.free: dict[int, list] = {}
        self.held = 0                    # bytes parked in `free`
        self.cap = int(os.environ.get("B2V_PINNED_POOL_MB", "2048")) << 20

    @staticmethod
    def _bucket(nbytes: int) -> int:
        """Power of two up to 64 MiB, then multiples of 64 MiB (no 2x waste on large meshes)."""
        if nbytes <= (64 << 20):
            return 1 << max(20, int(nbytes - 1).bit_length())
        return -(-nbytes // (64 << 20)) * (64 << 20)

    def take(self, nbytes: int) -> torch.Tensor:
        bucket = self._bucket(nbytes)
        lst = self.free.get(bucket)
        if lst:
            self.held -= bucket
            return lst.pop()
        return torch.empty(bucket, dtype=torch.uint8).pin_memory()

    def give(self, block: torch.Tensor) -> None:
        n = block.numel()
        lst = self.free.setdefault(n, [])
        if len(lst) < 4 and self.held + n <= self.cap:
            lst.append(block)
            self.held += n
        # otherwise the block is dropped and its page-locked memory released

    def trim(self) -> None:
        """Release every parked block."""
        self.free.clear()
        self.held = 0


_pool = _PinnedPool()


def trim_pinned_pool() -> None:
    """Release the page-locked result blocks parked by to_numpy() (cap: B2V_PINNED_POOL_MB, default 2048)."""
    _pool.trim()


def to_numpy(t: torch.Tensor) -> np.ndarray:
    """Dense device tensor -> numpy array backed by a pooled pinned block (one DMA, no
    second host copy). Synchronises."""
    import weakref
    t = t.contiguous()
    npdt = torch.empty(0, dtype=t.dtype).numpy().dtype
    nbytes = t.numel() * t.element_size()
    if nbytes == 0:
        return np.empty(tuple(t.shape), dtype=npdt)
    block = _pool.take(nbytes)
    base = block.numpy()                       # every view below keeps `base` alive
    weakref.finalize(base, _pool.give, block)
    with torch.cuda.device(t.device):
        block[:nbytes].copy_(t.view(torch.uint8).reshape(-1), non_blocking=True)
        torch.cuda.current_stream().synchronize()
    return base[:nbytes].view(npdt).reshape(tuple(t.shape))


def to_host(t: torch.Tensor, out: np.ndarray) -> None:
    """Dense device tensor -> host array `out` (written in place, any strides). Synchronises."""
    assert tuple(t.shape) == tuple(out.shape), (t.shape, out.shape)
    if out.size == 0:
        return
    if not out.flags.writeable:
        raise ValueError("output array is read-only")
    pit = None if out.flags.c_contiguous else _box_pitches(out)
    with torch.cuda.device(t.device):
        if out.flags.c_contiguous:
            _lib.call("b2v_copy3d_d2h", C.c_void_p(out.ctypes.data), _p(t), 1, 1, out.size, out.itemsize,
                      out.size * out.itemsize, out.size * out.itemsize, _stream())
            torch.cuda.current_stream().synchronize()
        elif pit is not None:
            dz, dy, dx = out.shape
            _lib.call("b2v_copy3d_d2h", C.c_void_p(out.ctypes.data), _p(t), dz, dy, dx, out.itemsize, pit[0], pit[1],
                      _stream())
            torch.cuda.current_stream().synchronize()
        else:
            tmp = np.empty(out.shape, dtype=out.dtype)
            _lib.call("b2v_copy3d_d2h", C.c_void_p(tmp.ctypes.data), _p(t), 1, 1, tmp.size, tmp.itemsize,
                      tmp.size * tmp.itemsize, tmp.size * tmp.itemsize, _stream())
            torch.cuda.current_stream().synchronize()
            out[...] = tmp


# ----------------------------------------------------------------------------- threshold
def _int_range(lo, hi):
    """Inclusive bounds on an integer image: a float bound is equivalent to ceil/floor."""
    lo = int(np.ceil(lo))
    hi = int(np.floor(hi))
    lo = max(lo, -(2 ** 31) + 1)
    hi = min(hi, 2 ** 31 - 1)
    return lo, hi


def threshold(img: torch.Tensor, lo, hi, out: torch.Tensor | None = None,
              preserve_markers: bool = False) -> torch.Tensor:
    """out = 255*[lo <= img <= hi] as uint8, same shape; with preserve_markers the old
    values 1, 2, 253, 254 of `out` survive (slice_.py:1238-1246 / :1731-1737)."""
    _dense(img, "img")
    if img.dtype != torch.int16:
        raise TypeError("threshold: image must be int16")
    if out is None:
        if preserve_markers:
            raise ValueError("preserve_markers needs the previous mask in `out`")
        out = torch.empty(img.shape, dtype=torch.uint8, device=img.device)
    _dense(out, "out")
    if out.dtype != torch.uint8 or out.shape != img.shape:
        raise TypeError("threshold: out must be uint8 with the image's shape")
    lo, hi = _int_range(lo, hi)
    with torch.cuda.device(img.device):
        _lib.call("b2v_threshold_i16", _p(img), img.numel(), lo, hi, _p(out), int(preserve_markers), _stream())
    return out


def threshold_masklayout(img: torch.Tensor, lo, hi, mask_padded: torch.Tensor, preserve_markers: bool,
                         only_dirty: bool) -> torch.Tensor:
    """Threshold into the padded Mask layout [dz+1][dy+1][dx+1] incl. axial flags."""
    _dense(img, "img")
    _dense(mask_padded, "mask_padded")
    dz, dy, dx = img.shape
    if img.dtype != torch.int16 or mask_padded.dtype != torch.uint8:
        raise TypeError("threshold_masklayout: int16 image and uint8 mask expected")
    if tuple(mask_padded.shape) != (dz + 1, dy + 1, dx + 1):
        raise ValueError("mask_padded must have shape (dz+1, dy+1, dx+1)")
    lo, hi = _int_range(lo, hi)
    with torch.cuda.device(img.device):
        _lib.call("b2v_threshold_i16_masklayout", _p(img), dz, dy, dx, lo, hi, _p(mask_padded),
                  int(preserve_markers), int(only_dirty), _stream())
    return mask_padded


# ----------------------------------------------------------------------------- projections
def mip(img: torch.Tensor, axis: int, kind: str = "max", out: torch.Tensor | None = None) -> torch.Tensor:
    """MaxIP / MinIP / MeanIP == tmp_array.max/min/mean(axis) (slice_.py:881-886)."""
    _dense(img, "img")
    if img.dim() != 3:
        raise ValueError("mip: 3-D volume expected")
    code = dtype_code(img)
    k = _KIND[kind]
    dz, dy, dx = img.shape
    oshape = [(dy, dx), (dz, dx), (dz, dy)][axis]
    odt = torch.float64 if kind == "mean" else img.dtype
    if out is None:
        out = torch.empty(oshape, dtype=odt, device=img.device)
    _dense(out, "out")
    if tuple(out.shape) != oshape or out.dtype != odt:
        raise TypeError("mip: bad output shape/dtype")
    lib = _lib.load()
    ws = _workspace(lib.b2v_mip_workspace_bytes(code, dz, dy, dx, axis, k), img.device)
    with torch.cuda.device(img.device):
        _lib.call("b2v_mip", _p(img), code, dz, dy, dx, axis, k, _p(out), _p(ws), _stream())
    return out


def minmax(img: torch.Tensor) -> torch.Tensor:
    """float32 [min, max] of the whole buffer, left on the device (mips.rs:113-122)."""
    _dense(img, "img")
    code = dtype_code(img)
    lib = _lib.load()
    ws = _workspace(lib.b2v_minmax_workspace_bytes(img.numel()), img.device)
    out = torch.empty(2, dtype=torch.float32, device=img.device)
    with torch.cuda.device(img.device):
        _lib.call("b2v_minmax_f32", _p(img), code, img.numel(), _p(out), _p(ws), _stream())
    return out


# ----------------------------------------------------------------------------- flood fill
def _seed_array(seeds) -> np.ndarray:
    s = np.array([tuple(int(c) for c in p) for p in seeds], dtype=np.int64).reshape(-1, 3)
    if (s < 0).any():
        raise OverflowError("can't convert negative int to unsigned")
    return np.ascontiguousarray(s)


def _strct_array(strct) -> np.ndarray:
    st = np.ascontiguousarray(strct, dtype=np.uint8)
    if st.ndim != 3:
        raise TypeError("strct must be a 3-D array")
    return st


def floodfill_threshold(data: torch.Tensor, seeds, t0, t1, fill: int, strct, out: torch.Tensor,
                        stats: dict | None = None) -> int:
    """Region grow from `seeds` ((x, y, z) triples) through voxels with t0 <= data <= t1 that
    are not already `fill` in `out`; reached voxels get out = fill (floodfill.rs:96-166).
    Returns the number of flood rounds. Synchronises the stream. `stats` (optional dict)
    receives `tiles`, the tile count of the flood, and `rounds`, the persistent kernel's own
    round count (0 when the host-driven rounds ran)."""
    _dense(data, "data"); _dense(out, "out")
    if out.dtype != torch.uint8 or out.shape != data.shape or data.dim() != 3:
        raise TypeError("floodfill_threshold: out must be uint8 with data's 3-D shape")
    code = dtype_code(data)
    s, st = _seed_array(seeds), _strct_array(strct)
    dz, dy, dx = data.shape
    lib = _lib.load()
    ws = _workspace(lib.b2v_floodfill_workspace_bytes(dz, dy, dx, len(s)), data.device)
    rounds = C.c_int(0)
    with torch.cuda.device(data.device):
        _lib.call("b2v_floodfill_threshold", _p(data), code, dz, dy, dx, C.c_void_p(s.ctypes.data), len(s),
                  float(t0), float(t1), int(fill), C.c_void_p(st.ctypes.data), *st.shape, _p(out), _p(ws), _stream(),
                  C.byref(rounds))
    if stats is not None and ws is not None:
        lay = (C.c_int64 * 8)()
        _lib.call("b2v_floodfill_layout", dz, dy, dx, max(len(s), 1), lay)
        ctl = ws[lay[6]: lay[6] + 64].view(torch.int32).cpu().tolist()
        stats.update(tiles=int(lay[4]), rounds=ctl[7])
    return rounds.value


def floodfill_threshold_inplace(data: torch.Tensor, seeds, t0, t1, fill, strct) -> int:
    """floodfill.rs:168-237: as floodfill_threshold, reading and writing `data` itself."""
    _dense(data, "data")
    if data.dim() != 3:
        raise TypeError("floodfill_threshold_inplace: 3-D volume expected")
    code = dtype_code(data)
    s, st = _seed_array(seeds), _strct_array(strct)
    dz, dy, dx = data.shape
    lib = _lib.load()
    ws = _workspace(lib.b2v_floodfill_workspace_bytes(dz, dy, dx, len(s)), data.device)
    rounds = C.c_int(0)
    with torch.cuda.device(data.device):
        _lib.call("b2v_floodfill_threshold_inplace", _p(data), code, dz, dy, dx, C.c_void_p(s.ctypes.data), len(s),
                  float(t0), float(t1), float(fill), C.c_void_p(st.ctypes.data), *st.shape, _p(ws), _stream(),
                  C.byref(rounds))
    return rounds.value


def floodfill(data: torch.Tensor, i: int, j: int, k: int, v, fill: int, out: torch.Tensor) -> int:
    """floodfill.rs:5-49: 6-connected fill of data == v from (x=i, y=j, z=k); seed always marked."""
    _dense(data, "data"); _dense(out, "out")
    if out.dtype != torch.uint8 or out.shape != data.shape or data.dim() != 3:
        raise TypeError("floodfill: out must be uint8 with data's 3-D shape")
    code = dtype_code(data)
    dz, dy, dx = data.shape
    lib = _lib.load()
    ws = _workspace(lib.b2v_floodfill_workspace_bytes(dz, dy, dx, 1), data.device)
    rounds = C.c_int(0)
    with torch.cuda.device(data.device):
        _lib.call("b2v_floodfill_equal", _p(data), code, dz, dy, dx, int(i), int(j), int(k), float(v), int(fill),
                  _p(out), _p(ws), _stream(), C.byref(rounds))
    return rounds.value


def fill_holes_automatically(mask: torch.Tensor, labels: torch.Tensor, nlabels: int, max_size: int) -> bool:
    """floodfill.rs:51-94. labels: int32 tensor holding the uint32 label image."""
    _dense(mask, "mask"); _dense(labels, "labels")
    if mask.dtype != torch.uint8:
        raise TypeError("Invalid mask type")
    if labels.dtype != torch.int32 or labels.shape != mask.shape:
        raise TypeError("labels must be a uint32 (int32-typed tensor) image of the mask's shape")
    lib = _lib.load()
    ws = _workspace(lib.b2v_fill_holes_workspace_bytes(int(nlabels)), mask.device)
    mod = C.c_int(0)
    with torch.cuda.device(mask.device):
        _lib.call("b2v_fill_holes", _p(mask), _p(labels), mask.numel(), int(nlabels), int(max_size), _p(ws),
                  _stream(), C.byref(mod))
    return bool(mod.value)
