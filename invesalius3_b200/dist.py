"""Z-sharded multi-GPU versions of the hot path: one process per GPU, torch.distributed
(NCCL over NVLink on the GPU box, gloo in the CPU protocol tests).

The reference's only decomposition is the Z-piece split of surface extraction
(invesalius/data/surface.py:1360-1381, stitched in surface_process.py:229-268); here every
op of the path is sharded the same way (SURVEY.md section 8e):

  threshold            independent voxels: no communication
  MaxIP/MinIP/MeanIP   axis 1/2: rows stay with their shard (optional all_gather);
                       axis 0: partial planes, one all_reduce
  MIDA / LMIP axis 1/2 all_reduce of the global (min, max) for MIDA, then local rays;
                       axis 0: the per-ray state is handed from shard to shard (bit-exact)
  contour-MIP          the contour volume on the extended slab (halo planes feed the central
                       differences), then the sharded MaxIP / LMIP / MIDA of its own planes
  watershed            local convergence with frozen halo planes, boundary planes swapped (costs,
                       then keys + label sets) until no halo plane improves
  labelling            local labels of the own planes, one all_gather of the counts; the next
                       shard's first plane of labels sent down (4 x dy x dx bytes); each boundary's
                       pairs reduced to a spanning forest (one pair per non-root label on the two
                       planes), the forests all_gathered and resolved alike on every rank, then one
                       relabel pass: SciPy's numbering of the whole volume, no iteration
  fill holes           per-shard label histogram, one all_reduce, local apply; fill_holes_auto
                       labels the unselected voxels with the sharded labelling first
  flood fill           local convergence on slab + one halo plane per inner side, then the
                       reached bits of the two shared planes are swapped with each neighbour
                       (2 x dy x dx/8 bytes) and merged; repeat until no shard gains a bit.
                       With a PeerLink (NVLink peer mailboxes) the whole loop — rounds, plane
                       exchange, the "anyone gained?" vote — runs inside ONE persistent kernel
                       per GPU (b2v_floodfill_threshold_peer); without one (gloo tests, no
                       peer access) it is staged through torch.distributed.
  marching cubes       each shard contours its slab plus the next shard's first plane; the
                       vertices of that shared plane are owned by the next shard, whose
                       per-word records (one plane) and vertex base are sent down; counts
                       are exchanged for the global bases (PeerLink: one small kernel writes
                       them into every mailbox; otherwise all_gather + send/recv).
                       Concatenating the shards' outputs in rank order is bit-identical to the
                       single-GPU mesh.

All tensors handed to these functions are "extended slabs": the shard's own planes plus
one halo plane below (if it has a lower neighbour) and above (if it has an upper one);
`exchange_halo` fills the halo planes. The orchestration is backend-agnostic (tensors may
live on CPU under gloo); the compute itself is delegated to a backend object — the
product backend is `DeviceBackend` (libb2v.so kernels); tests substitute a CPU checker.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch
import torch.distributed as dist


@dataclass
class ZShard:
    """This rank's slab of a [DZ, dy, dx] volume split evenly along z."""
    DZ: int
    rank: int
    world: int
    group: object = None

    @property
    def z0(self) -> int:
        return self.DZ * self.rank // self.world

    @property
    def z1(self) -> int:
        return self.DZ * (self.rank + 1) // self.world

    @property
    def has_lo(self) -> bool:
        return self.rank > 0

    @property
    def has_hi(self) -> bool:
        return self.rank < self.world - 1

    @property
    def ze0(self) -> int:          # first plane of the extended slab
        return self.z0 - int(self.has_lo)

    @property
    def ze1(self) -> int:
        return self.z1 + int(self.has_hi)

    @property
    def nz_ext(self) -> int:
        return self.ze1 - self.ze0

    def interior(self, ext: torch.Tensor) -> torch.Tensor:
        return ext[int(self.has_lo): ext.shape[0] - int(self.has_hi)]

    def bounds(self, r: int):
        return self.DZ * r // self.world, self.DZ * (r + 1) // self.world

    def local_seeds(self, seeds):
        """Global (x, y, z) seeds that fall inside the extended slab, in local coordinates."""
        out = []
        for s in seeds:
            x, y, z = (int(c) for c in s)
            if not (0 <= z < self.DZ):
                raise IndexError(f"seed {s} outside the volume")
            if self.ze0 <= z < self.ze1:
                out.append((x, y, z - self.ze0))
        return out


class PeerLink:
    """NVLink peer mailboxes of one job (csrc/peer.cuh): every rank allocates one mailbox in its
    HBM, exports it with cudaIpc, and maps everyone else's. The handles travel once through
    torch.distributed (all_gather_object); afterwards the sharded flood fill and the
    marching-cubes stitch exchange their boundary data with plain stores over NVLink from
    inside their own kernels — no NCCL call, no host round trip per exchange.
    `epoch` is the job-wide exchange counter every rank advances identically."""

    def __init__(self, shard: ZShard, dy: int, dx: int):
        from . import _lib, device
        device.require_cuda()
        self._lib = _lib
        lib = _lib.load()
        self.shard, self.dy, self.dx = shard, int(dy), int(dx)
        self.plane_bytes = self.dy * ((self.dx + 31) // 32) * 4
        self.bytes = int(lib.b2v_peer_mailbox_bytes(self.dy, self.dx))
        own = C.c_void_p(0)
        handle = (C.c_uint8 * 64)()
        _lib.call("b2v_peer_alloc", self.bytes, C.byref(own), handle)
        self.own = own.value
        handles = [None] * shard.world
        dist.all_gather_object(handles, bytes(handle), group=shard.group)
        self.ptrs = (C.c_void_p * shard.world)()
        self._mapped = []
        for r, h in enumerate(handles):
            if r == shard.rank:
                self.ptrs[r] = self.own
                continue
            p = C.c_void_p(0)
            buf = (C.c_uint8 * 64).from_buffer_copy(h)
            _lib.call("b2v_peer_open", buf, C.byref(p))
            self.ptrs[r] = p.value
            self._mapped.append(p.value)
        self.epoch = 1
        self.last_rounds = 0
        self.barrier()          # proves that every mailbox is mapped and writable from every rank

    def barrier(self):
        from .device import _stream
        self._lib.call("b2v_peer_barrier", self.shard.rank, self.shard.world, self.ptrs, self.plane_bytes, self.epoch,
                       _stream())
        self.epoch += 1

    def fits(self, dy: int, dx: int) -> bool:
        return int(dy) * ((int(dx) + 31) // 32) * 4 <= self.plane_bytes

    def mc_inbox(self, epoch: int) -> int:
        """Device address of the upper neighbour's plane-0 records for `epoch`."""
        return self.own + int(self._lib.load().b2v_peer_mc_inbox_offset(self.plane_bytes, epoch))

    def describe(self) -> str:
        return (f"peer mailboxes over NVLink (cudaIpc, {self.bytes >> 10} KiB per rank): flood planes + vote inside "
                f"the persistent kernel, MC counts/records by one exchange kernel; no NCCL on the data path")

    def close(self):
        for p in self._mapped:
            try:
                self._lib.call("b2v_peer_close", C.c_void_p(p))
            except Exception:   # noqa: BLE001
                pass
        self._mapped = []
        if self.own:
            try:
                self._lib.call("b2v_peer_free", C.c_void_p(self.own))
            except Exception:   # noqa: BLE001
                pass
            self.own = 0


def peer_link(shard: ZShard, dy: int, dx: int):
    """A PeerLink for shards with dy x dx planes, or None when the job cannot use one (gloo
    backend, CPU tensors, several ranks on one GPU, no peer access between the devices)."""
    if shard.world < 2 or not torch.cuda.is_available():
        return None
    if dist.get_backend(shard.group) != "nccl" or shard.world > 16:
        return None
    try:
        return PeerLink(shard, dy, dx)
    except Exception as e:   # noqa: BLE001
        import warnings
        warnings.warn(f"peer mailboxes unavailable, falling back to torch.distributed exchanges: {e}")
        return None


def _stage(shard: ZShard, t: torch.Tensor):
    """gloo moves host memory only: CUDA tensors are staged through the host under gloo
    (single-GPU protocol tests); under NCCL they travel device to device over NVLink."""
    if t is not None and t.is_cuda and dist.get_backend(shard.group) == "gloo":
        return t.cpu()
    return t


def _all_reduce(shard: ZShard, t: torch.Tensor, op):
    h = _stage(shard, t)
    dist.all_reduce(h, op=op, group=shard.group)
    if h is not t:
        t.copy_(h)
    return t


def _bytes(t: torch.Tensor) -> torch.Tensor:
    """Neither NCCL nor gloo moves int16: everything travels as raw bytes."""
    return t.contiguous().view(torch.uint8)


def _swap(shard: ZShard, send_lo, send_hi, like_lo=None, like_hi=None):
    """Send `send_lo` to the lower neighbour and `send_hi` to the upper one; returns what
    they sent us (recv_lo, recv_hi). Either side may be absent (None). Both neighbours
    must exchange tensors of the same shape and dtype."""
    ops, recv_lo, recv_hi = [], None, None
    if shard.has_lo:
        src = _stage(shard, _bytes(send_lo))
        recv_lo = torch.empty_like(src)
        ops.append(dist.P2POp(dist.isend, src, shard.rank - 1, group=shard.group))
        ops.append(dist.P2POp(dist.irecv, recv_lo, shard.rank - 1, group=shard.group))
    if shard.has_hi:
        src = _stage(shard, _bytes(send_hi))
        recv_hi = torch.empty_like(src)
        ops.append(dist.P2POp(dist.isend, src, shard.rank + 1, group=shard.group))
        ops.append(dist.P2POp(dist.irecv, recv_hi, shard.rank + 1, group=shard.group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    if recv_lo is not None:
        recv_lo = recv_lo.to(send_lo.device).view(send_lo.dtype).view(send_lo.shape)
    if recv_hi is not None:
        recv_hi = recv_hi.to(send_hi.device).view(send_hi.dtype).view(send_hi.shape)
    return recv_lo, recv_hi


def _send_up(shard: ZShard, t: torch.Tensor):
    """Blocking send of `t` to the next shard."""
    dist.send(_stage(shard, _bytes(t)), shard.rank + 1, group=shard.group)


def _recv_from_below(shard: ZShard, like: torch.Tensor) -> torch.Tensor:
    """Blocking receive, from the previous shard, of a tensor shaped like `like`."""
    buf = torch.empty_like(_stage(shard, _bytes(like)))
    dist.recv(buf, shard.rank - 1, group=shard.group)
    return buf.to(like.device).view(like.dtype).view(like.shape)


def _broadcast_from_last(shard: ZShard, t: torch.Tensor) -> torch.Tensor:
    h = _stage(shard, _bytes(t))
    dist.broadcast(h, shard.world - 1, group=shard.group)
    return h.to(t.device).view(t.dtype).view(t.shape)


def _rays_along_z(shard: ZShard, new_state, walk, out_like, gather):
    """Rays that cross the shards (MIDA / LMIP along z): the per-ray state travels up the chain
    of shards, every shard walking its own planes in turn — the operation order per ray is the
    whole-volume one, so the image is bit-exact. The last shard holds the image; with
    gather=True it is broadcast. (The chain is sequential; pipelining pixel tiles through it
    is the next step.)"""
    state = new_state()
    first, last = not shard.has_lo, not shard.has_hi
    if not first:
        state.copy_(_recv_from_below(shard, state))
    out = walk(state, first, last)
    if not last:
        _send_up(shard, state)
    if not gather:
        return out
    if out is None:
        out = out_like()
    return _broadcast_from_last(shard, out)


def _all_gather_rows(shard: ZShard, rows: torch.Tensor, sizes):
    """all_gather of per-shard row blocks of unequal height (padded to the tallest)."""
    m = max(sizes)
    r2 = rows.contiguous().reshape(rows.shape[0], -1)
    h = _stage(shard, _bytes(r2))
    if h.shape[0] < m:
        h = torch.cat([h, torch.zeros((m - h.shape[0], h.shape[1]), dtype=h.dtype, device=h.device)])
    buf = torch.empty((shard.world * m, h.shape[1]), dtype=h.dtype, device=h.device)
    dist.all_gather_into_tensor(buf, h.contiguous(), group=shard.group)
    parts = torch.cat([buf[r * m: r * m + n] for r, n in enumerate(sizes)])
    return parts.to(rows.device).view(rows.dtype).reshape((sum(sizes),) + tuple(rows.shape[1:]))


def exchange_halo(ext: torch.Tensor, shard: ZShard) -> torch.Tensor:
    """Fill the halo planes of an extended slab from the neighbours' boundary planes."""
    lo = int(shard.has_lo)
    n = ext.shape[0]
    first = ext[lo] if shard.has_lo else None
    last = ext[n - 1 - int(shard.has_hi)] if shard.has_hi else None
    recv_lo, recv_hi = _swap(shard, first, last)
    if recv_lo is not None:
        ext[0].copy_(recv_lo)
    if recv_hi is not None:
        ext[n - 1].copy_(recv_hi)
    return ext


# ------------------------------------------------------------------------------ device backend
class DeviceBackend:
    """Compute through libb2v.so on this rank's CUDA device."""

    def __init__(self):
        from . import _lib, device
        self._lib, self.dev = _lib, device
        device.require_cuda()

    # -- threshold / projections
    def threshold(self, img, lo, hi, out=None, preserve_markers=False):
        return self.dev.threshold(img, lo, hi, out, preserve_markers)

    def mip(self, img, axis, kind):
        return self.dev.mip(img, axis, kind)

    def sum_axis0(self, img):
        # partial sums for MeanIP axis 0 (tiny plane op); float64 volumes are summed in float64
        return img.sum(dim=0, dtype=torch.float64 if img.dtype.is_floating_point else torch.int64)

    def minmax(self, img):
        return self.dev.minmax(img)

    def mida(self, img, axis, wl, ww, minmax):
        from . import projection
        return projection.mida(img, axis, wl, ww, minmax=minmax)

    def lmip(self, img, axis, tmin, tmax):
        from . import projection
        return projection.lmip(img, axis, tmin, tmax)

    def fcm_volume(self, img, n, axis):
        from . import projection
        return projection.fcm_volume(img, n, axis)

    def ray_state(self, img):
        from . import projection
        return projection.ray_state(img)

    def mida_z(self, img, wl, ww, minmax, state, first, last):
        from . import projection
        return projection.mida_z_partial(img, wl, ww, minmax, state, first, last)

    def lmip_z(self, img, tmin, tmax, state, first, last):
        from . import projection
        return projection.lmip_z_partial(img, tmin, tmax, state, first, last)

    # -- flood fill
    def ff_begin(self, data, out, seeds, t0, t1, fill, strct):
        dev, lib = self.dev, self._lib.load()
        dz, dy, dx = data.shape
        s, st = dev._seed_array(seeds), dev._strct_array(strct)
        ws = dev._workspace(lib.b2v_floodfill_workspace_bytes(dz, dy, dx, max(len(s), 1)), data.device)
        lay = (C.c_int64 * 8)()
        self._lib.call("b2v_floodfill_layout", dz, dy, dx, max(len(s), 1), lay)
        state = dict(data=data, out=out, seeds=s, strct=st, t0=float(t0), t1=float(t1), fill=int(fill), ws=ws,
                     round=C.c_int(0), lay=list(lay), nseeds=max(len(s), 1), merged_round=None)
        self._staged(state, 1)
        return state

    def _staged(self, st, stages):
        dev = self.dev
        data, s, strct = st["data"], st["seeds"], st["strct"]
        dz, dy, dx = data.shape
        with torch.cuda.device(data.device):
            self._lib.call("b2v_floodfill_threshold_staged", stages, dev._p(data), dev.dtype_code(data), dz, dy, dx,
                           C.c_void_p(s.ctypes.data if len(s) else 0), len(s), st["t0"], st["t1"], st["fill"],
                           C.c_void_p(strct.ctypes.data), *strct.shape, dev._p(st["out"]), dev._p(st["ws"]),
                           dev._stream(), C.byref(st["round"]))

    def ff_converge(self, st):
        self._staged(st, 2)

    def _plane_view(self, st, z):
        off, pb = st["lay"][1], st["lay"][3]
        return st["ws"][off + z * pb: off + (z + 1) * pb].view(torch.int32)

    def ff_get_planes(self, st, zs):
        return torch.stack([self._plane_view(st, z) for z in zs])

    def ff_merge_planes(self, st, zs, planes):
        dev = self.dev
        dz, dy, dx = st["data"].shape
        r = st["round"].value
        st["merged_round"] = r
        with torch.cuda.device(st["data"].device):
            for z, pl in zip(zs, planes):
                pl = pl.contiguous()
                self._lib.call("b2v_floodfill_merge_plane", dz, dy, dx, st["nseeds"], dev._p(st["ws"]), int(z),
                               dev._p(pl), r, dev._stream())

    def ff_changed(self, st):
        """int32 [1] tensor: did the last merge add bits (is round `round` active)?"""
        off = st["lay"][2] + 4 * st["round"].value
        return st["ws"][off: off + 4].view(torch.int32).clone()

    def ff_finish(self, st):
        self._staged(st, 4)

    # -- fill holes (labels of the whole mask; sizes summed over the shards)
    def fh_hist(self, mask, labels, nlabels):
        dev, lib = self.dev, self._lib.load()
        ws = dev._workspace(lib.b2v_fill_holes_workspace_bytes(int(nlabels)), mask.device)
        st = dict(mask=mask, labels=labels, nlabels=int(nlabels), ws=ws, mod=C.c_int(0))
        self._fh(st, 1, 0)
        return st

    def _fh(self, st, stages, max_size):
        dev = self.dev
        with torch.cuda.device(st["mask"].device):
            self._lib.call("b2v_fill_holes_staged", stages, dev._p(st["mask"]), dev._p(st["labels"]), st["mask"].numel(),
                           st["nlabels"], int(max_size), dev._p(st["ws"]), dev._stream(), C.byref(st["mod"]))

    def fh_sizes(self, st):
        """int32 view (uint32 bits) of the label sizes inside the workspace: all-reduced in place."""
        return st["ws"][256: 256 + 4 * (st["nlabels"] + 1)].view(torch.int32)

    def fh_apply(self, st, max_size):
        self._fh(st, 2, max_size)
        return bool(st["mod"].value)

    # -- labelling (own planes only; labels are int32 tensors holding uint32 ids)
    def lb_local(self, fg, structure):
        from . import labeling
        return labeling.label_device(fg, structure)

    def lb_boundary(self, lo_plane, hi_plane, structure, base_lo, n_lo, n_hi):
        """int64 [m, 2] spanning-forest pairs (P, P(root)) of the boundary between lo_plane (my last
        plane) and hi_plane (the next shard's first plane)."""
        dev, lib = self.dev, self._lib.load()
        lo_plane, hi_plane = lo_plane.contiguous(), hi_plane.contiguous()
        ny, nx = lo_plane.shape
        ws = dev._workspace(lib.b2v_label_boundary_workspace_bytes(ny, nx, int(n_lo), int(n_hi)), lo_plane.device)
        m = C.c_int64(0)
        with torch.cuda.device(lo_plane.device):
            self._lib.call("b2v_label_boundary_count", dev._p(lo_plane), dev._p(hi_plane), ny, nx,
                           C.c_void_p(structure.ctypes.data), *structure.shape, int(n_lo), int(n_hi), dev._p(ws),
                           dev._stream(), C.byref(m))
            pairs = torch.empty((m.value, 2), dtype=torch.int64, device=lo_plane.device)
            self._lib.call("b2v_label_boundary_emit", dev._p(lo_plane), dev._p(hi_plane), ny, nx, int(n_lo), int(n_hi),
                           int(base_lo), m.value, dev._p(pairs), dev._p(ws), dev._stream())
        return pairs

    def lb_resolve(self, pairs, base, nlocal):
        """(lut, |M|): the int32 (uint32 bits) table [nlocal + 1] of my labels' final ids."""
        dev, lib = self.dev, self._lib.load()
        pairs = pairs.contiguous()
        ends = torch.unique(pairs.reshape(-1))          # sorted: compacts the endpoints
        lut = torch.empty(int(nlocal) + 1, dtype=torch.int32, device=pairs.device)
        ws = dev._workspace(lib.b2v_label_resolve_workspace_bytes(ends.numel()), pairs.device)
        nm = C.c_int64(0)
        with torch.cuda.device(pairs.device):
            self._lib.call("b2v_label_resolve", dev._p(pairs), pairs.shape[0], dev._p(ends), ends.numel(), int(base),
                           int(nlocal), dev._p(lut), dev._p(ws), dev._stream(), C.byref(nm))
        return lut, int(nm.value)

    def lb_relabel(self, labels, lut):
        with torch.cuda.device(labels.device):
            self._lib.call("b2v_label_relabel", self.dev._p(labels), labels.numel(), self.dev._p(lut), lut.numel(),
                           self.dev._stream())
        return labels

    # -- watershed (extended slab; halo planes frozen)
    def ws_preprocess(self, image_i16, use_ww_wl, wl, ww, global_min=None):
        """The uint16 cost image (LUT, or shift by the GLOBAL minimum: int16 arithmetic wraps like NumPy's)."""
        from . import watershed_process as wp
        if use_ww_wl:
            return wp.lut_u16(image_i16, ww, wl)
        out = torch.empty_like(image_i16)
        mm = torch.tensor([float(global_min), 0.0], dtype=torch.float32, device=image_i16.device)
        with torch.cuda.device(image_i16.device):
            self._lib.call("b2v_ws_shift_i16_with", self.dev._p(image_i16), image_i16.numel(), self.dev._p(mm),
                           self.dev._p(out), self.dev._stream())
        return out

    def ws_local_min(self, image_i16):
        return int(self.dev.minmax(image_i16)[0].item())

    def ws_gradient(self, pre, size):
        from . import watershed_process as wp
        return wp.morphological_gradient_u16(pre, size)

    def ws_begin(self, cost_u16, markers_i16, mode, frozen_lo, frozen_hi):
        dev, lib = self.dev, self._lib.load()
        nz, ny, nx = cost_u16.shape
        ws = dev._workspace(lib.b2v_ws_workspace_bytes(nz, ny, nx), cost_u16.device)
        st = dict(img=cost_u16, mk=markers_i16.contiguous(), mode=int(mode), lo=int(frozen_lo), hi=int(frozen_hi), ws=ws,
                  rounds=C.c_int(0), labels=None, amb=None)
        self._ws_run(st, 1)
        return st

    def _ws_run(self, st, stages):
        dev = self.dev
        nz, ny, nx = st["img"].shape
        with torch.cuda.device(st["img"].device):
            self._lib.call("b2v_ws_flood_staged", stages, dev._p(st["img"]), dev._p(st["mk"]), nz, ny, nx, st["mode"],
                           st["lo"], st["hi"], dev._p(st["labels"]), dev._p(st["amb"]), dev._p(st["ws"]), dev._stream(),
                           C.byref(st["rounds"]))

    def ws_converge(self, st, what):
        self._ws_run(st, 2 if what == 0 else 8)

    def ws_label_begin(self, st):
        self._ws_run(st, 4)

    def ws_get_plane(self, st, what, z):
        dev, lib = self.dev, self._lib.load()
        nz, ny, nx = st["img"].shape
        buf = torch.empty(int(lib.b2v_ws_plane_bytes(ny, nx, what)), dtype=torch.uint8, device=st["img"].device)
        with torch.cuda.device(buf.device):
            self._lib.call("b2v_ws_plane", 0, what, nz, ny, nx, st["mode"], st["lo"], st["hi"], int(z), dev._p(buf),
                           dev._p(st["ws"]), dev._stream(), None)
        return buf

    def ws_merge_plane(self, st, what, z, plane):
        dev = self.dev
        nz, ny, nx = st["img"].shape
        ch = C.c_int(0)
        plane = plane.contiguous()
        with torch.cuda.device(plane.device):
            self._lib.call("b2v_ws_plane", 1, what, nz, ny, nx, st["mode"], st["lo"], st["hi"], int(z), dev._p(plane),
                           dev._p(st["ws"]), dev._stream(), C.byref(ch))
        return int(ch.value)

    def ws_finish(self, st, want_ambiguous):
        st["labels"] = torch.empty(st["img"].shape, dtype=torch.int16, device=st["img"].device)
        st["amb"] = torch.empty(st["img"].shape, dtype=torch.uint8, device=st["img"].device) if want_ambiguous else None
        self._ws_run(st, 16)
        return st["labels"], st["amb"]

    # -- marching cubes
    def mc_count(self, vol, iso, skip_last):
        dev, lib = self.dev, self._lib.load()
        nz, ny, nx = vol.shape
        ws = dev._workspace(lib.b2v_mc_workspace_bytes(nz, ny, nx), vol.device)
        nv, nt = C.c_int64(0), C.c_int64(0)
        with torch.cuda.device(vol.device):
            self._lib.call("b2v_mc_count_shard", dev._p(vol), dev.dtype_code(vol), nz, ny, nx, float(iso),
                           int(bool(skip_last)), dev._p(ws), dev._stream(), C.byref(nv), C.byref(nt))
        lay = (C.c_int64 * 4)()
        self._lib.call("b2v_mc_layout", nz, ny, nx, lay)
        return dict(vol=vol, iso=float(iso), ws=ws, V=nv.value, T=nt.value, lay=list(lay), skip_last=bool(skip_last))

    def mc_plane0_records(self, st):
        off, pb = st["lay"][0], st["lay"][1]
        return st["ws"][off: off + pb].view(torch.int32).clone()

    def mc_emit(self, st, spacing, origin_index, flip_y, vbase, foreign, foreign_base):
        dev = self.dev
        vol = st["vol"]
        nz, ny, nx = vol.shape
        verts = torch.empty((st["V"], 3), dtype=torch.float32, device=vol.device)
        tris = torch.empty((st["T"], 3), dtype=torch.int32, device=vol.device)
        if st["V"] or st["T"]:
            with torch.cuda.device(vol.device):
                self._lib.call("b2v_mc_emit_shard", dev._p(vol), dev.dtype_code(vol), nz, ny, nx, st["iso"],
                               dev._p(st["ws"]), float(spacing[0]), float(spacing[1]), float(spacing[2]),
                               int(origin_index[0]), int(origin_index[1]), int(origin_index[2]), int(bool(flip_y)),
                               int(st["skip_last"]), int(vbase), dev._p(foreign), int(foreign_base), dev._p(verts),
                               dev._p(tris), dev._stream())
        return verts, tris


_default_backend = None


def _backend(b):
    global _default_backend
    if b is not None:
        return b
    if _default_backend is None:
        _default_backend = DeviceBackend()
    return _default_backend


# ------------------------------------------------------------------------------ sharded ops
def threshold(img_slab, lo, hi, shard: ZShard, out=None, preserve_markers=False, backend=None):
    """Independent voxels: purely local."""
    return _backend(backend).threshold(img_slab, lo, hi, out, preserve_markers)


def mip(img_slab, axis, kind, shard: ZShard, gather=True, backend=None):
    """MaxIP/MinIP/MeanIP of the whole volume from per-shard slabs (own planes only)."""
    be = _backend(backend)
    if axis == 0:
        if kind == "mean":
            part = be.sum_axis0(img_slab)
            _all_reduce(shard, part, dist.ReduceOp.SUM)
            # tensor / tensor is a true IEEE division (tensor / python-scalar multiplies by the
            # reciprocal on CUDA and would differ from NumPy's mean in the last bit)
            return part.to(torch.float64) / torch.full((), float(shard.DZ), dtype=torch.float64, device=part.device)
        part = be.mip(img_slab, 0, kind)
        # NCCL has no int16: integer planes travel as int32; float64 planes as they are
        wide = part if part.dtype.is_floating_point else part.to(torch.int32)
        _all_reduce(shard, wide, dist.ReduceOp.MAX if kind == "max" else dist.ReduceOp.MIN)
        return wide.to(img_slab.dtype)
    rows = be.mip(img_slab, axis, kind)
    if not gather:
        return rows
    sizes = [shard.bounds(r)[1] - shard.bounds(r)[0] for r in range(shard.world)]
    return _all_gather_rows(shard, rows, sizes)


def mida(img_slab, axis, wl, ww, shard: ZShard, gather=True, backend=None):
    """MIDA of the whole volume from per-shard slabs. The only global quantity is the (min,
    max) pair of mips.rs:113-122 — two 4-byte all_reduces. Rays along y or x (axis 1 / 2) stay
    inside a shard; rays along z (axis 0) cross the shards and hand their state (fmax, alpha,
    colour) from shard to shard (with gather=False only the last shard returns the image)."""
    be = _backend(backend)
    mm = be.minmax(img_slab).clone()
    lo, hi = mm[0:1].clone(), mm[1:2].clone()
    _all_reduce(shard, lo, dist.ReduceOp.MIN)
    _all_reduce(shard, hi, dist.ReduceOp.MAX)
    mm = torch.cat([lo, hi])
    if axis == 0:
        odt = {torch.int16: torch.int16, torch.uint8: torch.uint8, torch.float64: torch.uint8}[img_slab.dtype]
        return _rays_along_z(
            shard, lambda: be.ray_state(img_slab),
            lambda state, first, last: be.mida_z(img_slab, wl, ww, mm, state, first, last),
            lambda: torch.empty(img_slab.shape[1:], dtype=odt, device=img_slab.device), gather)
    rows = be.mida(img_slab, axis, wl, ww, mm)
    if not gather:
        return rows
    sizes = [shard.bounds(r)[1] - shard.bounds(r)[0] for r in range(shard.world)]
    return _all_gather_rows(shard, rows, sizes)


def lmip(img_slab, axis, tmin, tmax, shard: ZShard, gather=True, backend=None):
    """LMIP (mips.rs:7-86): rays along y or x are purely local rows; rays along z hand (running
    maximum, inside-range seen, finished) from shard to shard."""
    be = _backend(backend)
    if axis == 0:
        return _rays_along_z(
            shard, lambda: be.ray_state(img_slab),
            lambda state, first, last: be.lmip_z(img_slab, tmin, tmax, state, first, last),
            lambda: torch.empty(img_slab.shape[1:], dtype=img_slab.dtype, device=img_slab.device), gather)
    rows = be.lmip(img_slab, axis, tmin, tmax)
    if not gather:
        return rows
    sizes = [shard.bounds(r)[1] - shard.bounds(r)[0] for r in range(shard.world)]
    return _all_gather_rows(shard, rows, sizes)


def fast_countour_mip(img_ext, n, axis, wl, ww, tmip, shard: ZShard, gather=True, backend=None):
    """Contour-enhanced projection (mips.rs:215-279) of the Z-sharded volume: any axis, tmip 0
    (maximum), 1 (LMIP 700 / 3033) or 2 (MIDA). img_ext is the extended slab with valid halo planes
    (exchange_halo). As in the reference the contour volume comes first (b2v_fcm_volume): on the
    extended slab the central differences of a shard's first and last own plane read the
    neighbour's plane, and clamp only at the true ends of the volume (mips.rs:170-195), so the own
    planes are exact and the halo planes' values are dropped. The projection of the own planes is
    then the sharded projection of any volume: rows stay local for rays along y / x, partial planes
    are all-reduced (MaxIP) or the ray state travels up the chain of shards (LMIP, MIDA) for rays
    along z, and MIDA's extrema are all-reduced over the own planes of the contour volume."""
    if tmip not in (0, 1, 2):
        raise ValueError("fast_countour_mip: tmip must be 0, 1 or 2")
    if tmip == 1 and img_ext.dtype == torch.uint8:
        raise ValueError("fast_countour_mip: LMIP bounds 700/3033 do not fit uint8")   # the reference panics
    be = _backend(backend)
    tmp = shard.interior(be.fcm_volume(img_ext, n, axis)).contiguous()
    if tmip == 0:
        return mip(tmp, axis, "max", shard, gather=gather, backend=backend)
    if tmip == 1:
        return lmip(tmp, axis, 700, 3033, shard, gather=gather, backend=backend)
    return mida(tmp, axis, wl, ww, shard, gather=gather, backend=backend)


def _floodfill_peer(data_ext, seeds_local, t0, t1, fill, strct, out_ext, shard: ZShard, link: PeerLink):
    """The fused path: ONE persistent kernel per GPU runs the rounds, pushes / merges the boundary
    planes through the peer mailboxes and takes the job-wide vote (b2v_floodfill_threshold_peer)."""
    from . import _lib, device as dev
    s, st = dev._seed_array(seeds_local), dev._strct_array(strct)
    dz, dy, dx = data_ext.shape
    if dz < 2 or not link.fits(dy, dx):
        raise ValueError("the shard's planes do not fit this PeerLink")
    dev._dense(data_ext, "data"); dev._dense(out_ext, "out")
    if out_ext.dtype != torch.uint8 or out_ext.shape != data_ext.shape:
        raise TypeError("floodfill_threshold: out must be uint8 with data's 3-D shape")
    ws = dev._workspace(_lib.load().b2v_floodfill_workspace_bytes(dz, dy, dx, max(len(s), 1)), data_ext.device)
    rounds, used = C.c_int(0), C.c_int(0)
    try:
        with torch.cuda.device(data_ext.device):
            _lib.call("b2v_floodfill_threshold_peer", dev._p(data_ext), dev.dtype_code(data_ext), dz, dy, dx,
                      C.c_void_p(s.ctypes.data if len(s) else 0), len(s), float(t0), float(t1), int(fill),
                      C.c_void_p(st.ctypes.data), *st.shape, dev._p(out_ext), dev._p(ws), dev._stream(), shard.rank,
                      shard.world, link.ptrs, link.plane_bytes, link.epoch, C.byref(rounds), C.byref(used))
    finally:
        link.epoch += used.value
    link.last_rounds = rounds.value     # flood rounds inside the kernel (all exchanges together)
    return used.value


def floodfill_threshold(data_ext, seeds, t0, t1, fill, strct, out_ext, shard: ZShard, backend=None,
                        max_outer=10000, link: PeerLink | None = None):
    """Region grow over the Z-sharded volume. data_ext / out_ext are extended slabs with
    valid halo planes (exchange_halo). seeds are GLOBAL (x, y, z). Returns the number of
    outer (exchange) iterations. With `link` (and the device backend) the exchange is fused
    into the persistent flood kernel over NVLink peer memory; otherwise it is staged through
    torch.distributed."""
    if link is not None and backend is None:
        return _floodfill_peer(data_ext, shard.local_seeds(seeds), t0, t1, fill, strct, out_ext, shard, link)
    be = _backend(backend)
    st = be.ff_begin(data_ext, out_ext, shard.local_seeds(seeds), t0, t1, fill, strct)
    n = data_ext.shape[0]
    outer = 0
    while True:
        be.ff_converge(st)
        outer += 1
        # both copies of the two planes around each inner boundary: [halo, first own] below,
        # [last own, halo] above
        lo_z = [0, 1] if shard.has_lo else []
        hi_z = [n - 2, n - 1] if shard.has_hi else []
        send_lo = be.ff_get_planes(st, lo_z) if lo_z else None
        send_hi = be.ff_get_planes(st, hi_z) if hi_z else None
        recv_lo, recv_hi = _swap(shard, send_lo, send_hi)
        zs, planes = [], []
        if recv_lo is not None:
            zs += lo_z
            planes += [recv_lo[0], recv_lo[1]]
        if recv_hi is not None:
            zs += hi_z
            planes += [recv_hi[0], recv_hi[1]]
        be.ff_merge_planes(st, zs, planes)
        flag = be.ff_changed(st)
        _all_reduce(shard, flag, dist.ReduceOp.MAX)
        if int(flag.item()) == 0:
            break
        if outer >= max_outer:
            raise RuntimeError("sharded flood fill did not converge")
    be.ff_finish(st)
    return outer


def _marching_cubes_peer(vol, iso, spacing, origin_index, flip_y, shard: ZShard, link: PeerLink):
    """Counts and plane-0 records travel through the peer mailboxes (one exchange kernel queued
    behind classify); the host reads every rank's (V, T) in the same copy as its own."""
    from . import _lib, device as dev
    dev._dense(vol, "vol")
    nz, ny, nx = vol.shape
    if not link.fits(ny, nx):
        raise ValueError("the shard's planes do not fit this PeerLink")
    code = dev.dtype_code(vol)
    lib = _lib.load()
    ws = dev._workspace(lib.b2v_mc_workspace_bytes(nz, ny, nx), vol.device)
    counts = (C.c_int64 * (2 * shard.world))()
    epoch = link.epoch
    link.epoch += 1
    with torch.cuda.device(vol.device):
        _lib.call("b2v_mc_count_shard_peer", dev._p(vol), code, nz, ny, nx, float(iso), int(shard.has_hi), dev._p(ws),
                  dev._stream(), shard.rank, shard.world, link.ptrs, link.plane_bytes, epoch, counts)
        allc = np.frombuffer(counts, dtype=np.int64).reshape(shard.world, 2)
        vbases = np.cumsum(allc[:, 0]) - allc[:, 0]
        total_v, total_t = int(allc[:, 0].sum()), int(allc[:, 1].sum())
        if total_v >= 2 ** 31:
            raise ValueError("more than 2^31 vertices: int32 indices overflow")
        V, T = int(allc[shard.rank, 0]), int(allc[shard.rank, 1])
        verts = torch.empty((V, 3), dtype=torch.float32, device=vol.device)
        tris = torch.empty((T, 3), dtype=torch.int32, device=vol.device)
        fbase = int(vbases[shard.rank + 1]) if shard.has_hi else 0
        ox, oy, oz = origin_index
        if V or T:
            _lib.call("b2v_mc_emit_shard", dev._p(vol), code, nz, ny, nx, float(iso), dev._p(ws), float(spacing[0]),
                      float(spacing[1]), float(spacing[2]), int(ox), int(oy), int(oz + shard.z0), int(bool(flip_y)),
                      int(shard.has_hi), int(vbases[shard.rank]), C.c_void_p(link.mc_inbox(epoch)), fbase,
                      dev._p(verts), dev._p(tris), dev._stream())
    return verts, tris, int(vbases[shard.rank]), total_v, total_t


def marching_cubes(vol_ext_hi, iso, spacing, origin_index, flip_y, shard: ZShard, backend=None,
                   link: PeerLink | None = None):
    """Iso-surface of the Z-sharded volume. vol_ext_hi = this shard's own planes followed by
    the next shard's first plane (no lower halo). origin_index = (ox, oy, oz) of the GLOBAL
    volume; the shard's z offset is added here. Returns (vertices, triangles, vertex_base,
    total_vertices, total_triangles): triangle indices are global; concatenating all shards
    in rank order gives the single-GPU mesh."""
    if link is not None and backend is None:
        return _marching_cubes_peer(vol_ext_hi, iso, spacing, origin_index, flip_y, shard, link)
    be = _backend(backend)
    st = be.mc_count(vol_ext_hi, iso, skip_last=shard.has_hi)
    counts = torch.tensor([[st["V"], st["T"]]], dtype=torch.int64, device=vol_ext_hi.device)
    allc = _all_gather_rows(shard, counts, [1] * shard.world).cpu()
    vbases = torch.cumsum(allc[:, 0], 0) - allc[:, 0]
    total_v, total_t = int(allc[:, 0].sum()), int(allc[:, 1].sum())
    if total_v >= 2 ** 31:
        raise ValueError("more than 2^31 vertices: int32 indices overflow")
    # my plane-0 records go to the lower neighbour; I need the upper neighbour's
    rec = be.mc_plane0_records(st)
    _, foreign = _swap(shard, rec if shard.has_lo else None, rec if shard.has_hi else None,
                       like_lo=rec, like_hi=rec)
    fbase = int(vbases[shard.rank + 1]) if shard.has_hi else 0
    ox, oy, oz = origin_index
    verts, tris = be.mc_emit(st, spacing, (ox, oy, oz + shard.z0), flip_y, int(vbases[shard.rank]), foreign, fbase)
    return verts, tris, int(vbases[shard.rank]), total_v, total_t


def watershed(image_ext, markers_ext, bstruct, algorithm, mg_size, use_ww_wl, wl, ww, shard: ZShard, backend=None,
              return_ambiguous=False, max_outer=100000):
    """do_watershed (invesalius/data/watershed_process.py:19-60) over the Z-sharded volume.
    image_ext (int16) and markers_ext are extended slabs with valid halo planes. Returns the int16
    labels of the shard's OWN planes (with return_ambiguous also the uint8 mask of the voxels whose
    label depends on the reference's queue order) and the number of plane exchanges.

    Pre-processing is local (the shift needs the global minimum: one all_reduce; the gradient of
    the own planes needs one halo plane each side, so mg_size <= 3 along z; its halo planes are
    exchanged afterwards). Each phase of the flood then alternates local convergence (halo planes
    frozen) with a swap of the boundary planes — costs in phase 1, keys + label sets in phase 2 —
    until no shard's halo plane improves (all_reduce of the changed flag). The fixed point is the
    single-GPU one: costs only ever decrease towards the unique minimax field, keys towards the
    unique (hops, label) minimum, label sets grow towards the unique closure."""
    be = _backend(backend)
    st3 = np.asarray(bstruct)
    six = np.zeros((3, 3, 3), bool)
    six[1, 1, :] = six[1, :, 1] = six[:, 1, 1] = True
    if st3.shape != (3, 3, 3) or not np.array_equal(st3.astype(bool) | (np.arange(27).reshape(3, 3, 3) == 13), six):
        raise NotImplementedError("dist.watershed: 6-connected structuring element only")
    mode = 1 if algorithm == "Watershed" else 0
    if use_ww_wl:
        pre = be.ws_preprocess(image_ext, True, wl, ww)
    else:
        mn = torch.tensor([be.ws_local_min(shard.interior(image_ext))], dtype=torch.int32, device=image_ext.device)
        _all_reduce(shard, mn, dist.ReduceOp.MIN)
        pre = be.ws_preprocess(image_ext, False, wl, ww, global_min=int(mn.item()))
    if mode == 1:
        sz = mg_size if np.isscalar(mg_size) else mg_size[0]
        if int(sz) > 3:
            raise NotImplementedError("dist.watershed: mg_size > 3 along z needs more than one halo plane")
        pre = be.ws_gradient(pre, mg_size)
        exchange_halo(pre, shard)          # the halo planes' own gradient needs planes this shard does not hold
    mk = markers_ext.to(torch.int16)
    if mode == 0 and not use_ww_wl:
        mk = mk.to(torch.int8).to(torch.int16)      # markers.astype('int8'), watershed_process.py:57
    st = be.ws_begin(pre, mk, mode, shard.has_lo, shard.has_hi)
    n = pre.shape[0]
    exchanges = 0
    for what in (0, 1):
        if what == 1:
            be.ws_label_begin(st)
        while True:
            be.ws_converge(st, what)
            send_lo = be.ws_get_plane(st, what, 1) if shard.has_lo else None          # my first own plane
            send_hi = be.ws_get_plane(st, what, n - 2) if shard.has_hi else None      # my last own plane
            recv_lo, recv_hi = _swap(shard, send_lo, send_hi)
            exchanges += 1
            changed = 0
            if recv_lo is not None:
                changed |= be.ws_merge_plane(st, what, 0, recv_lo)
            if recv_hi is not None:
                changed |= be.ws_merge_plane(st, what, n - 1, recv_hi)
            flag = torch.tensor([changed], dtype=torch.int32, device=pre.device)
            _all_reduce(shard, flag, dist.ReduceOp.MAX)
            if int(flag.item()) == 0:
                break
            if exchanges >= max_outer:
                raise RuntimeError("sharded watershed did not converge")
    labels, amb = be.ws_finish(st, return_ambiguous)
    labels = shard.interior(labels)
    if return_ambiguous:
        return labels, shard.interior(amb), exchanges
    return labels, exchanges


def fill_holes_automatically(mask_slab, labels_slab, nlabels, max_size, shard: ZShard, backend=None) -> bool:
    """fill_holes_automatically (invesalius/data/mask.py:519-562 -> floodfill.rs:51-94) on a
    Z-sharded mask. labels_slab holds this shard's planes of the label image of the WHOLE mask
    (uint32 bits in an int32 tensor). The only global quantity is the size of every label: each
    shard histograms its planes, one all_reduce (uint32 sums wrap like the reference's) makes the
    sizes global, then every shard rewrites its own voxels. Returns the reference's bool (any label
    qualified), identical on every rank."""
    be = _backend(backend)
    st = be.fh_hist(mask_slab, labels_slab, nlabels)
    _all_reduce(shard, be.fh_sizes(st), dist.ReduceOp.SUM)
    return be.fh_apply(st, max_size)


def label(fg_slab, structure, shard: ZShard, backend=None):
    """scipy.ndimage.label of the Z-sharded volume: fg_slab is this shard's own planes (uint8 / bool,
    non-zero = feature, no halo). Returns (labels, total): an int32 tensor holding the uint32 labels of
    the own planes, numbered as SciPy numbers the whole volume, and the number of labels of the whole
    volume, identical on every rank.

    Each shard labels its slab (local labels 1..n_r in its raster order); provisional id base_r + l,
    base_r the lower shards' label count (one all_gather). With a structure 3 wide along z, the next
    shard sends its first plane of local labels down (4 dy dx bytes) and each boundary reduces its
    pairs to a spanning forest, one pair per non-root label on the two planes; the forests are
    all_gathered, every rank resolves them alike (union-find, root = smallest id) and relabels its
    slab through a table. Final = rank of the component's smallest provisional id, which is the rank
    of its first voxel in raster order: SciPy's numbering. Four collectives, whatever the volume."""
    from . import labeling
    if shard.DZ < shard.world:
        raise ValueError(f"dist.label: {shard.DZ} planes cannot give each of {shard.world} shards one")
    if fg_slab.dim() != 3 or fg_slab.shape[0] != shard.z1 - shard.z0:
        raise ValueError(f"dist.label: expected this shard's {shard.z1 - shard.z0} own planes")
    st = labeling._structure(structure, 3)
    be = _backend(backend)
    labels, n = be.lb_local(fg_slab, st)
    dev = labels.device
    counts = _all_gather_rows(shard, torch.tensor([[int(n)]], dtype=torch.int64, device=dev), [1] * shard.world)
    counts = [int(c) for c in counts.reshape(-1).cpu()]
    base = sum(counts[:shard.rank])
    pairs = torch.zeros((0, 2), dtype=torch.int64, device=dev)
    if st.shape[0] == 3 and st[2].any() and shard.world > 1:
        ops, hi_plane = [], None
        if shard.has_lo:
            ops.append(dist.P2POp(dist.isend, _stage(shard, labels[0].contiguous()), shard.rank - 1, group=shard.group))
        if shard.has_hi:
            hi_plane = _stage(shard, torch.empty_like(labels[0]))
            ops.append(dist.P2POp(dist.irecv, hi_plane, shard.rank + 1, group=shard.group))
        for req in dist.batch_isend_irecv(ops):
            req.wait()
        if shard.has_hi:
            pairs = be.lb_boundary(labels[-1], hi_plane.to(dev), st, base, counts[shard.rank], counts[shard.rank + 1])
        sizes = _all_gather_rows(shard, torch.tensor([[pairs.shape[0]]], dtype=torch.int64, device=dev), [1] * shard.world)
        sizes = [int(c) for c in sizes.reshape(-1).cpu()]
        if sum(sizes):      # padded here: a shard may have no pairs to send
            m = max(sizes)
            mine = torch.zeros((m, 2), dtype=torch.int64, device=dev)
            mine[:pairs.shape[0]] = pairs
            every = _all_gather_rows(shard, mine, [m] * shard.world)
            pairs = torch.cat([every[r * m: r * m + c] for r, c in enumerate(sizes)])
    lut, merged = be.lb_resolve(pairs, base, n)
    total = sum(counts) - merged
    if total >= 2 ** 32:
        raise ValueError("dist.label: more than 2^32 - 1 labels do not fit uint32")
    if n and (base or pairs.shape[0]):
        be.lb_relabel(labels, lut)
    return labels, total


def fill_holes_auto(mask_slab, conn, size, shard: ZShard, backend=None) -> bool:
    """labeling.fill_holes_auto (Mask.fill_holes_auto, mask.py:523-537) on a Z-sharded mask body:
    mask_slab is this shard's own planes (uint8), rewritten in place. The unselected voxels are labelled
    with dist.label, then fill_holes_automatically fills the components of at most `size` voxels with
    254. No label image of the whole mask exists anywhere. Returns the same bool on every rank."""
    from scipy.ndimage import generate_binary_structure
    if mask_slab.dtype != torch.uint8 or mask_slab.dim() != 3:
        raise TypeError("Invalid mask type")
    st = generate_binary_structure(3, {6: 1, 18: 2, 26: 3}[conn])
    labels, n = label((~(mask_slab > 127)).to(torch.uint8), st, shard, backend=backend)
    if n == 0:
        return False
    return fill_holes_automatically(mask_slab, labels, n, int(size), shard, backend=backend)
