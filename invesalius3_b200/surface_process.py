"""Surface extraction with the reference's piece semantics (numpy in, numpy out).

`contour_piece` reproduces what `create_surface_piece` does up to and including the
contour filter (invesalius/data/surface_process.py:71-186): ROI slicing, optional 1-voxel
border padding (`pad_image`, :52-68), the to_vtk extent/origin arithmetic
(converters.py:34-101), the Y flip about the origin and the iso values (127 on the mask
for Binary / ca_smoothing, tmin and tmax on the image for Default). It returns the mesh as
arrays instead of writing a .vtp; `contour` is the plain array-level entry point.

The pad is applied on the device (a padded copy of the piece), never on the host.

`create_surface_piece` is the reference's 20-argument entry itself (surface_process.py:71-201,
called in spawned worker processes by SurfaceManager, surface.py:1360-1430): memmaps in, the
name of a VTK XML PolyData file (.vtp) out. The file is written without VTK (`write_vtp`: inline
base64 arrays, triangles as Polys), readable by vtkXMLPolyDataReader — what join_process_surface
(surface_process.py:229-268) does next — and by `read_vtp` here.

`join_process_surface` is the reference's second stage (surface_process.py:204-472, run in one more
worker by surface.py:1413 and :1514): it joins the piece files into one surface with its normals,
volume and area. `join_surface_device` is its body on device tensors, composed of the device surface
modules (surface_clean, surface_normals, mesh_ops, surface_connectivity, surface_holes).
"""
from __future__ import annotations

import base64
import os
import queue
import tempfile
import xml.etree.ElementTree as ET
from dataclasses import dataclass

import numpy as np
import torch

from . import device as dev
from .device import _mesh_tensors
from .mesh import marching_cubes
from .mesh_ops import smooth_device
from .surface_clean import clean_polydata_device
from .surface_connectivity import select_largest_part_device
from .surface_holes import fill_holes_device
from .surface_normals import compute_normals_device, mass_properties_device


def contour(volume: np.ndarray, isovalues, spacing=(1.0, 1.0, 1.0), z0: int = 0, flip_y: bool = True,
            padding=(0, 0, 0), index_dtype=np.int32):
    """Iso-surfaces of `volume` (uint8 or int16, [z][y][x]) at each value of `isovalues`.

    spacing = (sx, sy, sz); z0 = index of the first slice in the full volume; padding =
    (px, py, pz) voxels already added in front of the data (subtracted from the indices as
    in converters.to_vtk). Returns (vertices float32 [V,3], faces [T,3] of `index_dtype`);
    the surfaces of successive isovalues are concatenated in order. int32 faces (what
    `invesalius_rs.Mesh` takes as FaceArray::I32, types.rs:63-70) halve the device->host
    traffic; pass index_dtype=np.int64 for vtkIdType-sized indices."""
    if not isinstance(volume, np.ndarray) or volume.ndim != 3:
        raise TypeError("contour: 3-D numpy volume expected")
    if volume.dtype not in (np.uint8, np.int16):
        raise TypeError("contour: volume must be uint8 or int16")
    isovalues = [float(v) for v in np.atleast_1d(isovalues)]
    t = dev.to_device(volume)
    return _contour_device(t, isovalues, spacing, z0, flip_y, padding, index_dtype)


def _contour_device(t: torch.Tensor, isovalues, spacing, z0, flip_y, padding, index_dtype=np.int32):
    px, py, pz = padding
    tdt = torch.int64 if np.dtype(index_dtype) == np.int64 else torch.int32
    vs, fs, base = [], [], 0
    for iso in isovalues:
        v, f = marching_cubes(t, iso, spacing, (-px, -py, z0 - pz), flip_y)
        vs.append(v)
        f = f.to(tdt)
        fs.append(f + base if base else f)
        base += v.shape[0]
    verts = torch.cat(vs) if len(vs) > 1 else vs[0]
    faces = torch.cat(fs) if len(fs) > 1 else fs[0]
    return dev.to_numpy(verts), dev.to_numpy(faces)


def _pad_device(t: torch.Tensor, pad_value: int, pad_bottom: bool, pad_top: bool) -> torch.Tensor:
    """pad_image (surface_process.py:52-68) on the device."""
    dz, dy, dx = t.shape
    z_iadd = 1 if pad_bottom else 0
    out = torch.full((dz + z_iadd + (1 if pad_top else 0), dy + 2, dx + 2), pad_value, dtype=t.dtype,
                     device=t.device)
    out[z_iadd:z_iadd + dz, 1:-1, 1:-1] = t
    return out


def contour_piece(image: np.ndarray | None, mask_matrix: np.ndarray | None, roi: slice, spacing, min_value=None,
                  max_value=None, from_binary: bool = True, fill_border_holes: bool = True, flip_y: bool = True,
                  index_dtype=np.int32, nz_full: int | None = None):
    """The contour part of create_surface_piece for one Z piece.

    image: int16 [dz][dy][dx] (needed unless from_binary); mask_matrix: the padded uint8
    Mask memmap [dz+1][dy+1][dx+1] (needed when from_binary); roi: slice(z_start, z_stop)
    as built by SurfaceManager.AddNewActor (surface.py:1375-1381, stop may exceed dz)."""
    if from_binary:
        if mask_matrix is None:
            raise ValueError("from_binary needs mask_matrix")
        nz_full = mask_matrix.shape[0] - 1 if nz_full is None else nz_full
        piece = mask_matrix[roi.start + 1:roi.stop + 1, 1:, 1:]
        pad_value, isovalues = 0, [127.0]
    else:
        if image is None:
            raise ValueError("the Default algorithm needs the image")
        nz_full = image.shape[0] if nz_full is None else nz_full
        piece = image[roi]
        pad_value, isovalues = int(np.iinfo(image.dtype).min), [float(min_value), float(max_value)]
    if piece.shape[0] == 0:
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), index_dtype)
    pad_bottom = roi.start == 0
    pad_top = roi.stop >= nz_full
    t = dev.to_device(piece)
    if fill_border_holes:
        t = _pad_device(t, pad_value, pad_bottom, pad_top)
        padding = (1, 1, int(pad_bottom))
    else:
        padding = (0, 0, 0)
    return _contour_device(t, isovalues, spacing, roi.start, flip_y, padding, index_dtype)


# ------------------------------------------------------------------ .vtp (VTK XML PolyData) without VTK
_VTK_TYPES = {np.dtype(np.float32): "Float32", np.dtype(np.int32): "Int32", np.dtype(np.int64): "Int64"}


def _b64(a: np.ndarray) -> str:
    """VTK "binary" DataArray payload: base64(uint32 byte count + raw little-endian data), no compressor."""
    raw = np.ascontiguousarray(a).tobytes()
    return base64.b64encode(np.uint32(len(raw)).tobytes() + raw).decode("ascii")


def _normals_block(tag: str, normals, n: int) -> str:
    """<PointData> / <CellData> holding one Float32 [n,3] array named Normals, set as the active normals."""
    a = np.ascontiguousarray(normals, dtype=np.float32).reshape(-1, 3)
    if a.shape[0] != n:
        raise ValueError(f"write_vtp: {tag} normals must have one row per {'point' if tag == 'PointData' else 'cell'}")
    return (f'   <{tag} Normals="Normals">\n    <DataArray type="Float32" Name="Normals" NumberOfComponents="3" '
            f'format="binary">\n     {_b64(a)}\n    </DataArray>\n   </{tag}>\n')


def write_vtp(filename: str, vertices: np.ndarray, faces: np.ndarray, point_normals=None, cell_normals=None) -> None:
    """Triangle mesh -> VTK XML PolyData (what vtkXMLPolyDataWriter emits for the contour output,
    surface_process.py:188-192: Points + Polys). vertices float32 [V,3], faces int32/int64 [T,3].
    point_normals float32 [V,3] and cell_normals float32 [T,3], when given, are written as the active
    normals of the point data and the cell data (what the viewer shades the joined surface with); without
    them the file is Points + Polys alone."""
    v = np.ascontiguousarray(vertices, dtype=np.float32).reshape(-1, 3)
    f = np.ascontiguousarray(faces).reshape(-1, 3)
    if f.dtype not in (np.int32, np.int64):
        f = f.astype(np.int64)
    offs = (np.arange(1, f.shape[0] + 1, dtype=f.dtype) * 3)
    it = _VTK_TYPES[f.dtype]
    data = ""
    if point_normals is not None:
        data += _normals_block("PointData", point_normals, v.shape[0])
    if cell_normals is not None:
        data += _normals_block("CellData", cell_normals, f.shape[0])
    with open(filename, "w") as fh:
        fh.write('<?xml version="1.0"?>\n<VTKFile type="PolyData" version="0.1" byte_order="LittleEndian">\n <PolyData>\n')
        fh.write(f'  <Piece NumberOfPoints="{v.shape[0]}" NumberOfVerts="0" NumberOfLines="0" NumberOfStrips="0" '
                 f'NumberOfPolys="{f.shape[0]}">\n')
        fh.write(data)
        fh.write('   <Points>\n    <DataArray type="Float32" Name="Points" NumberOfComponents="3" format="binary">\n')
        fh.write("     " + _b64(v) + "\n    </DataArray>\n   </Points>\n   <Polys>\n")
        fh.write(f'    <DataArray type="{it}" Name="connectivity" format="binary">\n     ' + _b64(f.reshape(-1)) +
                 "\n    </DataArray>\n")
        fh.write(f'    <DataArray type="{it}" Name="offsets" format="binary">\n     ' + _b64(offs) + "\n    </DataArray>\n")
        fh.write("   </Polys>\n  </Piece>\n </PolyData>\n</VTKFile>\n")


def read_vtp(filename: str, normals: bool = False):
    """Inverse of write_vtp (inline base64, uncompressed, UInt32 headers): (vertices, faces); with
    normals=True also the active point and cell normals, float32 [N,3] or None when the file has none:
    (vertices, faces, point_normals, cell_normals)."""
    root = ET.parse(filename).getroot()
    piece = root.find("PolyData").find("Piece")

    def arr(node):
        dt = {v: k for k, v in _VTK_TYPES.items()}[node.get("type")]
        raw = base64.b64decode((node.text or "").strip())
        n = int(np.frombuffer(raw[:4], np.uint32)[0]) if len(raw) >= 4 else 0
        return np.frombuffer(raw[4:4 + n], dt).copy()

    def active_normals(tag):
        block = piece.find(tag)
        name = None if block is None else block.get("Normals")
        if name is None:
            return None
        return next(arr(d) for d in block.findall("DataArray") if d.get("Name") == name).reshape(-1, 3)

    pts = arr(piece.find("Points").find("DataArray")).reshape(-1, 3)
    polys = {d.get("Name"): arr(d) for d in piece.find("Polys").findall("DataArray")}
    conn = polys["connectivity"].reshape(-1, 3)
    assert int(piece.get("NumberOfPoints")) == pts.shape[0] and int(piece.get("NumberOfPolys")) == conn.shape[0]
    if not normals:
        return pts, conn
    return pts, conn, active_normals("PointData"), active_normals("CellData")


def create_surface_piece(filename, shape, dtype, mask_filename, mask_shape, mask_dtype, roi, spacing, mode, min_value,
                         max_value, decimate_reduction, smooth_relaxation_factor, smooth_iterations, language,
                         flip_image, from_binary, algorithm, imagedata_resolution, fill_border_holes):
    """invesalius/data/surface_process.py:71-201 with its own signature and result: the two memmaps in
    (image `filename`, padded mask `mask_filename`), the name of the written .vtp piece out. Runs in
    a spawned worker process like the reference's (surface.py:1368-1369): everything it needs is
    imported here, CUDA initialises on first use. The arguments the reference's body ignores as well
    (mode, decimate_reduction, smooth_*, language, flip_image, imagedata_resolution) are accepted and
    ignored. algorithm "InVesalius 3.b2" (vtkImageGaussianSmooth before the contour) is not built."""
    if not from_binary and algorithm == "InVesalius 3.b2":
        raise NotImplementedError("create_surface_piece: the 'InVesalius 3.b2' pre-smoothing is not built on the device")
    mask = np.memmap(mask_filename, mode="r", dtype=mask_dtype, shape=tuple(mask_shape))
    image = None if from_binary else np.memmap(filename, mode="r", dtype=dtype, shape=tuple(shape))
    # contour_piece derives pad_top from the array it is given; the reference uses `shape` (the image's)
    verts, faces = contour_piece(image, mask if from_binary else None, roi, spacing, min_value, max_value,
                                 from_binary=bool(from_binary), fill_border_holes=bool(fill_border_holes), flip_y=True,
                                 index_dtype=np.int64, nz_full=int(shape[0]))
    fd, out = tempfile.mkstemp(suffix="_%d_%d.vtp" % (roi.start, roi.stop))
    os.close(fd)
    write_vtp(out, verts, faces)
    return out


# ------------------------------------------------------------------ join_process_surface on the device
@dataclass
class JoinedSurface:
    """The joined surface, on the pieces' device. points float32 [N,3], faces int64 [T,3] (vtkIdType's
    width), point_normals float32 [N,3] and cell_normals float32 [T,3]: the mesh as the final normals leave
    it. volume and area: vtkMassProperties of the mesh before those normals (the reference's
    `to_measure`). dropped_cells: the verts and lines the cleans made of degenerate triangles, which the
    join drops."""
    points: torch.Tensor
    faces: torch.Tensor
    point_normals: torch.Tensor
    cell_normals: torch.Tensor
    volume: float
    area: float
    dropped_cells: int


def _append(pieces):
    """vtkAppendPolyData: points concatenated in list order, each piece's faces offset by the points before
    it, pieces without points skipped."""
    vs, fs, base = [], [], 0
    for v, f in pieces:
        if _mesh_tensors(v, f, "join_surface_device") != 3 or not v.is_cuda:
            raise ValueError("join_surface_device: pieces of CUDA vertices [V,3] and faces [T,3] expected")
        if v.shape[0] == 0:
            continue
        vs.append(v)
        fs.append(f.to(torch.int64) + base)
        base += v.shape[0]
    if not vs:
        return None, None
    return torch.cat(vs), torch.cat(fs)


def _ncells(pair) -> int:
    return pair[0].numel() - 1


def _clean(points, faces):
    """vtkCleanPolyData (PointMergingOn, tolerance 0) keeping only the triangles: (points, faces, cell_ids of
    the triangles, verts and lines dropped)."""
    c = clean_polydata_device(points, faces)
    skip = _ncells(c.verts) + _ncells(c.lines)
    return c.points, c.polys, c.cell_ids[skip:], skip


def join_surface_device(pieces, algorithm, keep_largest, fill_holes, options, progress=None) -> JoinedSurface:
    """The body of join_process_surface (invesalius/data/surface_process.py:228-461) on device tensors.

    pieces: a list of (vertices float32 [V,3], faces int32 / int64 [T,3]) CUDA tensors in append order,
    for example the files of create_surface_piece or one whole-volume mesh.marching_cubes result. The
    point numbering of the result depends on that order; the reference appends its pieces in the order its
    pool callbacks arrive. The inputs are not modified. The steps, in the reference's order:

      append          vtkAppendPolyData (torch.cat)
      clean           surface_clean.clean_polydata_device, merging the points of the seams
      ca_smoothing    algorithm "ca_smoothing" only: normals at VTK's defaults (30 degrees, no
                      auto-orientation), a second clean with the cell normals carried through its cell_ids,
                      and mesh_ops.smooth_device with options["angle"], ["max distance"], ["min weight"] and
                      ["steps"] (a missing key raises KeyError). The smoothed points are the points from
                      then on, as the reference's Mesh writes through its views of the VTK points.
      largest part    keep_largest: surface_connectivity.select_largest_part_device in VTK's form (every
                      point the traversal numbered, in PointMap order)
      fill holes      fill_holes: surface_holes.fill_holes_device with hole size 300
      volume, area    surface_normals.mass_properties_device
      final normals   surface_normals.compute_normals_device at 80 degrees with auto-orientation

    Where a triangle's corners coincide exactly (a Default surface contoured at a value the int16 image
    takes), the clean turns it into a line or a vert. The join keeps only the triangles and counts the
    others in dropped_cells: no later step takes lines, and they add nothing to the volume or area. Mask
    surfaces (iso 127, which no mask value equals) have none. A surface without triangles after the first
    clean is empty: empty tensors, volume and area 0.0, and no filter runs on it.

    progress, if given, is called with the reference's messages from "Cleaning surface ..." on, under the
    same conditions and in the same order; join_process_surface sends "Joining surfaces ..." before it
    reads the pieces. Synchronises after every step: each module brings its counts to the host."""
    say = progress if progress is not None else (lambda msg: None)
    points, faces = _append(pieces)
    dropped = 0
    say("Cleaning surface ...")
    if points is not None:
        points, faces, _, dropped = _clean(points, faces)
        if faces.shape[0] == 0:
            points = None
    if algorithm == "ca_smoothing":
        say("Calculating normals ...")
        if points is not None:
            n = compute_normals_device(points, faces, 30.0, False)
            points, faces, cell_ids, more = _clean(n.points, n.faces)
            dropped += more
            cell_normals = n.cell_normals[cell_ids].contiguous()
        say("Context Aware smoothing ...")
        T, tmax, bmin, steps = (options[k] for k in ("angle", "max distance", "min weight", "steps"))
        if points is not None:
            faces4 = torch.cat((torch.full((faces.shape[0], 1), 3, dtype=torch.int64, device=faces.device), faces), 1)
            smooth_device(points, faces4, cell_normals, T, tmax, bmin, steps)
    if keep_largest:
        say("Finding the largest ...")
        if points is not None:
            points, faces, _, _ = select_largest_part_device(points, faces)
    if fill_holes:
        say("Filling holes ...")
        if points is not None:
            faces = fill_holes_device(points, faces, 300.0).faces
    if points is None:
        say("Calculating area and volume ...")
        d = pieces[0][0].device if pieces else torch.device("cuda", torch.cuda.current_device())
        z = torch.zeros((0, 3), dtype=torch.float32, device=d)
        return JoinedSurface(z, torch.zeros((0, 3), dtype=torch.int64, device=d), z.clone(), z.clone(), 0.0, 0.0,
                             dropped)
    volume, area = mass_properties_device(points, faces)
    n = compute_normals_device(points, faces, 80.0, True)
    say("Calculating area and volume ...")
    return JoinedSurface(n.points, n.faces, n.point_normals, n.cell_normals, float(volume), float(area), dropped)


def join_process_surface(filenames, algorithm, smooth_iterations, smooth_relaxation_factor, decimate_reduction,
                         keep_largest, fill_holes, options, msg_queue):
    """invesalius/data/surface_process.py:204-472 with its own signature and result: the piece files of
    create_surface_piece in, (the name of the joined .vtp, {"volume": float, "area": float}) out. Runs in
    a spawned worker process like the reference's (surface.py:1413, :1514); CUDA initialises on first use.
    The pieces are joined in the order of `filenames` by join_surface_device, and the file holds the points,
    the triangles and both normals arrays. Progress messages go through msg_queue.put_nowait; a full queue
    is printed and ignored. smooth_iterations and smooth_relaxation_factor are accepted and ignored, as the
    reference's smoother is commented out. A falsy decimate_reduction (the reference's vtkQuadricDecimation
    branch, which no quality preset reaches) raises NotImplementedError before any work."""
    if not decimate_reduction:
        raise NotImplementedError("join_process_surface: vtkQuadricDecimation (decimate_reduction falsy) is not built "
                                  "on the device")

    def send_message(msg):
        try:
            msg_queue.put_nowait(msg)
        except queue.Full as e:
            print(e)

    dev.require_cuda()
    send_message("Joining surfaces ...")
    pieces = []
    for fn in filenames:
        v, f = read_vtp(fn)
        pieces.append((torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()))
    r = join_surface_device(pieces, algorithm, keep_largest, fill_holes, options, send_message)
    fd, out = tempfile.mkstemp(suffix="_full.vtp")
    os.close(fd)
    write_vtp(out, *(t.cpu().numpy() for t in (r.points, r.faces, r.point_normals, r.cell_normals)))
    return out, {"volume": r.volume, "area": r.area}
