"""The surface join on the device (surface_process.join_surface_device and join_process_surface) against its
sequential checker (oracle/join.py), bit for bit: points, faces, both normals, the bits of the volume and the
area, and the dropped verts and lines. Also the seams, the reference's entry in a spawned pool with its
messages, and the edge cases."""
import os
import queue

import numpy as np
import pytest

from join_cases import CA_OPTIONS, SPACING, noise_case, padded_mask, rois, triangle_rows

pytestmark = pytest.mark.gpu

ALGORITHMS = ["Default", "Binary", "ca_smoothing"]


@pytest.fixture(scope="module")
def sp():
    from invesalius3_b200 import device, surface_process
    device.require_cuda()
    return surface_process


def _on_device(pieces):
    import torch
    return [(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()) for v, f in pieces]


def device_pieces(sp, algorithm, mm, img, lo=226, hi=3071, fill_border_holes=True, index_dtype=np.int32,
                  spacing=SPACING):
    """create_surface_piece's meshes (contour_piece) over AddNewActor's pieces, as numpy arrays"""
    binary = algorithm != "Default"
    dz = (mm.shape[0] - 1) if binary else img.shape[0]
    return [sp.contour_piece(img, mm, roi, spacing, lo, hi, from_binary=binary, fill_border_holes=fill_border_holes,
                             index_dtype=index_dtype, nz_full=dz) for roi in rois(dz)]


def check_join(sp, pieces, algorithm, keep_largest, fill_holes, options=CA_OPTIONS):
    import torch
    from oracle import join as oj
    got = sp.join_surface_device(_on_device(pieces), algorithm, keep_largest, fill_holes, options)
    want = oj.join(pieces, algorithm, keep_largest, fill_holes, options)
    assert got.faces.dtype == torch.int64
    assert np.array_equal(got.faces.cpu().numpy(), want["faces"])
    for k in ("points", "point_normals", "cell_normals"):
        g = getattr(got, k).cpu().numpy()
        assert g.dtype == np.float32 and np.array_equal(g.view(np.uint32), want[k].view(np.uint32)), k
    assert np.float64(got.volume).view(np.uint64) == np.float64(want["volume"]).view(np.uint64)
    assert np.float64(got.area).view(np.uint64) == np.float64(want["area"]).view(np.uint64)
    assert got.dropped_cells == want["dropped_cells"]
    if algorithm != "Default":
        assert got.dropped_cells == 0          # iso 127: no mask value lies on it
    return got


@pytest.mark.parametrize("algorithm", ALGORITHMS)
@pytest.mark.parametrize("keep_largest", [False, True])
@pytest.mark.parametrize("fill_holes", [False, True])
@pytest.mark.parametrize("seed,fill_border_holes", [(1, True), (2, False)])
def test_noise(sp, algorithm, keep_largest, fill_holes, seed, fill_border_holes):
    mm, img = noise_case(seed)
    pieces = device_pieces(sp, algorithm, mm, img, fill_border_holes=fill_border_holes,
                           index_dtype=np.int64 if seed == 2 else np.int32)
    assert len(pieces) == 3
    got = check_join(sp, pieces, algorithm, keep_largest, fill_holes)
    assert got.faces.shape[0] > 10_000


@pytest.mark.parametrize("thr", ["thr_0", "thr_1"])
@pytest.mark.parametrize("keep_largest", [False, True])
@pytest.mark.parametrize("fill_holes", [False, True])
def test_cranium_crop_default(sp, cranium, thr, keep_largest, fill_holes):
    lo, hi = (int(x) for x in cranium[thr])
    img = np.ascontiguousarray(cranium["matrix_crop"])
    pieces = device_pieces(sp, "Default", None, img, lo, hi, spacing=tuple(float(s) for s in cranium["spacing"]))
    got = check_join(sp, pieces, "Default", keep_largest, fill_holes)
    assert got.dropped_cells > 0


def _cranium_mask(cranium, i):
    full = tuple(int(s) for s in cranium["full_shape"])
    return padded_mask(np.unpackbits(cranium[f"mask_{i}_bits_full"])[:np.prod(full)].reshape(full) * np.uint8(255))


@pytest.mark.parametrize("i", [0, 1])
@pytest.mark.parametrize("algorithm", ["Binary", "ca_smoothing"])
@pytest.mark.parametrize("keep_largest", [False, True])
@pytest.mark.parametrize("fill_holes", [False, True])
def test_cranium_full_size(sp, cranium, i, algorithm, keep_largest, fill_holes):
    mm = _cranium_mask(cranium, i)
    # mask 0 without the border padding: its surface is open where the skull meets the volume's border
    pieces = device_pieces(sp, algorithm, mm, None, spacing=tuple(float(s) for s in cranium["spacing"]),
                           fill_border_holes=bool(i))
    assert mm.shape[0] - 1 == 108 and len(pieces) == 6
    check_join(sp, pieces, algorithm, keep_largest, fill_holes)


@pytest.mark.parametrize("algorithm,keep_largest,fill_holes", [("Binary", True, True), ("ca_smoothing", False, False)])
def test_phantom_512_in_pieces(sp, algorithm, keep_largest, fill_holes):
    import torch
    from invesalius3_b200 import device as dev, phantom
    vol = phantom.ct((512, 512, 512), seed=2)
    mm = padded_mask(dev.threshold(torch.from_numpy(vol).cuda(), 226, 3071).cpu().numpy())
    del vol
    pieces = device_pieces(sp, algorithm, mm, None, spacing=(1.0, 1.0, 1.0))
    del mm
    assert len(pieces) == 26
    got = check_join(sp, pieces, algorithm, keep_largest, fill_holes)
    assert got.faces.shape[0] > 10 ** 6


# ---- seams ------------------------------------------------------------------------------------------------
def _seam_check(sp, mm, spacing, fill_border_holes):
    import torch
    from invesalius3_b200 import surface_clean as sc
    dz = mm.shape[0] - 1
    pieces = device_pieces(sp, "Binary", mm, None, spacing=spacing, fill_border_holes=fill_border_holes)
    v = torch.cat([torch.from_numpy(p[0]) for p in pieces]).cuda()
    base = np.cumsum([0] + [len(p[0]) for p in pieces])
    f = torch.cat([torch.from_numpy(p[1].astype(np.int64) + b) for p, b in zip(pieces, base)]).cuda()
    a = sc.clean_polydata_device(v, f)
    V, F = sp.contour_piece(None, mm, slice(0, dz), spacing, from_binary=True, fill_border_holes=fill_border_holes)
    b = sc.clean_polydata_device(torch.from_numpy(V).cuda(), torch.from_numpy(F).cuda())
    assert a.points.shape[0] == b.points.shape[0] < v.shape[0]
    ra = triangle_rows(a.points.cpu().numpy(), a.polys.cpu().numpy())
    rb = triangle_rows(b.points.cpu().numpy(), b.polys.cpu().numpy())
    assert len(ra) > 1000 and np.array_equal(ra, rb)
    joined = sp.join_surface_device(_on_device(pieces), "Binary", False, False, {})
    assert joined.faces.shape[0] == len(ra)


@pytest.mark.parametrize("seed,fill_border_holes", [(1, True), (2, False)])
def test_seams_noise(sp, seed, fill_border_holes):
    _seam_check(sp, noise_case(seed)[0], SPACING, fill_border_holes)


@pytest.mark.parametrize("i", [0, 1])
def test_seams_cranium(sp, cranium, i):
    _seam_check(sp, _cranium_mask(cranium, i), tuple(float(s) for s in cranium["spacing"]), True)


# ---- the reference's entry ----------------------------------------------------------------------------------
def _piece_worker(args):
    from invesalius3_b200 import surface_process
    return surface_process.create_surface_piece(*args)


def _join_worker(args):
    from invesalius3_b200 import surface_process
    return surface_process.join_process_surface(*args)


def _write_inputs(tmp_path, mm, img):
    img_fn, mask_fn = str(tmp_path / "matrix.dat"), str(tmp_path / "mask.dat")
    np.memmap(img_fn, mode="w+", dtype=np.int16, shape=img.shape)[:] = img
    m = np.memmap(mask_fn, mode="w+", dtype=np.uint8, shape=mm.shape)
    m[:] = mm
    m.flush()
    return img_fn, mask_fn


def _piece_jobs(img_fn, mask_fn, img, mm, algorithm):
    return [(img_fn, img.shape, "int16", mask_fn, mm.shape, "uint8", roi, SPACING, "CONTOUR", 226, 3071, 0.4, 0.0, 0,
             "en", False, algorithm != "Default", algorithm, 0, True) for roi in rois(img.shape[0])]


def _pieces_of(sp, names):
    return [sp.read_vtp(fn) for fn in names]


@pytest.mark.parametrize("algorithm", ALGORITHMS)
def test_join_process_surface_in_spawned_pool(sp, tmp_path, algorithm):
    """The two stages of AddNewActor, each in spawned workers: create_surface_piece per piece, then
    join_process_surface with a one-message Manager queue. The file and measures equal join_surface_device."""
    import multiprocessing as mp
    mm, img = noise_case(3)
    img_fn, mask_fn = _write_inputs(tmp_path, mm, img)
    ctx = mp.get_context("spawn")
    with ctx.Pool(2) as pool, ctx.Manager() as manager:
        names = pool.map(_piece_worker, _piece_jobs(img_fn, mask_fn, img, mm, algorithm))
        q = manager.Queue(1)
        out, measures = pool.apply(_join_worker, ((names, algorithm, 2, 0.3, 0.4, True, True, CA_OPTIONS, q),))
        assert q.get_nowait() == "Joining surfaces ..."
    try:
        assert out.endswith("_full.vtp") and set(measures) == {"volume", "area"}
        v, f, pn, cn = sp.read_vtp(out, normals=True)
        want = sp.join_surface_device(_on_device(_pieces_of(sp, names)), algorithm, True, True, CA_OPTIONS)
        assert np.array_equal(v, want.points.cpu().numpy()) and np.array_equal(f, want.faces.cpu().numpy())
        assert np.array_equal(pn, want.point_normals.cpu().numpy())
        assert np.array_equal(cn, want.cell_normals.cpu().numpy())
        assert measures == {"volume": want.volume, "area": want.area}
        assert type(measures["volume"]) is float and measures["volume"] > 0
    finally:
        for fn in names + [out]:
            os.unlink(fn)


def _expected_messages(algorithm, keep_largest, fill_holes):
    m = ["Joining surfaces ...", "Cleaning surface ..."]
    if algorithm == "ca_smoothing":
        m += ["Calculating normals ...", "Context Aware smoothing ..."]
    if keep_largest:
        m.append("Finding the largest ...")
    if fill_holes:
        m.append("Filling holes ...")
    return m + ["Calculating area and volume ..."]


@pytest.fixture(scope="module")
def piece_files(sp, tmp_path_factory):
    mm, img = noise_case(4, (45, 24, 28))
    d = tmp_path_factory.mktemp("pieces")
    files = {}
    for algorithm in ALGORITHMS:
        files[algorithm] = []
        for k, (v, f) in enumerate(device_pieces(sp, algorithm, mm, img, index_dtype=np.int64)):
            fn = str(d / f"{algorithm}_{k}.vtp")
            sp.write_vtp(fn, v, f)
            files[algorithm].append(fn)
    return files


def _run(sp, names, algorithm, keep_largest, fill_holes, options=CA_OPTIONS, q=None, decimate=0.4):
    out, measures = sp.join_process_surface(names, algorithm, 2, 0.3, decimate, keep_largest, fill_holes, options,
                                            q if q is not None else queue.Queue())
    r = sp.read_vtp(out, normals=True)
    os.unlink(out)
    return r, measures


@pytest.mark.parametrize("algorithm", ALGORITHMS)
@pytest.mark.parametrize("keep_largest", [False, True])
@pytest.mark.parametrize("fill_holes", [False, True])
def test_messages(sp, piece_files, algorithm, keep_largest, fill_holes):
    q = queue.Queue()
    _run(sp, piece_files[algorithm], algorithm, keep_largest, fill_holes, q=q)
    got = []
    while not q.empty():
        got.append(q.get_nowait())
    assert got == _expected_messages(algorithm, keep_largest, fill_holes)


def test_full_queue_is_printed_and_ignored(sp, piece_files, capsys):
    q = queue.Queue(1)
    _run(sp, piece_files["Binary"], "Binary", True, True, q=q)
    assert q.get_nowait() == "Joining surfaces ..." and q.empty()
    assert capsys.readouterr().out.count("\n") >= 4


# ---- edge cases --------------------------------------------------------------------------------------------
def test_empty_mask(sp, tmp_path):
    mm = padded_mask(np.zeros((45, 16, 16), np.uint8))
    names = []
    for k, (v, f) in enumerate(device_pieces(sp, "Binary", mm, None, index_dtype=np.int64)):
        names.append(str(tmp_path / f"{k}.vtp"))
        sp.write_vtp(names[-1], v, f)
    for algorithm in ("Binary", "ca_smoothing"):
        (v, f, pn, cn), measures = _run(sp, names, algorithm, True, True)
        assert v.shape == f.shape == pn.shape == cn.shape == (0, 3)
        assert measures == {"volume": 0.0, "area": 0.0}
    r = sp.join_surface_device([], "Binary", True, True, {})
    assert r.points.shape == r.faces.shape == (0, 3) and (r.volume, r.area, r.dropped_cells) == (0.0, 0.0, 0)


def test_refusals(sp, piece_files):
    q = queue.Queue()
    for d in (0, 0.0, None):
        with pytest.raises(NotImplementedError, match="vtkQuadricDecimation"):
            sp.join_process_surface(piece_files["Binary"], "Binary", 0, 0, d, True, True, {}, q)
    assert q.empty()
    for missing in CA_OPTIONS:
        opts = {k: v for k, v in CA_OPTIONS.items() if k != missing}
        with pytest.raises(KeyError):
            _run(sp, piece_files["ca_smoothing"], "ca_smoothing", False, False, options=opts)
    _run(sp, piece_files["Binary"], "Binary", False, False, options={})     # the other algorithms read no option


def test_empty_piece_skipped_and_one_piece(sp):
    import torch
    mm, img = noise_case(8)
    pieces = device_pieces(sp, "ca_smoothing", mm, img)
    empty = (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
    a = sp.join_surface_device(_on_device(pieces), "ca_smoothing", True, True, CA_OPTIONS)
    b = sp.join_surface_device(_on_device([empty] + pieces[:2] + [empty] + pieces[2:]), "ca_smoothing", True, True,
                               CA_OPTIONS)
    for k in ("points", "faces", "point_normals", "cell_normals"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k
    assert (a.volume, a.area) == (b.volume, b.area)
    # one whole-volume piece, as mesh.marching_cubes gives it
    whole = sp.contour_piece(None, mm, slice(0, 45), SPACING, from_binary=True)
    for algorithm in ("Binary", "ca_smoothing"):
        check_join(sp, [whole], algorithm, True, True)


def test_inputs_not_modified(sp):
    import torch
    mm, img = noise_case(9)
    for algorithm in ALGORITHMS:
        pieces = _on_device(device_pieces(sp, algorithm, mm, img))
        before = [(v.clone(), f.clone()) for v, f in pieces]
        sp.join_surface_device(pieces, algorithm, True, True, CA_OPTIONS)
        assert all(torch.equal(v, v0) and torch.equal(f, f0) for (v, f), (v0, f0) in zip(pieces, before))
