"""Host side of the surface join: the .vtp writer and reader with normals, and the join's checker
(oracle/join.py) against the checkers it is composed of, step by step. No GPU needed."""
import hashlib

import numpy as np
import pytest

from join_cases import CA_OPTIONS, SPACING, host_pieces, noise_case, triangle_rows

V4 = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1.5]], np.float32)
F2 = np.array([[0, 1, 2], [0, 3, 1]], np.int64)

# what write_vtp wrote before it took normals, for V4 / F2
PLAIN_INT64 = """<?xml version="1.0"?>
<VTKFile type="PolyData" version="0.1" byte_order="LittleEndian">
 <PolyData>
  <Piece NumberOfPoints="4" NumberOfVerts="0" NumberOfLines="0" NumberOfStrips="0" NumberOfPolys="2">
   <Points>
    <DataArray type="Float32" Name="Points" NumberOfComponents="3" format="binary">
     MAAAAAAAAAAAAAAAAAAAAAAAgD8AAAAAAAAAAAAAAAAAAIA/AAAAAAAAAAAAAAAAAADAPw==
    </DataArray>
   </Points>
   <Polys>
    <DataArray type="Int64" Name="connectivity" format="binary">
     MAAAAAAAAAAAAAAAAQAAAAAAAAACAAAAAAAAAAAAAAAAAAAAAwAAAAAAAAABAAAAAAAAAA==
    </DataArray>
    <DataArray type="Int64" Name="offsets" format="binary">
     EAAAAAMAAAAAAAAABgAAAAAAAAA=
    </DataArray>
   </Polys>
  </Piece>
 </PolyData>
</VTKFile>
"""
PLAIN_INT32_SHA256 = "6cf2c0360d8efba41943138e89a0178731ab094e0789cae8855552c1993d7763"


@pytest.fixture(scope="module")
def sp():
    from invesalius3_b200 import surface_process
    return surface_process


def test_writer_bytes_without_normals(sp, tmp_path):
    fn = str(tmp_path / "a.vtp")
    sp.write_vtp(fn, V4, F2)
    assert open(fn, "rb").read() == PLAIN_INT64.encode()
    sp.write_vtp(fn, V4, F2.astype(np.int32))
    assert hashlib.sha256(open(fn, "rb").read()).hexdigest() == PLAIN_INT32_SHA256


@pytest.mark.parametrize("dtype", [np.int32, np.int64])
def test_round_trip_with_normals(sp, tmp_path, dtype):
    rng = np.random.default_rng(3)
    v = rng.normal(size=(50, 3)).astype(np.float32)
    f = rng.integers(0, 50, (70, 3)).astype(dtype)
    pn, cn = rng.normal(size=(50, 3)).astype(np.float32), rng.normal(size=(70, 3)).astype(np.float32)
    fn = str(tmp_path / "n.vtp")
    for point_normals, cell_normals in ((pn, cn), (pn, None), (None, cn), (None, None)):
        sp.write_vtp(fn, v, f, point_normals, cell_normals)
        gv, gf, gpn, gcn = sp.read_vtp(fn, normals=True)
        assert gv.dtype == np.float32 and np.array_equal(gv, v)
        assert gf.dtype == dtype and np.array_equal(gf, f)
        for got, want in ((gpn, point_normals), (gcn, cell_normals)):
            assert (got is None) if want is None else (got.dtype == np.float32 and np.array_equal(got, want))
        gv2, gf2 = sp.read_vtp(fn)
        assert np.array_equal(gv2, v) and np.array_equal(gf2, f)
    with pytest.raises(ValueError):
        sp.write_vtp(fn, v, f, pn[:-1])


def test_round_trip_no_points(sp, tmp_path):
    fn = str(tmp_path / "e.vtp")
    z = np.zeros((0, 3), np.float32)
    for normals in ((None, None), (z, z)):
        sp.write_vtp(fn, z, np.zeros((0, 3), np.int64), *normals)
        v, f, pn, cn = sp.read_vtp(fn, normals=True)
        assert v.shape == (0, 3) and f.shape == (0, 3) and f.dtype == np.int64
        assert (pn is None) == (normals[0] is None) and (pn is None or pn.shape == (0, 3))
        assert (cn is None) == (normals[1] is None) and (cn is None or cn.shape == (0, 3))


def _by_hand(orc, pieces, algorithm, keep_largest, fill_holes, options):
    """The join written out step by step with the checkers."""
    from oracle import clean as oc, connectivity as ocn, fill_holes as ofh, normals as on
    base = np.cumsum([0] + [len(v) for v, _ in pieces])
    pts = np.concatenate([v for v, _ in pieces])
    faces = np.concatenate([f.astype(np.int64) + b for (_, f), b in zip(pieces, base)])
    c = oc.clean_polydata(pts, faces)
    nvl = len(c["verts"][1]) + len(c["lines"][1]) // 2
    pts, faces = c["points"], c["polys"][1].reshape(-1, 3)
    if algorithm == "ca_smoothing":
        n = on.compute_normals(pts, faces, 30.0, False)
        c = oc.clean_polydata(n["points"], n["faces"])
        assert len(c["verts"][1]) == len(c["lines"][1]) == 0
        pts, faces = c["points"].copy(), c["polys"][1].reshape(-1, 3)
        F4 = np.concatenate([np.full((len(faces), 1), 3, np.int64), faces], 1)
        orc.ca_smoothing(pts, F4, np.ascontiguousarray(n["cell_normals"][c["cell_ids"]]), options["angle"],
                         options["max distance"], options["min weight"], options["steps"])
    if keep_largest:
        pts, faces, _, _ = ocn.select_largest_part(pts, faces)
    if fill_holes:
        faces = ofh.fill_holes(pts, faces, 300)["faces"]
    volume, area = on.mass_properties(pts, faces)
    n = on.compute_normals(pts, faces, 80, True)
    return n, volume, area, nvl


@pytest.mark.parametrize("algorithm", ["Default", "Binary", "ca_smoothing"])
@pytest.mark.parametrize("keep_largest", [False, True])
@pytest.mark.parametrize("fill_holes", [False, True])
def test_checker_is_the_composed_checkers(orc, algorithm, keep_largest, fill_holes):
    from oracle import join as oj
    mm, img = noise_case(5, (45, 20, 24))
    if algorithm == "Default":
        pieces = host_pieces(orc, img, [226.0, 3071.0], fill_border_holes=False)
    else:
        pieces = host_pieces(orc, mm[1:, 1:, 1:], [127.0], fill_border_holes=False)
    assert len(pieces) == 3
    got = oj.join(pieces, algorithm, keep_largest, fill_holes, CA_OPTIONS)
    n, volume, area, dropped = _by_hand(orc, pieces, algorithm, keep_largest, fill_holes, CA_OPTIONS)
    for k in ("points", "faces", "point_normals", "cell_normals"):
        assert got[k].dtype == n[k].dtype and np.array_equal(got[k], n[k]), k
    assert got["faces"].dtype == np.int64
    assert (got["volume"], got["area"], got["dropped_cells"]) == (volume, area, dropped)
    assert (dropped > 0) == (algorithm == "Default")


def test_checker_edges(orc):
    from oracle import join as oj
    empty = (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64))
    r = oj.join([empty, empty], "ca_smoothing", True, True, CA_OPTIONS)
    assert r["points"].shape == r["faces"].shape == (0, 3) and (r["volume"], r["area"]) == (0.0, 0.0)
    mm, _ = noise_case(6, (30, 16, 16))
    pieces = host_pieces(orc, mm[1:, 1:, 1:], [127.0])
    a = oj.join(pieces, "Binary", True, True, {})
    b = oj.join(pieces[:1] + [empty] + pieces[1:], "Binary", True, True, {})
    assert all(np.array_equal(a[k], b[k]) for k in ("points", "faces", "point_normals", "cell_normals"))
    with pytest.raises(KeyError):
        oj.join(pieces, "ca_smoothing", False, False, {"angle": 0.7, "max distance": 3.0, "min weight": 0.5})


@pytest.mark.parametrize("fill_border_holes", [True, False])
def test_seams_merge_to_the_whole_contour(orc, fill_border_holes):
    """The appended pieces, cleaned, hold the triangles of the whole volume's contour, cleaned."""
    from oracle import clean as oc, join as oj
    mm, _ = noise_case(7)
    body = mm[1:, 1:, 1:]
    pts, faces = oj.append(host_pieces(orc, body, [127.0], fill_border_holes=fill_border_holes))
    whole = body
    origin = (0, 0, 0)
    if fill_border_holes:
        whole = np.zeros(tuple(s + 2 for s in body.shape), np.uint8)
        whole[1:-1, 1:-1, 1:-1] = body
        origin = (-1, -1, -1)
    V, F = orc.marching_cubes(whole, 127.0, SPACING, origin, True)
    a, b = oc.clean_polydata(pts, faces), oc.clean_polydata(V, F)
    assert len(a["points"]) == len(b["points"]) < len(pts)
    assert np.array_equal(triangle_rows(a["points"], a["polys"][1]), triangle_rows(b["points"], b["polys"][1]))
