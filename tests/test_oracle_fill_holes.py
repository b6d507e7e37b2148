"""The hole filler's C checker (oracle/fill_holes.c) against an independent plain-Python restatement
(fill_holes_meshes.fill_holes_py) and closed forms."""
import numpy as np
import pytest

import fill_holes_meshes as fm
from connectivity_meshes import dense_random, shuffled_spheres
from oracle import fill_holes as ofh
from smoothing_meshes import fin, grid_patch, with_degenerate, with_unused
from visibility_meshes import icosphere


def _agree(v, f, hole_size=1.0):
    got = ofh.fill_holes(v, f, hole_size)
    faces, lines, loops = fm.fill_holes_py(v, f, hole_size)
    assert np.array_equal(got["faces"], faces)
    assert got["lines"] == lines
    assert len(got["npts"]) == len(loops)
    for k, (first, npts, r, status) in enumerate(loops):
        assert got["first_line"][k] == first and got["npts"][k] == npts and got["status"][k] == status
        assert got["radius"][k].view(np.uint64) == np.float64(r).view(np.uint64)
    return got


MESHES = {
    "icosphere_minus_one": fm.icosphere_minus_one,
    "cube_minus_quad": fm.cube_minus_quad,
    "grid": lambda: grid_patch(12, 9, 1),
    "deleted_icosphere": lambda: fm.random_deletion(*icosphere(1.0, 3), 0.3, 1),
    "deleted_spheres": lambda: fm.random_deletion(*shuffled_spheres(5, 2), 0.4, 2),
    "dense": lambda: dense_random(300, 80, 3),
    "fin": fin,
    "degenerate": lambda: with_degenerate(*grid_patch(8, 7, 2), seed=5),
    "unused": lambda: with_unused(*fm.icosphere_minus_one(), seed=3),
    "bowtie": fm.bowtie,
    "collinear": fm.collinear_loop,
    "tube": lambda: fm.open_tube(40),
}


@pytest.mark.parametrize("name", list(MESHES))
@pytest.mark.parametrize("hole_size", [0.05, 1.0, 300.0])
def test_checker_equals_restatement(name, hole_size):
    _agree(*MESHES[name](), hole_size)


def test_icosphere_minus_one_face_gets_one_triangle():
    v, f = fm.icosphere_minus_one()
    got = _agree(v, f)
    assert len(got["faces"]) == len(f) + 1 and list(got["status"]) == [ofh.FILLED]
    gone = set(icosphere(1.0, 2)[1][len(icosphere(1.0, 2)[1]) // 3].tolist())
    assert set(got["faces"][-1].tolist()) == gone


def test_cube_minus_quad_gets_two_triangles():
    v, f = fm.cube_minus_quad()
    got = _agree(v, f, 5.0)
    assert len(got["faces"]) == len(f) + 2 and got["lines"] == 4 and list(got["npts"]) == [4]
    assert set(got["faces"][-2:].reshape(-1).tolist()) == {0, 1, 2, 3}


def test_open_grid_radius_and_threshold():
    v, f = grid_patch(10, 7, 0, jitter=0.0)
    got = _agree(v, f, 100.0)
    assert list(got["npts"]) == [2 * (9 + 6)] and got["lines"] == 30
    r = got["radius"][0]
    assert np.hypot(9, 6) / 2 <= r <= np.hypot(9, 6)            # the sphere holds the loop's two far corners
    assert _agree(v, f, r)["status"][0] == ofh.FILLED
    assert _agree(v, f, np.nextafter(r, 0))["status"][0] == ofh.TOO_LARGE
    assert len(_agree(v, f, np.nextafter(r, 0))["faces"]) == len(f)


def test_closed_surface_and_too_few_lines():
    v, f = icosphere(1.0, 2)
    got = _agree(v, f)
    assert got["lines"] == 0 and np.array_equal(got["faces"], f) and len(got["npts"]) == 0
    v, f = fm.closed_plus_sliver()
    got = _agree(v, f, 1e30)
    assert got["lines"] == 2 and np.array_equal(got["faces"], f) and len(got["npts"]) == 0


def _line_id(v, f, line):
    lines = [(int(t[i]), int(t[(i + 1) % 3])) for c, t in enumerate(f) for i in range(3)
             if not any(d != c and t[(i + 1) % 3] in f[d] for d in np.nonzero((f == t[i]).any(1))[0])]
    return lines.index(line)


def test_two_holes_sharing_a_point_depend_on_the_line_ids():
    """Point 12 has four lines. The first hole's chain from 12 runs 12 -> 7 (forward), (6, 7) (backward,
    the flipped neighbour), 6 -> 12 (forward); it is traced from 12 only when line (12, 7) comes before
    line (6, 7). The second hole's lines all run forward from 12, so it is always filled."""
    n = len(fm.bowtie()[1])
    outcomes = set()
    for seed in range(16):
        v, f = fm.bowtie(np.random.default_rng(seed).permutation(n))
        got = _agree(v, f, 2.0)
        new = {tuple(sorted(t)) for t in got["faces"][n:].tolist()}
        first = (6, 7, 12) in new
        assert first == (_line_id(v, f, (12, 7)) < _line_id(v, f, (6, 7)))
        assert (12, 17, 18) in new
        outcomes.add(first)
    assert outcomes == {True, False}


def test_degenerate_pieces_and_failures():
    got = _agree(*fm.collinear_loop(), 5.0)
    assert list(got["status"]) == [ofh.FAILED] and len(got["faces"]) == 2
    got = _agree(*with_degenerate(*grid_patch(8, 7, 2), seed=5), 20.0)
    assert ofh.FILLED in got["status"]
    got = _agree(*dense_random(300, 80, 3), 2.0)                 # dangling chains: no loop closes
    assert got["lines"] > 3
    v, f = fin()
    _agree(v, f, 2.0)
    with pytest.raises(ValueError):
        ofh.fill_holes(v, np.array([[0, 1, len(v)]], np.int32))
    with pytest.raises(ValueError):
        ofh.fill_holes(v, f, float("nan"))
