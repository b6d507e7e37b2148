"""Context-aware smoothing on the device at its edges, bit for bit against the CPU checker (oracle/mesh.c) and
the NumPy restatement of mesh.rs (ca_smoothing_model.py): the mesh family and every parameter edge, the
propagation rounds (T = inf with NaN normals), the face-ring limit, the interface, and full-size surfaces."""
import time

import numpy as np
import pytest

import ca_smoothing_model as M
from connectivity_meshes import fan, strip
from ca_smoothing_model import PARAMS
from smoothing_meshes import grid_patch

pytestmark = pytest.mark.gpu

INF, NAN = float("inf"), float("nan")
FAMILY = {**M.family(), **M.sized_family()}


def _same(a, b):
    return np.array_equal(a, b, equal_nan=True)         # NaN payloads differ between host and device


def _device(V, F4, N, p):
    from invesalius3_b200 import mesh_ops
    v = V.copy()
    mesh_ops.context_aware_smoothing(v, F4, N, *p)
    return v


def _checker(orc, V, F4, N, p):
    v = V.copy()
    orc.ca_smoothing(v, F4, N, *p)
    return v


def _model(V, F4, N, p, schedule="sequential"):
    v = V.copy()
    M.ca_smoothing(v, F4, N, *p, schedule=schedule)
    return v


@pytest.mark.parametrize("name", list(FAMILY))
def test_family_equals_checker_and_model(orc, name):
    V, F4, N = FAMILY[name]
    for p in PARAMS:
        got = _device(V, F4, N, p)
        assert _same(got, _checker(orc, V, F4, N, p)), p
        assert _same(got, _model(V, F4, N, p)), p


def test_leading_column_any_value(orc):
    """The leading column is a key of the reference's map only: out of range (negative, past V, beyond
    int32) it is ignored, in range it adds its face to that vertex's seed test."""
    V, F4, N = M.as_mesh(*grid_patch(6, 5, seed=9, jitter=0.5))
    F4[:, 0] = np.resize([-5, len(V), len(V) + 100, 1 << 40, 3, 7], len(F4))
    for p in [(0.7, 3.0, -0.5, 4), (INF, 3.0, 0.1, 2)]:
        got = _device(V, F4, N, p)
        assert _same(got, _checker(orc, V, F4, N, p)) and _same(got, _model(V, F4, N, p)), p


# ---- the propagation rounds: T = inf, NaN normals on chosen faces ---------------------------------------------
def _one_seed_faces(F4, nv):
    """(faces that are the first face of exactly one vertex, excluding face 0, and that vertex of each)."""
    first = M.first_face(F4, nv)
    has = first >= 0
    owners = np.bincount(first[has], minlength=len(F4))
    owner = np.full(len(F4), -1, np.int64)
    owner[first[has]] = np.flatnonzero(has)
    faces = np.flatnonzero(owners == 1)
    faces = faces[faces > 0]
    return faces, owner[faces]


def _rounds_case(orc, V, F4, N, p, disjoint):
    got = _device(V, F4, N, p)
    assert _same(got, _model(V, F4, N, p, schedule="rounds")), p
    if disjoint:
        assert _same(got, _checker(orc, V, F4, N, p)), p
    return got


def test_rounds_one_nan_face(orc):
    V, F4, N = M.as_mesh(*grid_patch(24, 20, seed=4, jitter=0.5))
    faces, _ = _one_seed_faces(F4, len(V))
    N[faces[len(faces) // 2]] = np.nan
    for tmax in (2.5, 6.0, INF):
        got = _rounds_case(orc, V, F4, N, (INF, tmax, 0.1, 3), disjoint=True)
        assert not _same(got, _device(V, F4, M.face_normals(V, F4[:, 1:]), (INF, tmax, 0.1, 3)))


def test_rounds_two_far_apart_nan_faces(orc):
    """Seeds 12 and 62 of a strip, 25 apart: tmax below half their distance (disjoint balls, every schedule
    agrees) and above it (the rounds compete for the vertices between them)."""
    V, F4, N = M.as_mesh(*strip(80))
    N[[10, 60]] = np.nan
    for tmax in (4.0, 12.0, 13.0, 20.0, INF):
        for bmin in (0.1, -0.5):
            _rounds_case(orc, V, F4, N, (INF, tmax, bmin, 2), disjoint=tmax < 12.5)


def test_rounds_tie_goes_to_the_smallest_seed(orc):
    V, F4, N = M.tie()
    for p in [(INF, 3.0, 0.1, 1), (INF, 3.0, -0.5, 4), (INF, 2.0, 0.3, 2)]:
        got = _rounds_case(orc, V, F4, N, p, disjoint=False)
        other = V.copy()
        M.ca_smoothing(other, F4, N, *p, schedule="rounds", variant="largest_seed")
        assert not _same(got, other), p


@pytest.mark.parametrize("name", ["sized2049", "sized4097", "shuffled_spheres", "dense_random"])
def test_rounds_many_seeds(orc, name):
    """Several NaN faces on a mesh with long random edges: many seeds whose balls overlap, many rounds."""
    V, F4, N = FAMILY[name]
    N = N.copy()
    N[np.random.default_rng(1).choice(len(F4), 6, replace=False)] = np.nan
    for tmax in (1.5, INF):
        _rounds_case(orc, V, F4, N, (INF, tmax, 0.1, 2), disjoint=False)


# ---- the face-ring limit -------------------------------------------------------------------------------------
def test_ring_of_96_faces_works_and_97_raises(orc):
    V, F4, N = M.as_mesh(*fan(96))
    p = (0.7, 3.0, 0.1, 3)
    assert _same(_device(V, F4, N, p), _checker(orc, V, F4, N, p))
    V, F4, N = M.as_mesh(*fan(97))
    with pytest.raises(ValueError, match="96 faces"):
        _device(V, F4, N, p)


def test_degenerate_ring_counts_faces_not_entries(orc):
    """[3, 0, 0, k] holds vertex 0 twice: 49 such faces are 49 faces (98 entries) and work; 97 are refused."""
    def ring(n):
        v = (np.random.default_rng(n).random((n + 1, 3)) * 4).astype(np.float32)
        return M.as_mesh(v, [(0, 0, k) for k in range(1, n + 1)])
    for p in [(0.7, 3.0, 0.1, 3), (NAN, 3.0, -0.5, 2)]:
        V, F4, N = ring(49)
        got = _device(V, F4, N, p)
        assert _same(got, _checker(orc, V, F4, N, p)) and _same(got, _model(V, F4, N, p))
        V, F4, N = ring(96)
        assert _same(_device(V, F4, N, p), _checker(orc, V, F4, N, p))
    V, F4, N = ring(97)
    with pytest.raises(ValueError, match="96 faces"):
        _device(V, F4, N, (0.7, 3.0, 0.1, 1))


# ---- the interface -------------------------------------------------------------------------------------------
def test_interface(orc):
    import torch
    from invesalius3_b200 import invesalius_rs, mesh_ops
    V, F4, N = M.as_mesh(*grid_patch(9, 8, seed=6, jitter=0.7))
    p = (0.7, 3.0, 0.1, 5)
    want = _checker(orc, V, F4, N, p)
    assert not _same(want, V)
    for dt in (np.int64, np.int32, np.uint32, np.uint64):
        v = V.copy()
        mesh_ops.context_aware_smoothing(v, F4.astype(dt), N, *p)
        assert _same(v, want), dt
    v = V.copy()
    mesh_ops.context_aware_smoothing(v, F4, N.astype(np.float64), *p)     # float32-representable float64
    assert _same(v, want)
    with pytest.raises(NotImplementedError):
        mesh_ops.context_aware_smoothing(V.copy(), F4, N.astype(np.float64) + 1e-12, *p)
    m = mesh_ops.Mesh(vertices=V.copy(), faces=F4, normals=N)
    m2 = mesh_ops.Mesh(other=m)
    mesh_ops.ca_smoothing(m, *p)
    assert _same(m.vertices, want) and _same(m2.vertices, V)           # the copy is untouched
    invesalius_rs.ca_smoothing(m2, *p)
    assert _same(m2.vertices, want)
    a = np.full((len(V), 4), 7.0, np.float32)                            # a strided view, smoothed in place
    a[:, :3] = V
    mesh_ops.context_aware_smoothing(a[:, :3], F4, N, *p)
    assert _same(a[:, :3], want) and (a[:, 3] == 7.0).all()
    tv, tf, tn = (torch.from_numpy(x).cuda() for x in (V.copy(), F4, N))
    mesh_ops.smooth_device(tv, tf, tn, *p)
    assert _same(tv.cpu().numpy(), want)


def test_errors():
    import torch
    from invesalius3_b200 import mesh_ops
    V, F4, N = M.as_mesh(*grid_patch(5, 5, seed=2))
    for n in (1 << 32, (1 << 32) + 5, -1):
        with pytest.raises(OverflowError):
            mesh_ops.context_aware_smoothing(V.copy(), F4, N, 0.7, 3.0, 0.1, n)
        with pytest.raises(OverflowError):
            mesh_ops.smooth_device(*(torch.from_numpy(x).cuda() for x in (V.copy(), F4, N)), 0.7, 3.0, 0.1, n)
    for col, bad in [(1, len(V)), (2, -1), (3, len(V) + 1000)]:
        f = F4.copy()
        f[3, col] = bad
        with pytest.raises(ValueError, match="outside the vertex array"):
            mesh_ops.context_aware_smoothing(V.copy(), f, N, 0.7, 3.0, 0.1, 1)


# ---- full-size surfaces --------------------------------------------------------------------------------------
def _full_size(orc, V, F, label):
    F4, N = M.as_mesh(V, F)[1:]
    timings = []
    for p in [(0.7, 3.0, 0.1, 3), (0.7, 3.0, 0.1, 10)]:
        t0 = time.perf_counter()
        got = _device(V, F4, N, p)
        timings.append(time.perf_counter() - t0)
        assert _same(got, _checker(orc, V, F4, N, p)), p
        assert np.abs(got - V).max() > 1e-3
    # the rounds at full size: four seeds, each the only new vertex of a NaN-normal face, their tmax-balls
    # disjoint, so the device must equal the sequential checker
    tmax = 6.0
    cand, owner = _one_seed_faces(F4, len(V))
    seeds, faces = [], []
    for k in np.linspace(0, len(cand) - 1, 64).astype(int):
        s = owner[k]
        if all(np.linalg.norm(V[s].astype(np.float64) - V[t]) > 2 * tmax + 1 for t in seeds):
            seeds.append(s)
            faces.append(cand[k])
        if len(seeds) == 4:
            break
    assert len(seeds) == 4
    N2 = N.copy()
    N2[faces] = np.nan
    p = (INF, tmax, 0.1, 3)
    t0 = time.perf_counter()
    got = _device(V, F4, N2, p)
    timings.append(time.perf_counter() - t0)
    assert _same(got, _checker(orc, V, F4, N2, p))
    assert not _same(got, _device(V, F4, N, p))        # the seeds did move their neighbourhoods
    print(f"{label}: V={len(V)} T={len(F)} device call (incl. copies) s: n_iters 3 {timings[0]:.3f}, "
          f"n_iters 10 {timings[1]:.3f}, T=inf with 4 seeds {timings[2]:.3f}")


def test_cranium_surface(orc, cranium):
    import torch
    from invesalius3_b200.mesh import marching_cubes
    full = tuple(int(s) for s in cranium["full_shape"])
    mask = np.unpackbits(cranium["mask_0_bits_full"])[:np.prod(full)].reshape(full) * np.uint8(255)
    sx, sy, sz = (float(s) for s in cranium["spacing"])
    V, F = marching_cubes(torch.from_numpy(mask).cuda(), 127, (sx, sy, sz), (0, 0, 0), True)
    V, F = V.cpu().numpy(), F.cpu().numpy()
    assert len(F) > 100_000
    _full_size(orc, V, F, "cranium")


def test_phantom_512_bone_surface(orc):
    import torch
    from invesalius3_b200 import device as dev, phantom
    from invesalius3_b200.mesh import marching_cubes
    vol = phantom.ct((512, 512, 512), seed=2)
    mask = dev.threshold(torch.from_numpy(vol).cuda(), 226, 3071)
    del vol
    V, F = marching_cubes(mask, 127, (1.0, 1.0, 1.0), (0, 0, 0), True)
    del mask
    V, F = V.cpu().numpy(), F.cpu().numpy()
    assert len(F) > 5_000_000
    _full_size(orc, V, F, "phantom 512^3 bone")
