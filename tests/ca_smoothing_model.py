"""Context-aware smoothing (invesalius_rs.context_aware_smoothing, mesh.rs:27-395) restated in NumPy from the
crate's source, independently of oracle/mesh.c, to check that checker; and the meshes its tests run on.

Stages, each as the crate writes it:
  build_map_vface            every column of a face row is a key, the leading 3 included, in (face, column)
                             order. Keys outside [0, V) are never looked up, so they are dropped here.
  build_vertex_connectivity  columns 1..3 x 1..3 of each face, first appearance only.
  find_staircase_artifacts   the max / min tracking with its `else if`; nalgebra's 3-vector dot product is
                             (a0*b0 + a1*b1) + a2*b2.
  propagate_weights          see `propagate_weights` for its two schedules.
  taubin_smooth              lambda 0.5, mu -0.53: D in float64, each vertex summing its neighbours in
                             adjacency order, then x = (w * l) * d cast to float32 and added in float32.

`variant` names one deliberate change, used to show that the test meshes tell the variants apart:
  "reversed_neighbours"  each adjacency list reversed (a different float64 summation order);
  "no_column0"           the leading column left out of map_vface;
  "w(ld)"                x = w * (l * d);
  "fused_d"              d = d + p_i - p_j evaluated left to right, (d + p_i) - p_j;
  "largest_seed"         ties between equal offers in a round go to the largest seed ("rounds" only).
"""
from __future__ import annotations

import math

import numpy as np

from connectivity_meshes import dense_random, fan, shuffled_spheres, strip
from smoothing_meshes import fin, folded_sheet, grid_patch, hexagon_fan, with_degenerate, with_unused

F64_MAX = float(np.finfo(np.float64).max)
LAMBDA, MU = 0.5, -0.53
VARIANTS = ("reversed_neighbours", "no_column0", "w(ld)", "fused_d", "largest_seed")


def map_vface(faces, nv, column0=True):
    vf = [[] for _ in range(nv)]
    cols = range(4) if column0 else range(1, 4)
    for f_id, row in enumerate(np.asarray(faces).tolist()):
        for c in cols:
            if 0 <= row[c] < nv:
                vf[row[c]].append(f_id)
    return vf


def adjacency(faces, nv):
    adj = [[] for _ in range(nv)]
    for row in np.asarray(faces).tolist():
        tri = row[1:]
        if not all(0 <= v < nv for v in tri):
            raise IndexError("face entry outside the vertex array")
        for vi in tri:
            for vj in tri:
                if vi != vj and vj not in adj[vi]:
                    adj[vi].append(vj)
    return adj


def staircase_seeds(normals, vf, t):
    """The vertices find_staircase_artifacts returns, ascending."""
    nrm = np.asarray(normals).astype(np.float64).tolist()
    t = float(t)
    out = []
    for v, f_ids in enumerate(vf):
        max_z = max_y = max_x = -F64_MAX
        min_z = min_y = min_x = F64_MAX
        for f in f_ids:
            nx, ny, nz = nrm[f]
            of_z = 1.0 - abs((nx * 0.0 + ny * 0.0) + nz * 1.0)
            of_y = 1.0 - abs((nx * 0.0 + ny * 1.0) + nz * 0.0)
            of_x = 1.0 - abs((nx * 1.0 + ny * 0.0) + nz * 0.0)
            if of_z > max_z:
                max_z = of_z
            elif of_z < min_z:
                min_z = of_z
            if of_y > max_y:
                max_y = of_y
            elif of_y < min_y:
                min_y = of_y
            if of_x > max_x:
                max_x = of_x
            elif of_x < min_x:
                min_x = of_x
            if abs(max_z - min_z) >= t or abs(max_y - min_y) >= t or abs(max_x - min_x) >= t:
                out.append(v)
                break
    return out


def propagate_weights(pos, adj, seeds, tmax, bmin, schedule="sequential", largest_seed=False):
    """(weights float64 [V], squared distances [V], seed of each vertex [V]).

    The crate runs each frontier with rayon: every frontier vertex reads its seed when its task starts and
    lowers a neighbour's distance by compare-and-swap, storing its seed after a successful swap. Both
    schedules here are executions of that loop:
      "sequential"  one task at a time, in frontier order (each task sees every earlier swap), and a vertex
                    enters the next frontier once per successful swap;
      "rounds"      every task reads its seed before any swap of the round lands, and the offers to each
                    vertex land smallest first, so only the smallest offer swaps (if it is strictly below
                    the vertex's distance) and the vertex enters the next frontier once. Among equal
                    smallest offers the first to land stays (a later equal one is not below it); here
                    that is the smallest seed's (`largest_seed` flips it).
    Both give the same result whenever no vertex receives offers from two seeds, e.g. when the seeds'
    tmax-balls are disjoint."""
    P = np.asarray(pos).astype(np.float64).tolist()
    n = len(P)
    dist = [math.inf] * n
    seed = [-1] * n
    for s in seeds:
        dist[s], seed[s] = 0.0, s
    tmax_sq = tmax * tmax

    def sqdist(a, b):
        dx, dy, dz = P[a][0] - P[b][0], P[a][1] - P[b][1], P[a][2] - P[b][2]
        return dx * dx + dy * dy + dz * dz

    def accepts(d_sq, old):
        return not (d_sq >= old and math.isfinite(old))

    frontier = list(seeds)
    while frontier:
        nxt = []
        if schedule == "sequential":
            for v in frontier:
                s = seed[v]
                for vj in adj[v]:
                    d_sq = sqdist(vj, s)
                    if d_sq > tmax_sq or not accepts(d_sq, dist[vj]):
                        continue
                    dist[vj], seed[vj] = d_sq, s
                    nxt.append(vj)
        elif schedule == "rounds":
            best = {}
            for v in frontier:
                s = seed[v]
                for vj in adj[v]:
                    d_sq = sqdist(vj, s)
                    if d_sq > tmax_sq or not accepts(d_sq, dist[vj]):
                        continue
                    b = best.get(vj)
                    if b is None or d_sq < b[0] or (d_sq == b[0] and (s > b[1] if largest_seed else s < b[1])):
                        best[vj] = (d_sq, s)
            for vj, (d_sq, s) in best.items():
                dist[vj], seed[vj] = d_sq, s
            nxt = sorted(best)
        else:
            raise ValueError(schedule)
        frontier = nxt
    d = np.array(dist, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):        # tmax = 0: 0 / 0 and 1 / 0, as IEEE has them
        w = np.where(np.isfinite(d), (1.0 - np.sqrt(d) / np.float64(tmax)) * (1.0 - np.float64(bmin)) + bmin, bmin)
    return w, d, np.array(seed)


def taubin(vertices, adj, w, n_iters, product="(wl)d", fused_d=False):
    """vertices float32 [V,3], modified in place."""
    nv = len(vertices)
    deg = np.array([len(a) for a in adj], np.int64)
    width = int(deg.max()) if nv else 0
    A = np.zeros((nv, max(width, 1)), np.int64)
    for i, a in enumerate(adj):
        A[i, :len(a)] = a
    for _ in range(n_iters):
        for lm in (LAMBDA, MU):
            p = vertices.astype(np.float64)
            d = np.zeros((nv, 3), np.float64)
            for k in range(width):
                pj = p[A[:, k]]
                step = (d + p) - pj if fused_d else d + (p - pj)
                d = np.where((k < deg)[:, None], step, d)
            d = np.where((deg > 0)[:, None], d / np.maximum(deg, 1)[:, None].astype(np.float64), d)
            x = (w * lm)[:, None] * d if product == "(wl)d" else w[:, None] * (lm * d)
            vertices += x.astype(np.float32)


def ca_smoothing(vertices, faces, normals, T, tmax, bmin, n_iters, schedule="sequential", variant=None):
    """vertices float32 [V,3] (smoothed in place), faces integer [M,4], normals [M,3]; returns the weights."""
    assert variant is None or variant in VARIANTS
    faces = np.asarray(faces).astype(np.int64)
    nv = len(vertices)
    adj = adjacency(faces, nv)
    if variant == "reversed_neighbours":
        adj = [a[::-1] for a in adj]
    vf = map_vface(faces, nv, column0=variant != "no_column0")
    seeds = staircase_seeds(normals, vf, T)
    w, _, _ = propagate_weights(vertices, adj, seeds, float(tmax), float(bmin), schedule, variant == "largest_seed")
    taubin(vertices, adj, w, int(n_iters), "w(ld)" if variant == "w(ld)" else "(wl)d", variant == "fused_d")
    return w


# ---- meshes ------------------------------------------------------------------------------------------------
def face_normals(v, f3):
    """float32 unit normals of float32 vertices; a degenerate triangle gets (0, 0, 0)."""
    a, b, c = (v[f3[:, k]].astype(np.float64) for k in range(3))
    n = np.cross(b - a, c - a)
    n /= np.maximum(np.linalg.norm(n, axis=1), 1e-30)[:, None]
    return np.ascontiguousarray(n.astype(np.float32))


def as_mesh(v, f3, col0=3):
    f3 = np.asarray(f3, np.int64).reshape(-1, 3)
    F4 = np.ascontiguousarray(np.c_[np.full(len(f3), col0, np.int64), f3])
    v = np.ascontiguousarray(v, np.float32)
    return v, F4, face_normals(v, f3)


def soup(n, seed=0):
    """n triangles that share no vertex."""
    rng = np.random.default_rng(seed)
    return (rng.random((3 * n, 3)) * 4).astype(np.float32), np.arange(3 * n).reshape(n, 3)


def duplicates():
    """A grid patch with some faces repeated, some repeated reversed."""
    v, f = grid_patch(5, 4, seed=3, jitter=0.4)
    return v, np.concatenate([f, f[[0, 5, 9]], f[[2, 5, 11]][:, ::-1]])


def non_manifold_edge():
    """Four triangles on the edge (0, 1)."""
    v = np.array([[0, 0, 0], [1, 0, 0], [0.5, 1, 0], [0.5, -1, 0.1], [0.5, 0.2, 1], [0.4, 0.1, -1]], np.float32)
    return v, np.array([(0, 1, 2), (1, 0, 3), (0, 1, 4), (5, 1, 0)])


def bow_tie():
    """Two triangle fans that meet at one vertex (0) only."""
    v = np.array([[0, 0, 0], [1, 0.2, 0], [1, 1, 0.3], [0.1, 1, 0], [-1, -0.2, 0], [-1, -1, 0.2], [0, -1, 0.1]],
                 np.float32)
    return v, np.array([(0, 1, 2), (0, 2, 3), (0, 4, 5), (0, 5, 6)])


def column0_only(seed=0):
    """A grid patch whose leading column names vertices no face holds (7 of them), one face row each."""
    v, f = grid_patch(4, 4, seed=seed, jitter=0.3)
    nv = len(v)
    v = np.concatenate([v, (np.random.default_rng(seed).random((7, 3)) * 3).astype(np.float32)])
    V, F4, N = as_mesh(v, f)
    F4[:7, 0] = np.arange(nv, nv + 7)
    return V, F4, N


def tiny(nv):
    """1, 2 or 3 vertices: faces over them (degenerate where they must be); the leading 3 is out of range."""
    v = np.array([[0, 0, 0], [1, 0.5, 0], [0.2, 1, 0.7]], np.float32)[:nv]
    f = {1: [(0, 0, 0)], 2: [(0, 1, 1), (1, 0, 0)], 3: [(0, 1, 2)]}[nv]
    return v, np.array(f)


def sized(nv, seed=0):
    """nv random points, each in six random triangles (some degenerate)."""
    rng = np.random.default_rng(seed)
    f = np.concatenate([rng.permutation(nv) for _ in range(6)])
    return rng.random((nv, 3)).astype(np.float32) * 10, f[:len(f) // 3 * 3].reshape(-1, 3)


def cancellation(n=40, seed=0):
    """n pairs of triangles (c, a, s1), (c, b, s2) with c, s1, s2 in [1, 2)^3, a = +2^40 and b = -2^40 in
    every coordinate: the float64 sum over c's neighbours cancels the large terms, and what is left depends
    on the order and grouping of the additions."""
    rng = np.random.default_rng(seed)
    v = np.empty((5 * n, 3), np.float32)
    v[:] = 1 + rng.random((5 * n, 3))
    v[1::5], v[3::5] = 2.0 ** 40, -2.0 ** 40
    return v, np.array([t for k in range(0, 5 * n, 5) for t in ((k, k + 1, k + 2), (k, k + 3, k + 4))])


def tie():
    """Seeds 2 and 3 (faces 0 and 1: degenerate, NaN normals) at the same distance from vertex 0, whose
    only other neighbours (1, 6) are nearer to seed 2 than to seed 3. Use with T = inf."""
    v = np.array([[0, 0, 0], [0.4, 1, 0], [1, 0, 0], [-1, 0, 0], [-1, 1, 0], [1, -1, 0], [-0.3, 1.5, 0]], np.float32)
    V, F4, N = as_mesh(v, [(3, 3, 3), (2, 2, 2), (3, 0, 4), (2, 0, 5), (0, 1, 6)])
    N[:2] = np.nan
    return V, F4, N


def midpoint_pairs(n=400, seed=0):
    """Pairs of points joined by one degenerate face, one coordinate in [1, 2) and the other in [-1, -0.5):
    their difference often has 25 significant bits, i.e. is a float32 rounding midpoint. With no seeds and
    bmin = MIDPOINT_BMIN, w * mu is exactly -1, so the mu step's x = -d lands on such midpoints exactly,
    and a product rounded in another order falls to either side of them."""
    rng = np.random.default_rng(seed)
    v = np.empty((2 * n, 3), np.float32)
    v[0::2] = 1 + rng.random((n, 3))
    v[1::2] = -0.5 - rng.random((n, 3)) / 2
    return v, np.array([(2 * k, 2 * k, 2 * k + 1) for k in range(n)])


MIDPOINT_BMIN = 1.0 / 0.53            # MIDPOINT_BMIN * -0.53 == -1.0 in float64

# (T, tmax, bmin, n_iters): each edge of T, tmax, bmin and n_iters, the propagation rounds (T = inf), and the
# midpoint probe
INF, NAN = math.inf, math.nan
PARAMS = [(0.7, 3.0, 0.1, 7), (0.0, 3.0, 0.1, 7), (-1.0, 3.0, 0.1, 7), (NAN, 3.0, 0.1, 7),
          (0.7, INF, 0.1, 7), (0.7, 1e-300, 0.1, 7), (0.7, 0.0, 0.1, 7),
          (0.7, 3.0, 0.0, 7), (0.7, 3.0, 1.0, 7), (0.7, 3.0, -0.5, 7),
          (0.7, 3.0, 0.1, 0), (0.7, 3.0, 0.1, 1),
          (INF, 3.0, 0.1, 3), (NAN, 3.0, MIDPOINT_BMIN, 3)]


def family():
    """name -> (vertices float32 [V,3], faces int64 [M,4], normals float32 [M,3])."""
    out = {
        "grid_patch": as_mesh(*grid_patch(7, 6, seed=1, jitter=0.6)),
        "fin": as_mesh(*fin()),
        "with_degenerate": as_mesh(*with_degenerate(*grid_patch(6, 5, seed=2, jitter=0.5), seed=4)),
        "with_unused": as_mesh(*with_unused(*grid_patch(6, 6, seed=5, jitter=0.5), seed=5)),
        "folded_sheet": as_mesh(*folded_sheet(7)),
        "hexagon_fan": as_mesh(*hexagon_fan()),
        "strip": as_mesh(*strip(11)),
        "fan12": as_mesh(*fan(12)),
        "shuffled_spheres": as_mesh(*shuffled_spheres(3, 7)),
        "dense_random": as_mesh(*dense_random(120, 30, 3)),
        "soup": as_mesh(*soup(9)),
        "duplicates": as_mesh(*duplicates()),
        "non_manifold_edge": as_mesh(*non_manifold_edge()),
        "bow_tie": as_mesh(*bow_tie()),
        "column0_only": column0_only(),
        "tiny1": as_mesh(*tiny(1)),
        "tiny2": as_mesh(*tiny(2)),
        "tiny3": as_mesh(*tiny(3)),
        "cancellation": as_mesh(*cancellation()),
        "midpoint_pairs": as_mesh(*midpoint_pairs()),
        "tie": tie(),
    }
    return out


def sized_family():
    """Vertex counts around the 2048-entry blocks of the adjacency scan."""
    return {f"sized{n}": as_mesh(*sized(n, seed=n)) for n in (2047, 2048, 2049, 4097)}


def first_face(F4, nv):
    """The first face of each vertex in map_vface order (-1: none)."""
    first = np.full(nv + 1, len(F4), np.int64)
    col = F4.reshape(-1)
    ok = (col >= 0) & (col < nv)
    np.minimum.at(first, np.where(ok, col, nv), np.repeat(np.arange(len(F4)), 4))
    first = first[:nv]
    return np.where(first == len(F4), -1, first)
