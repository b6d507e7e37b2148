"""gloo tests (CPU) of the Z-sharded labelling in invesalius3_b200/dist.py: dist.label and
dist.fill_holes_auto over 2, 3 and 4 ranks, uneven shards, single-plane shards. The compute goes
through a CPU checker backend: ndimage.label per slab and a NumPy restatement of the boundary
pairs, their spanning forest, the union-find resolve and the lookup table. The concatenated labels
must equal scipy.ndimage.label of the whole volume bit for bit."""
import numpy as np
import pytest
import torch
from scipy import ndimage
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from dist_common import global_volume, run_ranks
from test_dist_gloo import CpuBackend

WORLDS = (2, 3, 4)


# ---- NumPy restatement of the three device stages
def _set_roots(ids, edges):
    """Root (smallest id) of every id's set under the edges (index pairs into ids)."""
    n = len(ids)
    if n == 0:
        return ids.copy()
    g = coo_matrix((np.ones(len(edges)), (edges[:, 0], edges[:, 1])), shape=(n, n)) if len(edges) else coo_matrix((n, n))
    _, comp = connected_components(g, directed=False)
    low = np.full(comp.max() + 1, np.iinfo(np.int64).max, np.int64)
    np.minimum.at(low, comp, ids)
    return low[comp]


def structure3(structure):
    from invesalius3_b200 import labeling
    return labeling._structure(structure, 3)


def pad3(structure):
    """The structure as SciPy takes it: 3 wide on every axis (a 1-wide axis padded with zeros)."""
    st = structure3(structure)
    out = np.zeros((3, 3, 3), np.uint8)
    out[(3 - st.shape[0]) // 2:][:st.shape[0], (3 - st.shape[1]) // 2:][:, :st.shape[1], (3 - st.shape[2]) // 2:][
        :, :, :st.shape[2]] = st
    return out


def boundary_raw_pairs(lo, hi, structure, n_lo):
    """Every (node below, node above) pair the structure's z = +1 offsets make between two planes of
    local labels; node = label below, n_lo + label above."""
    st = structure3(structure)
    ny, nx = lo.shape
    out = []
    if st.shape[0] != 3:
        return np.zeros((0, 2), np.int64)
    zp = np.zeros((3, 3), bool)
    oy0, ox0 = (3 - st.shape[1]) // 2, (3 - st.shape[2]) // 2
    zp[oy0: oy0 + st.shape[1], ox0: ox0 + st.shape[2]] = st[2].astype(bool)
    for oy, ox in np.argwhere(zp):
        dy, dx = oy - 1, ox - 1
        a = lo[max(0, -dy): ny - max(0, dy), max(0, -dx): nx - max(0, dx)].astype(np.int64)
        b = hi[max(0, dy): ny + min(0, dy), max(0, dx): nx + min(0, dx)].astype(np.int64)
        keep = (a > 0) & (b > 0)
        out.append(np.stack([a[keep], n_lo + b[keep]], 1))
    return np.concatenate(out) if out else np.zeros((0, 2), np.int64)


def boundary_forest(lo, hi, structure, base_lo, n_lo):
    """b2v_label_boundary_count / _emit: (P, P(root)) for every non-root label on the two planes, in
    the order of each label's first voxel (lower plane first, raster order)."""
    lo = np.asarray(lo).view(np.uint32).astype(np.int64)
    hi = np.asarray(hi).view(np.uint32).astype(np.int64)
    raw = boundary_raw_pairs(lo, hi, structure, n_lo)
    if len(raw) == 0:
        return np.zeros((0, 2), np.int64)
    nodes = np.concatenate([lo.ravel(), np.where(hi.ravel() > 0, n_lo + hi.ravel(), 0)])
    nodes = nodes[nodes > 0]
    ids, first = np.unique(nodes, return_index=True)
    root = _set_roots(ids, np.searchsorted(ids, raw))
    order = np.argsort(first, kind="stable")
    keep = order[root[order] != ids[order]]
    return np.stack([base_lo + ids[keep], base_lo + root[keep]], 1).astype(np.int64)


def resolve(pairs, base, nlocal):
    """b2v_label_resolve: (lut [nlocal + 1] uint32, |M|)."""
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    ends = np.unique(pairs)
    root = _set_roots(ends, np.searchsorted(ends, pairs))
    merged = np.sort(ends[root != ends])
    p = base + np.arange(1, nlocal + 1, dtype=np.int64)
    r = p.copy()                      # R = root(P), P itself when it is no endpoint
    if len(ends):
        k = np.minimum(np.searchsorted(ends, p), len(ends) - 1)
        hit = ends[k] == p
        r[hit] = root[k[hit]]
    lut = np.zeros(nlocal + 1, np.uint32)
    lut[1:] = (r - np.searchsorted(merged, r)).astype(np.uint32)
    return lut, len(merged)


class LabelCpuBackend(CpuBackend):
    """The labelling stages of dist.py's backend protocol in NumPy / SciPy."""

    def lb_local(self, fg, structure):
        lab, n = ndimage.label(fg.numpy(), pad3(structure), output=np.uint32)
        return torch.from_numpy(lab.view(np.int32)), int(n)

    def lb_boundary(self, lo_plane, hi_plane, structure, base_lo, n_lo, n_hi):
        return torch.from_numpy(boundary_forest(lo_plane.numpy(), hi_plane.numpy(), structure, base_lo, n_lo))

    def lb_resolve(self, pairs, base, nlocal):
        lut, merged = resolve(pairs.numpy(), base, nlocal)
        return torch.from_numpy(lut.view(np.int32)), merged

    def lb_relabel(self, labels, lut):
        a = labels.numpy().view(np.uint32)
        a[...] = lut.numpy().view(np.uint32)[a]
        return labels


# ---- the matrix
def structures():
    cross = np.zeros((1, 3, 3), np.uint8); cross[0, 1, :] = cross[0, :, 1] = 1
    zline = np.ones((3, 1, 1), np.uint8)
    return {"s6": ndimage.generate_binary_structure(3, 1), "s18": ndimage.generate_binary_structure(3, 2),
            "s26": ndimage.generate_binary_structure(3, 3), "cross133": cross, "zline311": zline}


def helix(shape, turns=3.0, radius=1.6):
    """A tube along x whose centre circles in (z, y): it crosses every z plane of the middle several times."""
    nz, ny, nx = shape
    z, y, x = np.mgrid[:nz, :ny, :nx].astype(np.float64)
    out = np.zeros(shape, bool)
    t = np.linspace(0, 1, 8 * nx)
    cz = (nz - 1) / 2 + (nz / 2 - 1.5) * np.cos(2 * np.pi * turns * t)
    cy = (ny - 1) / 2 + (ny / 2 - 2.5) * np.sin(2 * np.pi * turns * t)
    cx = 1 + (nx - 3) * t
    for a, b, c in zip(cz, cy, cx):
        out |= (z - a) ** 2 + (y - b) ** 2 + (x - c) ** 2 <= radius ** 2
    return out


def u_shapes(shape):
    """Two U shapes: one whose arms meet only in the bottom plane, one whose arms meet only in the top
    plane; each arm is its own local component in every other shard."""
    nz, ny, nx = shape
    v = np.zeros(shape, bool)
    v[:, 2, 2] = v[:, 2, 6] = True; v[0, 2, 2:7] = True              # joined at z = 0
    v[:, ny - 3, 3] = v[:, ny - 3, 9] = True; v[nz - 1, ny - 3, 3:10] = True   # joined at z = nz - 1
    return v


def label_cases(world):
    """(name, uint8 volume) pairs; the shapes are chosen per world size (uneven shards, DZ == world)."""
    rng = np.random.default_rng(100 + world)
    cases = []
    for dens in (0.3, 0.5, 0.7):
        cases.append((f"noise{dens}", (rng.random((11, 13, 17)) < dens)))
    g = global_volume()
    cases += [("ct", g >= 300), ("ct_complement", g < 300)]
    cases.append(("helix", helix((13, 14, 40))))
    cases.append(("u_shapes", u_shapes((11, 12, 14))))
    v = rng.random((11, 13, 17)) < 0.5
    from invesalius3_b200 import dist as d
    z0, z1 = d.ZShard(11, 1, world).z0, d.ZShard(11, 1, world).z1
    v[z0:z1] = False
    cases.append(("empty_shard", v))
    cases.append(("all_foreground", np.ones((11, 6, 7), bool)))
    cases.append(("all_background", np.zeros((11, 6, 7), bool)))
    cases.append(("dz_eq_world", rng.random((world, 9, 10)) < 0.55))
    cases.append(("one_plane_shard", rng.random((world + 1, 9, 10)) < 0.55))
    return [(n, a.astype(np.uint8)) for n, a in cases]


def fill_cases():
    rng = np.random.default_rng(11)
    mask = (ndimage.gaussian_filter(rng.normal(size=(23, 20, 45)), 1.0) > 0.02).astype(np.uint8) * 255
    mask[5, 3:8, 10:30] = 128      # > 127: selected
    mask[9, 4, 4] = 127            # not selected
    return {"blobs": mask, "sparse": (rng.random((13, 11, 19)) < 0.6).astype(np.uint8) * 255}


FILL_SIZES = (3, 50, 10 ** 7)


def run_label_matrix(rank, world, device, make_backend, to_dev, to_host):
    from invesalius3_b200 import dist as d
    be = make_backend()
    res = {}
    for name, vol in label_cases(world):
        shard = d.ZShard(vol.shape[0], rank, world)
        for sname, st in structures().items():
            fg = to_dev(torch.from_numpy(np.ascontiguousarray(vol[shard.z0:shard.z1])))
            lab, total = d.label(fg, st, shard, backend=be)
            res[("label", name, sname)] = (to_host(lab).numpy().view(np.uint32).copy(), total)
    for name, mask in fill_cases().items():
        shard = d.ZShard(mask.shape[0], rank, world)
        for conn in (6, 18, 26):
            for size in FILL_SIZES:
                m = to_dev(torch.from_numpy(mask[shard.z0:shard.z1].copy()))
                ret = d.fill_holes_auto(m, conn, size, shard, backend=be)
                res[("fill", name, conn, size)] = (ret, to_host(m).numpy().copy())
    return res


def rank_label(rank, world, device):
    return run_label_matrix(rank, world, device, LabelCpuBackend, lambda t: t, lambda t: t)


def check_label_matrix(out, world, orc):
    for name, vol in label_cases(world):
        for sname, st in structures().items():
            want, n = ndimage.label(vol, pad3(st), output=np.uint32)
            got = np.concatenate([out[r][("label", name, sname)][0] for r in range(world)])
            assert got.dtype == np.uint32 and np.array_equal(got, want), (name, sname)
            assert [out[r][("label", name, sname)][1] for r in range(world)] == [n] * world, (name, sname)
    for name, mask in fill_cases().items():
        for conn in (6, 18, 26):
            st = ndimage.generate_binary_structure(3, {6: 1, 18: 2, 26: 3}[conn])
            lab, n = ndimage.label(~(mask > 127), st, output=np.uint32)
            for size in FILL_SIZES:
                want = mask.copy()
                ret = orc.fill_holes_automatically(want, lab, int(n), size) if n else False
                got = np.concatenate([out[r][("fill", name, conn, size)][1] for r in range(world)])
                assert np.array_equal(got, want), (name, conn, size)
                assert all(out[r][("fill", name, conn, size)][0] == ret for r in range(world)), (name, conn, size)


@pytest.mark.parametrize("world", WORLDS)
def test_label_and_fill_holes_auto_ranks(orc, world):
    check_label_matrix(run_ranks("rank_label", "test_dist_label_gloo", world=world), world, orc)


def test_cases_cross_boundaries():
    """The matrix does what it claims: components span shards, the U arms meet only at one end, the
    (1,3,3) cross makes no boundary pairs and 26-connected noise makes many."""
    from invesalius3_b200 import dist as d
    st = structures()
    u = u_shapes((11, 12, 14))
    lab, n = ndimage.label(u, st["s6"])
    assert n == 2
    assert ndimage.label(u[1:], st["s6"])[1] == 3 and ndimage.label(u[:-1], st["s6"])[1] == 3
    h = helix((13, 14, 40))
    for world in WORLDS:
        for r in range(world - 1):
            z = d.ZShard(13, r, world).z1
            across = (h[z - 1] & h[z]).any(axis=0).astype(int)          # x where the tube passes the boundary
            assert np.count_nonzero(np.diff(np.r_[0, across]) == 1) >= 2, (world, r)
    rng = np.random.default_rng(0)
    a = ndimage.label(rng.random((2, 30, 30)) < 0.5, st["s26"], output=np.uint32)[0]
    assert len(boundary_forest(a[0], a[1], st["cross133"], 0, int(a[0].max()))) == 0
    raw = boundary_raw_pairs(a[0].astype(np.int64), a[1].astype(np.int64), st["s26"], int(a[0].max()))
    forest = boundary_forest(a[0], a[1], st["s26"], 0, int(a[0].max()))
    assert len(raw) > 1000 and 0 < len(forest) <= len(np.unique(a[:2][a[:2] > 0]))


def test_resolve_restatement_closed_forms():
    """Three provisional ids per rank, two ranks: 2~4 and 1~5 merge, so the finals are 1 2 3 2 1 4 and
    the total is 6 - 2."""
    pairs = np.array([[4, 2], [5, 1]], np.int64)
    assert resolve(pairs, 0, 3)[0].tolist() == [0, 1, 2, 3]
    lut, merged = resolve(pairs, 3, 3)
    assert lut.tolist() == [0, 2, 1, 4] and merged == 2


def test_empty_shard_raises():
    from invesalius3_b200 import dist as d
    shard = d.ZShard(2, 2, 3)
    with pytest.raises(ValueError):
        d.label(torch.zeros((0, 4, 4), dtype=torch.uint8), None, shard, backend=LabelCpuBackend())
    with pytest.raises(ValueError):
        d.fill_holes_auto(torch.zeros((0, 4, 4), dtype=torch.uint8), 6, 10, shard, backend=LabelCpuBackend())
