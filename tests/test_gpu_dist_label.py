"""Z-sharded labelling with the CUDA backend: dist.label and dist.fill_holes_auto over 2, 3 and 4
ranks sharing one GPU through gloo, and over NCCL with one rank per GPU where there are two or more.
The concatenated labels must equal scipy.ndimage.label and labeling.label_device of the whole volume
bit for bit, and the sharded fill must equal labeling.fill_holes_auto on the whole mask. The three
new C entries (boundary forest, resolve, relabel) are also compared directly with the NumPy
restatement of tests/test_dist_label_gloo.py."""
import numpy as np
import pytest
import torch
from scipy import ndimage

from dist_common import run_ranks
from test_dist_label_gloo import (FILL_SIZES, boundary_forest, boundary_raw_pairs, check_label_matrix, fill_cases,
                                  label_cases, resolve, run_label_matrix, structures)

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda", torch.cuda.current_device())


def rank_label_device(rank, world, device):
    from invesalius3_b200 import dist as d
    return run_label_matrix(rank, world, device, d.DeviceBackend, lambda t: t.to(_dev()), lambda t: t.cpu())


def _check_against_device(out, world):
    """The same volumes through the single-GPU labelling and fill."""
    from invesalius3_b200 import device as dev, labeling
    for name, vol in label_cases(world):
        for sname, st in structures().items():
            want, n = labeling.label_device(dev.to_device(vol), st)
            got = np.concatenate([out[r][("label", name, sname)][0] for r in range(world)])
            assert np.array_equal(got, want.cpu().numpy().view(np.uint32)), (name, sname)
            assert out[0][("label", name, sname)][1] == n, (name, sname)
    for name, mask in fill_cases().items():
        for conn in (6, 18, 26):
            for size in FILL_SIZES:
                want = mask.copy()
                ret = labeling.fill_holes_auto(want, conn, size)
                got = np.concatenate([out[r][("fill", name, conn, size)][1] for r in range(world)])
                assert np.array_equal(got, want), (name, conn, size)
                assert all(out[r][("fill", name, conn, size)][0] == ret for r in range(world)), (name, conn, size)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_label_ranks_one_gpu_gloo(orc, world):
    out = run_ranks("rank_label_device", "test_gpu_dist_label", world=world, device="cuda")
    check_label_matrix(out, world, orc)
    _check_against_device(out, world)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_label_ranks_nccl(orc):
    world = min(4, torch.cuda.device_count())
    out = run_ranks("rank_label_device", "test_gpu_dist_label", world=world, device="nccl")
    check_label_matrix(out, world, orc)
    _check_against_device(out, world)


# ---- the C entries on their own
def _two_slabs(vol, st, split):
    """Local labels of vol[:split] and vol[split:] (the planes around the boundary) and their counts."""
    lo, n_lo = ndimage.label(vol[:split], _pad(st), output=np.uint32)
    hi, n_hi = ndimage.label(vol[split:], _pad(st), output=np.uint32)
    return lo[-1], hi[0], int(n_lo), int(n_hi)


def _pad(st):
    from test_dist_label_gloo import pad3
    return pad3(st)


def _boundary(lo, hi, st, base_lo, n_lo, n_hi):
    from invesalius3_b200 import dist as d, labeling
    lo_t = torch.from_numpy(np.ascontiguousarray(lo).view(np.int32)).cuda()
    hi_t = torch.from_numpy(np.ascontiguousarray(hi).view(np.int32)).cuda()
    return d.DeviceBackend().lb_boundary(lo_t, hi_t, labeling._structure(st, 3), base_lo, n_lo, n_hi).cpu().numpy()


@pytest.mark.parametrize("sname", list(structures()))
@pytest.mark.parametrize("density", [0.3, 0.5, 0.7])
def test_boundary_forest_matches_restatement(sname, density):
    st = structures()[sname]
    rng = np.random.default_rng(int(density * 10))
    for shape, split, base_lo in (((6, 33, 70), 3, 0), ((4, 1, 300), 2, 12345), ((5, 70, 1), 1, 7), ((2, 128, 96), 1, 2 ** 33)):
        vol = rng.random(shape) < density
        lo, hi, n_lo, n_hi = _two_slabs(vol, st, split)
        got = _boundary(lo, hi, st, base_lo, n_lo, n_hi)
        want = boundary_forest(lo, hi, st, base_lo, n_lo)
        assert got.dtype == np.int64 and np.array_equal(got, want), (shape, split)


def test_boundary_forest_is_bounded_by_the_labels():
    """64x256x256 noise, 26-connected: at most one pair per distinct label on the two planes, against
    tens of thousands of raw voxel pairs."""
    st = structures()["s26"]
    vol = np.random.default_rng(5).random((64, 256, 256)) < 0.3
    lo, hi, n_lo, n_hi = _two_slabs(vol, st, 32)
    got = _boundary(lo, hi, st, 0, n_lo, n_hi)
    distinct = len(np.unique(lo[lo > 0])) + len(np.unique(hi[hi > 0]))
    raw = boundary_raw_pairs(lo.astype(np.int64), hi.astype(np.int64), st, n_lo)
    assert 0 < len(got) <= distinct < len(raw)
    assert len(np.unique(got[:, 0])) == len(got)                       # one pair per label
    assert np.array_equal(got, boundary_forest(lo, hi, st, 0, n_lo))


def test_resolve_and_relabel_match_numpy():
    from invesalius3_b200 import dist as d
    be = d.DeviceBackend()
    rng = np.random.default_rng(9)
    st = structures()["s18"]
    vol = rng.random((12, 40, 50)) < 0.45
    cuts = [0, 3, 4, 8, 12]
    labs = [ndimage.label(vol[a:b], _pad(st), output=np.uint32) for a, b in zip(cuts[:-1], cuts[1:])]
    counts = [int(n) for _, n in labs]
    bases = np.cumsum([0] + counts[:-1]).tolist()
    pairs = np.concatenate([boundary_forest(labs[r][0][-1], labs[r + 1][0][0], st, bases[r], counts[r])
                            for r in range(len(labs) - 1)])
    assert len(pairs) > 20
    for r in range(len(labs)):
        lut, merged = be.lb_resolve(torch.from_numpy(pairs).cuda(), bases[r], counts[r])
        want_lut, want_merged = resolve(pairs, bases[r], counts[r])
        assert merged == want_merged
        assert np.array_equal(lut.cpu().numpy().view(np.uint32), want_lut), r
    whole, n = ndimage.label(vol, _pad(st), output=np.uint32)
    assert sum(counts) - merged == n
    # no pairs at all: the table adds the base
    lut, merged = be.lb_resolve(torch.zeros((0, 2), dtype=torch.int64, device="cuda"), 40, 5)
    assert merged == 0 and lut.cpu().numpy().tolist() == [0, 41, 42, 43, 44, 45]
    # relabel: vector and scalar paths (offset views), values beyond the table unchanged
    table = rng.integers(0, 2 ** 32, 1000, dtype=np.uint64).astype(np.uint32)
    lut_t = torch.from_numpy(table.view(np.int32)).cuda()
    for n_vox, off in ((1 << 16, 0), (4099, 0), (4099, 1), (7, 3), (1, 2)):
        vals = rng.integers(0, 1100, n_vox + off).astype(np.uint32)
        buf = torch.from_numpy(vals.view(np.int32)).cuda()
        view = buf[off:]
        be.lb_relabel(view, lut_t)
        want = vals.copy()
        sel = want[off:] < 1000
        want[off:][sel] = table[want[off:][sel]]
        assert np.array_equal(buf.cpu().numpy().view(np.uint32), want), (n_vox, off)


def test_resolve_rejects_missing_endpoints():
    from invesalius3_b200 import _lib, device as dev
    pairs = torch.tensor([[5, 2]], dtype=torch.int64, device="cuda")
    ends = torch.tensor([2, 6], dtype=torch.int64, device="cuda")
    lut = torch.empty(4, dtype=torch.int32, device="cuda")
    lib = _lib.load()
    ws = dev._workspace(lib.b2v_label_resolve_workspace_bytes(2), lut.device)
    import ctypes as C
    nm = C.c_int64(0)
    with pytest.raises(ValueError):
        _lib.call("b2v_label_resolve", dev._p(pairs), 1, dev._p(ends), 2, 0, 3, dev._p(lut), dev._p(ws), dev._stream(),
                  C.byref(nm))
