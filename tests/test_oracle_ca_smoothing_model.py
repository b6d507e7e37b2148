"""The CPU checker of context-aware smoothing (oracle/mesh.c) against the NumPy restatement written from
mesh.rs (ca_smoothing_model.py): equal bit for bit, the seed rule of find_staircase_artifacts pinned, and the
test meshes shown to tell apart the ways a restatement could be subtly wrong."""
import numpy as np
import pytest

import ca_smoothing_model as M
from ca_smoothing_model import PARAMS

INF, NAN = float("inf"), float("nan")
FAMILY = M.family()
SIZED = M.sized_family()


def _same(a, b):
    return np.array_equal(a, b, equal_nan=True)


def _checker(orc, V, F4, N, p):
    v = V.copy()
    return v, orc.ca_smoothing(v, F4, N, *p, return_weights=True)


def _model(V, F4, N, p, **kw):
    v = V.copy()
    return v, M.ca_smoothing(v, F4, N, *p, **kw)


@pytest.mark.parametrize("name", list(FAMILY))
def test_checker_equals_sequential_model(orc, name):
    V, F4, N = FAMILY[name]
    for p in PARAMS:
        (vc, wc), (vm, wm) = _checker(orc, V, F4, N, p), _model(V, F4, N, p)
        assert _same(wc, wm) and _same(vc, vm), p


@pytest.mark.parametrize("name", list(SIZED))
def test_checker_equals_sequential_model_sized(orc, name):
    V, F4, N = SIZED[name]
    for p in [(0.7, 3.0, 0.1, 3), (NAN, 3.0, -0.5, 2)]:
        (vc, wc), (vm, wm) = _checker(orc, V, F4, N, p), _model(V, F4, N, p)
        assert _same(wc, wm) and _same(vc, vm), p


def _referenced(F4, nv):
    e = F4.reshape(-1)
    return np.unique(e[(e >= 0) & (e < nv)])


@pytest.mark.parametrize("name", list(FAMILY))
def test_seed_rule(orc, name):
    """Finite T (negative and 0 included): every referenced vertex, the leading column counting. T = NaN:
    none. T = inf: exactly the vertices whose first face in map_vface order has a NaN normal. Read from the
    checker's weights too: with bmin = -0.5 and tmax = 1e-300 a seed weighs 1 and every other vertex -0.5."""
    V, F4, N = FAMILY[name]
    nv = len(V)
    N = N.copy()
    N[np.random.default_rng(nv).random(len(F4)) < 0.3] = np.nan
    first = M.first_face(F4, nv)
    if nv > 3 and F4[0, 0] == 3:
        assert first[3] == 0                       # row 0's leading 3
    on_nan = [v for v in range(nv) if first[v] >= 0 and np.isnan(N[first[v]]).any()]
    vf = M.map_vface(F4, nv)
    for T, want in [(0.7, _referenced(F4, nv)), (0.0, _referenced(F4, nv)), (-1.0, _referenced(F4, nv)),
                    (NAN, []), (INF, on_nan)]:
        assert M.staircase_seeds(N, vf, T) == [int(v) for v in want], T
        _, w = _checker(orc, V, F4, N, (T, 1e-300, -0.5, 0))
        assert np.array_equal(np.flatnonzero(w == 1.0), np.asarray(want, np.int64)), T
        assert np.all((w == 1.0) | (w == -0.5))


VARIANT_CASES = {
    "reversed_neighbours": (0.7, 3.0, 0.1, 7),
    "fused_d": (0.7, 3.0, 0.1, 7),
    "no_column0": (0.7, 3.0, -0.5, 2),
    "w(ld)": (NAN, 3.0, M.MIDPOINT_BMIN, 3),
    "largest_seed": (INF, 3.0, 0.1, 1),
}


@pytest.mark.parametrize("variant", M.VARIANTS)
def test_family_tells_each_variant_apart(variant):
    p = VARIANT_CASES[variant]
    schedule = "rounds" if variant == "largest_seed" else "sequential"
    differ = []
    for name, (V, F4, N) in FAMILY.items():
        (va, wa), (vb, wb) = _model(V, F4, N, p, schedule=schedule), _model(V, F4, N, p, schedule=schedule, variant=variant)
        if not (_same(va, vb) and _same(wa, wb)):
            differ.append(name)
    assert differ, variant


def test_schedules_agree_when_seed_balls_are_disjoint(orc):
    """Seeds 12 and 62 of a strip (faces 10 and 60 with NaN normals, T = inf), 25 apart: every schedule
    gives the same weights while tmax < 12.5; above that the seeds compete for the vertices between them."""
    from connectivity_meshes import strip
    V, F4, N = M.as_mesh(*strip(80))
    N[[10, 60]] = np.nan
    assert M.staircase_seeds(N, M.map_vface(F4, len(V)), INF) == [12, 62]
    for tmax in (4.0, 10.0, 20.0):
        p = (INF, tmax, 0.2, 2)
        (vs, ws), (vr, wr), (vc, wc) = _model(V, F4, N, p), _model(V, F4, N, p, schedule="rounds"), _checker(orc, V, F4, N, p)
        assert _same(ws, wc) and _same(vs, vc)
        assert (np.isfinite(ws) & (ws > 0.2)).sum() > 2 * tmax      # the weights did propagate
        if tmax < 12.5:
            assert _same(ws, wr) and _same(vs, vr)


def test_rounds_tie_goes_to_the_smallest_seed():
    V, F4, N = M.tie()
    adj = M.adjacency(F4, len(V))
    seeds = M.staircase_seeds(N, M.map_vface(F4, len(V)), INF)
    assert seeds == [2, 3]
    _, d, s = M.propagate_weights(V, adj, seeds, 3.0, 0.1, "rounds")
    assert s[0] == 2 and d[0] == 1.0 and s[1] == 2
    _, d2, s2 = M.propagate_weights(V, adj, seeds, 3.0, 0.1, "rounds", largest_seed=True)
    assert s2[0] == 3 and s2[1] == 3 and d2[1] > d[1]
