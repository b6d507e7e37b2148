"""Meshes for the connectivity tests, and a plain-Python restatement of vtkPolyDataConnectivityFilter's
TraverseAndMark (real wave lists, written independently of oracle/connectivity.c) to check the checker."""
from __future__ import annotations

import numpy as np

from visibility_meshes import icosphere


def traverse_py(nv: int, faces: np.ndarray, seeds=None):
    """(region [T], point_map [V], sizes) by the contract in oracle/connectivity.c's header."""
    f = [tuple(int(x) for x in row) for row in np.asarray(faces).reshape(-1, 3)]
    links = [[] for _ in range(nv)]
    for t, tri in enumerate(f):
        for p in tri:
            links[p].append(t)
    region = [-1] * len(f)
    pmap = [-1] * nv
    counter = [0]

    def mark(wave, r):
        n = 0
        while wave:
            nxt = []
            for c in wave:
                if region[c] >= 0:
                    continue
                region[c] = r
                n += 1
                for p in f[c]:
                    if pmap[p] < 0:
                        pmap[p] = counter[0]
                        counter[0] += 1
                    nxt.extend(links[p])
            wave = nxt
        return n

    sizes = []
    if seeds is None:
        for t in range(len(f)):
            if region[t] < 0:
                sizes.append(mark([t], len(sizes)))
    else:
        wave = []
        for s in seeds:
            if s >= 0:
                wave.extend(links[s])
        sizes.append(mark(wave, 0))
    return np.array(region, np.int32), np.array(pmap, np.int32), np.array(sizes, np.int64)


def strip(n: int):
    """A triangle strip of n triangles over two rows of points (point ids in strip order)."""
    k = n // 2 + 2
    v = np.zeros((2 * k, 3), np.float32)
    v[0::2, 0] = np.arange(k)
    v[1::2, 0] = np.arange(k) + 0.5
    v[1::2, 1] = 1.0
    f = np.array([(i, i + 1, i + 2) for i in range(n)], np.int32)
    return v, f


def shuffled_spheres(count: int, seed: int):
    """`count` disjoint icospheres of random levels, faces shuffled, points permuted, plus unused points."""
    rng = np.random.default_rng(seed)
    vs, fs, off = [], [], 0
    for i in range(count):
        v, f = icosphere(1.0, int(rng.integers(0, 3)), center=(3.0 * i, 0.0, 0.0))
        vs.append(v)
        fs.append(f + off)
        off += len(v)
    vs.append(rng.random((7, 3)).astype(np.float32))        # unused points
    v = np.concatenate(vs)
    f = np.concatenate(fs)
    perm = rng.permutation(len(v))
    inv = np.empty_like(perm)
    inv[perm] = np.arange(len(v))
    return v[perm], inv[f][rng.permutation(len(f))].astype(np.int32)


def dense_random(nt: int, nv: int, seed: int):
    """Random triangles over few points: repeated and degenerate corners, several regions, unused points."""
    rng = np.random.default_rng(seed)
    f = rng.integers(0, nv, (nt, 3)).astype(np.int32)
    return rng.random((nv + 3, 3)).astype(np.float32), f


def fan(n: int):
    """n triangles around one point (id 0), plus a separate triangle."""
    ring = n + 1
    v = np.zeros((ring + 4, 3), np.float32)
    a = np.linspace(0, 2 * np.pi, ring, endpoint=False)
    v[1:ring + 1, 0], v[1:ring + 1, 1] = np.cos(a), np.sin(a)
    f = [(0, 1 + i, 2 + i) for i in range(n)] + [(ring + 1, ring + 2, ring + 3)]
    return v, np.array(f, np.int32)


def noise_volume(n: int, p: float, seed: int) -> np.ndarray:
    """uint8 [n,n,n] mask (255 inside) of voxels set with probability p: many small fragments."""
    return (np.random.default_rng(seed).random((n, n, n)) < p).astype(np.uint8) * np.uint8(255)
