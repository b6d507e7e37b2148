"""The checker of the volume rendering's data preparation (oracle/raycasting.c) against an independent NumPy
restatement: the flip and shift as array expressions, the convolution on zero-padded slices with the in-bounds
shifted products added in the contract's tap and weight order (a padded tap adds 0.0 * 0.0, and adding +0.0 to a
non-negative sum is exact), and the histogram from np.bincount. The identity kernel pins the boundary rule: the
other reading of it (the weight at the tap's own position) would return the image unchanged. CPU only."""
import numpy as np
import pytest

from oracle import raycasting as orc

# volume.py's "Basic Smooth 5x5", as it builds the weights: [i / 60.0 for i in Kernels[name]]
SMOOTH = [i / 60.0 for i in (1, 1, 1, 1, 1, 1, 4, 4, 4, 1, 1, 4, 12, 4, 1, 1, 4, 4, 4, 1, 1, 1, 1, 1, 1)]
IDENTITY = [0.0] * 12 + [1.0] + [0.0] * 12
SHAPES = [(1, 1, 1), (1, 3, 4), (3, 5, 5), (7, 9, 11), (2, 64, 80)]


def random_kernel(seed: int, total: float = 0.999) -> list:
    """Non-negative, non-symmetric weights summing to about `total`."""
    w = np.random.default_rng(seed).random(25) ** 2
    return (w * (total / w.sum())).tolist()


def near_limit_kernel(seed: int) -> list:
    """Weights whose 65535-fold sum is just below 65536: the largest sums reach past 65535."""
    w = random_kernel(seed, 65535.75 / 65535.0)
    assert 65535.0 * sum(w) < 65536.0
    return w


KERNELS = {"smooth": SMOOTH, "identity": IDENTITY, "random0": random_kernel(0), "random1": random_kernel(1),
           "near_limit": near_limit_kernel(2)}


def image(shape, kind: str, seed: int = 0) -> np.ndarray:
    """'full': int16 noise with -32768 and 32767 present; 'positive': min > 0; 'constant'; 'ct': CT-like values."""
    rng = np.random.default_rng(seed)
    if kind == "full":
        m = rng.integers(-32768, 32768, size=shape, dtype=np.int16)
        m.flat[0], m.flat[-1] = -32768, 32767
        return m
    if kind == "positive":
        return rng.integers(17, 3000, size=shape, dtype=np.int16)
    if kind == "constant":
        return np.full(shape, -1000, np.int16)
    return rng.integers(-1024, 3072, size=shape, dtype=np.int16)


KINDS = ["full", "positive", "constant", "ct"]


# ---- the NumPy restatement ------------------------------------------------------------------------------------
def np_flip_shift(m: np.ndarray):
    lo, hi = float(m.min()), float(m.max())
    return (m[:, ::-1, :].astype(np.float64) + abs(lo)).astype(np.uint16), (lo, hi)


def np_convolve(u: np.ndarray, w) -> np.ndarray:
    w = np.asarray(w, np.float64)
    dz, dy, dx = u.shape
    p = np.zeros((dz, dy + 4, dx + 4))
    p[:, 2:-2, 2:-2] = u
    ys, xs = np.arange(dy), np.arange(dx)
    k = np.zeros((dy, dx), np.int64)
    total = np.zeros(u.shape)
    for b in range(5):
        yin = (ys + b - 2 >= 0) & (ys + b - 2 < dy)
        for a in range(5):
            inb = yin[:, None] & ((xs + a - 2 >= 0) & (xs + a - 2 < dx))[None, :]
            wk = np.where(inb, w[np.minimum(k, 24)], 0.0)
            total = total + p[:, b:b + dy, a:a + dx] * wk
            k += inb
    return np.minimum(np.trunc(total), 65535).astype(np.uint16)


def np_chain(u, kernels):
    for w in kernels:
        u = np_convolve(u, w)
    return u


def np_histogram(m: np.ndarray):
    lo, hi = int(m.min()), int(m.max())
    r = hi - lo
    return np.bincount((m.astype(np.int64) - lo).ravel(), minlength=r + 1)[:r], float(lo), float(hi)


def identity_border(u: np.ndarray) -> np.ndarray:
    """The identity kernel under the contract's rule, voxel by voxel: the 13th in-bounds tap, or 0."""
    dz, dy, dx = u.shape
    out = np.empty_like(u)
    for y in range(dy):
        for x in range(dx):
            taps = [(y + b - 2, x + a - 2) for b in range(5) for a in range(5)
                    if 0 <= y + b - 2 < dy and 0 <= x + a - 2 < dx]
            out[:, y, x] = u[:, taps[12][0], taps[12][1]] if len(taps) > 12 else 0
    return out


def cases():
    return [(f"{kind}_{'x'.join(map(str, s))}", s, kind) for s in SHAPES for kind in KINDS]


# ---- tests ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,shape,kind", cases())
def test_flip_shift(name, shape, kind):
    m = image(shape, kind)
    u, rng = orc.flip_shift(m)
    want_u, want_rng = np_flip_shift(m)
    assert rng == want_rng
    assert np.array_equal(u, want_u)


@pytest.mark.parametrize("kernel", sorted(KERNELS))
@pytest.mark.parametrize("name,shape,kind", cases())
def test_convolve(name, shape, kind, kernel):
    u, _ = orc.flip_shift(image(shape, kind))
    assert np.array_equal(orc.convolve(u, KERNELS[kernel]), np_convolve(u, KERNELS[kernel]))


@pytest.mark.parametrize("name,shape,kind", cases())
def test_histogram(name, shape, kind):
    m = image(shape, kind)
    counts, lo, hi = orc.histogram(m)
    want, wlo, whi = np_histogram(m)
    assert (lo, hi) == (wlo, whi) and counts.dtype == np.int64
    assert np.array_equal(counts, want)
    if kind == "constant":
        assert counts.size == 0


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 3, 4), (2, 4, 7), (3, 5, 5), (2, 9, 11), (1, 6, 40)])
def test_identity_kernel_pins_the_border_rule(shape):
    u, _ = orc.flip_shift(image(shape, "full", seed=3))
    got = orc.convolve(u, IDENTITY)
    assert np.array_equal(got, identity_border(u))
    assert np.array_equal(got[:, 2:-2, 2:-2], u[:, 2:-2, 2:-2])
    assert not np.array_equal(got, u)      # the positional rule would give u back


@pytest.mark.parametrize("passes", [0, 1, 2, 3])
def test_chains(passes):
    u, _ = orc.flip_shift(image((3, 33, 47), "full", seed=4))
    kernels = [SMOOTH, random_kernel(5), near_limit_kernel(6)][:passes]
    got = orc.convolve_chain(u, kernels)
    assert np.array_equal(got, np_chain(u, kernels))
    if passes == 0:
        assert np.array_equal(got, u)


def test_cranium(cranium):
    m = cranium["matrix_crop"]
    u, rng = orc.flip_shift(m)
    want_u, want_rng = np_flip_shift(m)
    assert rng == want_rng and np.array_equal(u, want_u)
    for w in (SMOOTH, IDENTITY, random_kernel(7)):
        assert np.array_equal(orc.convolve(u, w), np_convolve(u, w))
    assert np.array_equal(orc.convolve_chain(u, [SMOOTH, SMOOTH]), np_chain(u, [SMOOTH, SMOOTH]))
    counts, lo, hi = orc.histogram(m)
    want, wlo, whi = np_histogram(m)
    assert (lo, hi) == (wlo, whi) and np.array_equal(counts, want)


BAD_KERNELS = {
    "24_weights": [1 / 60.0] * 24,
    "negative": SMOOTH[:5] + [-SMOOTH[5]] + SMOOTH[6:],
    "nan": SMOOTH[:12] + [float("nan")] + SMOOTH[13:],
    "sum_too_large": [1.0 / 24] * 25,
}


@pytest.mark.parametrize("bad", sorted(BAD_KERNELS))
def test_rejected_kernels(bad):
    u, _ = orc.flip_shift(image((2, 6, 7), "ct"))
    with pytest.raises(ValueError):
        orc.convolve(u, BAD_KERNELS[bad])


def test_rejected_float32_image():
    m = image((2, 6, 7), "ct").astype(np.float32)
    with pytest.raises(TypeError):
        orc.flip_shift(m)
    with pytest.raises(TypeError):
        orc.histogram(m)
