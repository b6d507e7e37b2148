"""CPU checker for the porous-scaffold TPMS and Blobs generators — TEST INFRASTRUCTURE ONLY.

A NumPy / SciPy restatement of plugins/porous_creation/schwarzp.py:11-34 and of the float64 image_normalize
(imagedata_utils.py:580-587), written from the surfaces' definitions in the plugin's broadcast form:

  create_schwarzp   the six triply periodic minimal surfaces on np.ogrid axes (NumPy broadcasting, left to right)
  create_blobs      np.random.random((sz, sy, sx)) and a separable Gaussian: one scipy.ndimage.correlate1d pass
                    per axis with the normalised, reversed exp(-x^2 / (2 sigma^2)) kernel of radius
                    int(4 sigma + 0.5), in mode "reflect"; no pass at all for sigma <= 1e-15
  image_normalize   (image - imin) * ((max_ - min_) / (imax - imin)) + min_ into int16, or min_ on a constant image
  schwarzp_i16_slabs  image_normalize(create_schwarzp(...)) in z-slabs, two passes (global min / max, then the
                    normalise), so a 1000^3 field is never held on the host
"""
from __future__ import annotations

import numpy as np
from scipy import ndimage as ndi

SURFACES = ("Schwarz P", "Schwarz D", "Gyroid", "Neovius", "iWP", "P_W_Hybrid")


def axes(init_x, end_x, init_y, end_y, init_z, end_z, sx=256, sy=256, sz=256):
    """(z, y, x) sparse grids of sz, sy and sx points from init to end, inclusive."""
    return np.ogrid[init_z:end_z:complex(0, sz), init_y:end_y:complex(0, sy), init_x:end_x:complex(0, sx)]


def surface(method, z, y, x):
    """The level-set function of a TPMS on broadcastable axes; None for an unknown method."""
    if method == "Schwarz P":
        return np.cos(x) + np.cos(y) + np.cos(z)
    if method == "Schwarz D":
        return (np.sin(x) * np.sin(y) * np.sin(z) + np.sin(x) * np.cos(y) * np.cos(z)
                + np.cos(x) * np.sin(y) * np.cos(z) + np.cos(x) * np.cos(y) * np.sin(z))
    if method == "Gyroid":
        return np.cos(x) * np.sin(y) + np.cos(y) * np.sin(z) + np.cos(z) * np.sin(x)
    if method == "Neovius":
        return 3 * (np.cos(x) + np.cos(y) + np.cos(z)) + 4 * np.cos(x) * np.cos(y) * np.cos(z)
    pairs = np.cos(x) * np.cos(y) + np.cos(y) * np.cos(z) + np.cos(z) * np.cos(x)
    if method == "iWP":
        return pairs - np.cos(x) * np.cos(y) * np.cos(z)
    if method == "P_W_Hybrid":
        return 4.0 * pairs - 3 * np.cos(x) * np.cos(y) * np.cos(z) + 2.4
    return None


def create_schwarzp(method, init_x, end_x, init_y, end_y, init_z, end_z, sx=256, sy=256, sz=256):
    return surface(method, *axes(init_x, end_x, init_y, end_y, init_z, end_z, sx, sy, sz))


def gaussian_weights(sigma: float) -> np.ndarray:
    """The correlation weights of a Gaussian of standard deviation sigma, truncated at 4 sigma."""
    radius = int(4.0 * sigma + 0.5)
    k = np.arange(-radius, radius + 1)
    w = np.exp(-0.5 / (sigma * sigma) * k ** 2)
    return (w / w.sum())[::-1]


def gaussian(image: np.ndarray, sigma) -> np.ndarray:
    out = np.array(image, dtype=np.float64)
    sigma = float(sigma)
    if not sigma > 1e-15:
        return out
    w = gaussian_weights(sigma)
    for axis in range(out.ndim):
        out = ndi.correlate1d(out, w, axis, mode="reflect")
    return out


def create_blobs(sx=256, sy=256, sz=256, gaussian_sigma=5):
    return gaussian(np.random.random((sz, sy, sx)), gaussian_sigma)


def image_normalize(image, min_=0.0, max_=1.0):
    imin, imax = image.min(), image.max()
    out = np.empty(image.shape, np.int16)
    if imin == imax:
        out[:] = min_
    else:
        out[:] = (image - imin) * ((max_ - min_) / (imax - imin)) + min_
    return out


def schwarzp_i16_slabs(method, init_x, end_x, init_y, end_y, init_z, end_z, sx, sy, sz, min_=-1000, max_=1000,
                       slab=16):
    """image_normalize(create_schwarzp(...), min_, max_), evaluated slab by slab along z (the field is elementwise,
    so every slab equals the same rows of the whole field)."""
    z, y, x = axes(init_x, end_x, init_y, end_y, init_z, end_z, sx, sy, sz)
    imin, imax = np.inf, -np.inf
    for k in range(0, z.shape[0], slab):
        f = surface(method, z[k:k + slab], y, x)
        imin, imax = min(imin, f.min()), max(imax, f.max())
    out = np.empty((z.shape[0], y.shape[1], x.shape[2]), np.int16)
    for k in range(0, z.shape[0], slab):
        if imin == imax:
            out[k:k + slab] = min_
        else:
            out[k:k + slab] = (surface(method, z[k:k + slab], y, x) - imin) * ((max_ - min_) / (imax - imin)) + min_
    return out
