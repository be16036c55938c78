"""NumPy restatement of skimage.feature.local_binary_pattern (the library behind the reference's getLBP2DImage,
radiomics/imageoperations.py:1094-1166), vectorised over the pixels of a 2-D image: one array operation per rounding step
(NumPy's elementwise ufuncs never contract to FMA), the per-pixel loop order of the library's Cython
_local_binary_pattern and the bilinear interpolation of its _shared/interpolation.pxd (mode 'C', cval 0).

scikit-image is not a dependency: this module is both the test oracle and, through a skimage.feature stub, what the golden
generator hands to the reference's own wrapper (tests/golden/make_golden_lbp2d.py).
"""
from __future__ import annotations

import numpy as np

METHODS = {"default": 0, "ror": 1, "uniform": 2, "nri_uniform": 3, "var": 4}


def offsets(P, R):
    """(rp, cp): the library's rounded sample offsets, rows then columns"""
    rr = - R * np.sin(2 * np.pi * np.arange(P, dtype=np.float64) / P)
    cc = R * np.cos(2 * np.pi * np.arange(P, dtype=np.float64) / P)
    return np.round(rr, 5), np.round(cc, 5)


def _pixels(image, r, c):
    rows, cols = image.shape
    inside = (r >= 0) & (r < rows) & (c >= 0) & (c < cols)
    out = np.zeros(r.shape, np.float64)
    out[inside] = image[r[inside], c[inside]]
    return out


def bilinear(image, r, c):
    """the library's bilinear_interpolation at float positions (r, c) (arrays), corners outside the image read 0"""
    minr, minc = np.floor(r).astype(np.int64), np.floor(c).astype(np.int64)
    maxr, maxc = np.ceil(r).astype(np.int64), np.ceil(c).astype(np.int64)
    dr = r - minr.astype(np.float64)
    dc = c - minc.astype(np.float64)
    tl, tr = _pixels(image, minr, minc), _pixels(image, minr, maxc)
    bl, br = _pixels(image, maxr, minc), _pixels(image, maxr, maxc)
    with np.errstate(invalid="ignore", over="ignore"):
        wc, wr = 1 - dc, 1 - dr
        top = wc * tl + dc * tr
        bottom = wc * bl + dc * br
        return wr * top + dr * bottom


def textures(image, P, R):
    """(P, rows, cols) samples t_k of every pixel, and the image as float64"""
    image = np.ascontiguousarray(image, dtype=np.float64)
    rows, cols = image.shape
    r, c = np.meshgrid(np.arange(rows, dtype=np.float64), np.arange(cols, dtype=np.float64), indexing="ij")
    rp, cp = offsets(P, R)
    return np.stack([bilinear(image, r + rp[k], c + cp[k]) for k in range(P)]), image


def codes(bits, P, method):
    """per-pixel code of the sign bits `bits` ((P, ...) of 0/1) for the integer methods"""
    bits = bits.astype(np.int64)
    default = np.zeros(bits.shape[1:], np.int64)
    for k in range(P):
        default += bits[k] << k
    if method == "default":
        return default.astype(np.float64)
    if method == "ror":
        best, v = default.copy(), default.copy()
        for _ in range(1, P):
            v = (v >> 1) | ((v & 1) << (P - 1))
            best = np.minimum(best, v)
        return best.astype(np.float64)
    changes = (bits[:-1] != bits[1:]).sum(axis=0) if P > 1 else np.zeros(bits.shape[1:], np.int64)
    n_ones = bits.sum(axis=0)
    if method == "uniform":
        return np.where(changes <= 2, n_ones, P + 1).astype(np.float64)
    # nri_uniform
    first_one = np.argmax(bits == 1, axis=0)
    first_zero = np.argmax(bits == 0, axis=0)
    rot = np.where(first_one == 0, n_ones - first_zero, P - first_one)
    out = 1 + (n_ones - 1) * P + rot
    out = np.where(n_ones == 0, 0, out)
    out = np.where(n_ones == P, P * (P - 1) + 1, out)
    out = np.where(changes > 2, P * (P - 1) + 2, out)
    return out.astype(np.float64)


def local_binary_pattern(image, P, R, method="default"):
    """skimage.feature.local_binary_pattern(image, P, R, method) for a 2-D image -> float64 (rows, cols).  An unknown
    method raises KeyError, as the library's method dictionary does."""
    method = method.lower()
    METHODS[method]
    image = np.asarray(image)
    if image.ndim != 2:
        raise ValueError(f"local_binary_pattern: 2-D image expected, got {image.ndim}-D")
    P, R = int(P), float(R)
    t, img = textures(image, P, R)
    if method == "var":
        s = np.zeros(img.shape, np.float64)
        sq = np.zeros(img.shape, np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            for k in range(P):
                s = s + t[k]
                sq = sq + t[k] * t[k]
            v = (sq - (s * s) / P) / P
        return np.where(v != 0, v, np.nan)
    with np.errstate(invalid="ignore"):
        bits = (t - img[None]) >= 0
    return codes(bits, P, method)


def lbp2d_volume(image, P=8, R=1.0, method="uniform", axis=0):
    """float64 LBP of every slice of a 3-D image cut along `axis` (swapaxes(0, axis)), or of a 2-D image; no cast"""
    image = np.asarray(image)
    if image.ndim == 2:
        return local_binary_pattern(image, P, R, method)
    v = image.swapaxes(0, axis)
    out = np.stack([local_binary_pattern(v[i], P, R, method) for i in range(v.shape[0])])
    return np.ascontiguousarray(out.swapaxes(0, axis))
