"""NumPy / SciPy restatement of getLBP3DImage (reference radiomics/imageoperations.py:1169-1314), chunked over the ROI
voxels so that the (voxels, vertices) sample matrix never exceeds `chunk` rows.  Same steps as the reference: cubic
B-spline samples by scipy.ndimage.map_coordinates (mode='constant', output in the image's dtype), scipy.stats.kurtosis,
sign bits against the centre, spherical-harmonic coefficients (sph_harm_y with the reference's swapped angles), per level
the complex sum of squares and the real part of its square root.

Besides the maps it returns, per ROI voxel, the smallest margin that could flip a sign bit: |sample - centre| before the
cast for float images, the distance of the sample to the nearest .5 rounding point for integer images."""
from __future__ import annotations

import numpy as np
from scipy import ndimage
from scipy.special import sph_harm_y
from scipy.stats import kurtosis


def harmonics(vertices, levels, radius):
    v = np.asarray(vertices, dtype=np.float64)
    theta = np.arccos(np.true_divide(v[:, 2], radius))
    phi = np.arctan2(v[:, 1], v[:, 0])
    # the reference's sph_harm(m, n, theta, phi) took the azimuth third: phi lands in the polar slot
    cols = [sph_harm_y(n, m, phi, theta) for n in range(levels) for m in range(-n, n + 1)]
    n_ix = np.array([n for n in range(levels) for _ in range(-n, n + 1)])
    return np.stack(cols, axis=1), n_ix


def prefilter(img):
    return ndimage.spline_filter(np.asarray(img), order=3, output=np.float64, mode="constant")


def lbp3d(img, roi, vertices, levels, radius, chunk=8192, coef=None, coords=None):
    """img (Z,Y,X), roi boolean (Z,Y,X), vertices (Nv, 3) in (z, y, x) voxel offsets.
    Returns dict: coords (3, Np) of the ROI voxels (np.nonzero order), maps (levels + 1, Np) float64 (m1..mL, kurtosis),
    margin (Np,), m2 and mean (Np,) of the samples (kurtosis is NaN where m2 <= (eps * mean)^2).
    `coef`: the image's prefilter(img), if already computed; `coords` (3, Np): evaluate these voxels instead of the ROI's."""
    img = np.asarray(img)
    verts = np.asarray(vertices, dtype=np.float64)
    Y, n_ix = harmonics(verts, levels, radius)
    if coef is None:
        coef = prefilter(img)
    coords = np.array(np.nonzero(roi)) if coords is None else np.asarray(coords)
    Np = coords.shape[1]
    maps = np.empty((levels + 1, Np))
    margin = np.empty(Np)
    m2s = np.empty(Np)
    means = np.empty(Np)
    is_int = np.issubdtype(img.dtype, np.integer)
    for b in range(0, Np, chunk):
        c = coords[:, b:b + chunk]
        pts = c.T[None, :, :] + verts[:, None, :]                       # (Nv, n, 3)
        raw = ndimage.map_coordinates(coef, pts.T, order=3, mode="constant", prefilter=False, output=np.float64)
        f = ndimage.map_coordinates(coef, pts.T, order=3, mode="constant", prefilter=False, output=img.dtype)
        centre = img[tuple(c)]
        if is_int:
            a = np.abs(raw)
            margin[b:b + chunk] = np.abs(a - np.floor(a) - 0.5).min(axis=1)
        else:
            margin[b:b + chunk] = np.abs(raw - centre[:, None]).min(axis=1)
        mean = f.mean(axis=1)
        means[b:b + chunk] = mean
        m2s[b:b + chunk] = ((f - mean[:, None].astype(f.dtype)) ** 2).mean(axis=1)
        maps[levels, b:b + chunk] = np.real(kurtosis(f, axis=1))
        s = np.greater_equal(f, centre[:, None]).astype(int)             # (n, Nv)
        ck = (s[:, :, None] * Y[None, :, :]).sum(axis=1)                  # (n, K)
        for n in range(levels):
            g = (ck[:, None, n_ix == n] * Y[None, :, n_ix == n]).sum(axis=2)   # (n, Nv)
            maps[n, b:b + chunk] = np.real(np.sqrt((g ** 2).sum(axis=1)))
    return {"coords": coords, "maps": maps, "margin": margin, "m2": m2s, "mean": means}
