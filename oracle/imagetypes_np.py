"""NumPy restatement of the square, square root, logarithm, exponential and gradient image types (reference
radiomics/imageoperations.py:973-1091), written from their definitions: every statistic is taken over the whole image,
the arithmetic is float64 and each step rounds once, in the order the reference (NumPy) and ITK use.

* square:      (c x)^2, c = 1 / sqrt(M)                      M = max|x|; the sign is not kept
* squareroot:  sign(x) sqrt(|x| M), 0 and NaN unchanged
* logarithm:   sign(x) log(|x| + 1), then times M / max|that|  (the second maximum is taken here, not shortcut)
* exponential: exp(c x), c = log(M) / M
* gradient:    ITK GradientMagnitudeImageFilter: per axis of the image, x first, the inner product of the neighbours
               (f[i-1], f[i], f[i+1]) -- clamped to the edge -- with (-0.5, 0, 0.5) / spacing, accumulated as
               sqrt(((0 + gx^2) + gy^2) + gz^2); a 2-D image has two axes.
"""
from __future__ import annotations

import numpy as np

POINTWISE = ("square", "squareroot", "logarithm", "exponential")


def _f64(img):
    return np.asarray(img).astype(np.float64)


def _signed_log(x):
    t = x.copy()
    pos, neg = x > 0, x < 0
    t[pos] = np.log(x[pos] + 1.0)
    t[neg] = -np.log(1.0 - x[neg])
    return t


def scalar(img, kind):
    """the whole-image scalar of a per-voxel type, as a NumPy float64"""
    x = _f64(img)
    m = np.abs(x).max()
    with np.errstate(divide="ignore", invalid="ignore"):
        if kind == "square":
            return np.float64(1.0) / np.sqrt(m)
        if kind == "squareroot":
            return m
        if kind == "logarithm":
            return m / np.abs(_signed_log(x)).max()
        if kind == "exponential":
            return np.log(m) / m
    raise ValueError(kind)


def square(img):
    x = _f64(img)
    with np.errstate(invalid="ignore"):
        t = x * scalar(x, "square")
        return t * t


def squareroot(img):
    x = _f64(img)
    m = scalar(x, "squareroot")
    out = x.copy()
    pos, neg = x > 0, x < 0
    out[pos] = np.sqrt(x[pos] * m)
    out[neg] = -np.sqrt(np.abs(x[neg]) * m)
    return out


def logarithm(img):
    x = _f64(img)
    with np.errstate(invalid="ignore"):
        return _signed_log(x) * scalar(x, "logarithm")


def exponential(img):
    x = _f64(img)
    with np.errstate(invalid="ignore", over="ignore"):
        return np.exp(x * scalar(x, "exponential"))


def pointwise(img, kind):
    return {"square": square, "squareroot": squareroot, "logarithm": logarithm, "exponential": exponential}[kind](img)


def gradient(img, spacing=None):
    """`spacing`: one value per array axis (z, y, x order), or None for unit weights"""
    f = _f64(img)
    w = np.ones(f.ndim)
    if spacing is not None:
        sp = np.asarray(spacing, dtype=np.float64)
        if sp.shape != (f.ndim,):
            raise ValueError("one spacing per axis")
        if (sp == 0).any():
            raise ValueError("image spacing cannot be zero")
        w = 1.0 / sp
    acc = np.zeros_like(f)
    with np.errstate(invalid="ignore", over="ignore"):
        for ax in range(f.ndim - 1, -1, -1):
            n = f.shape[ax]
            below = np.take(f, np.maximum(np.arange(n) - 1, 0), axis=ax)
            above = np.take(f, np.minimum(np.arange(n) + 1, n - 1), axis=ax)
            g = ((-0.5 * w[ax]) * below + 0.0 * f) + (0.5 * w[ax]) * above
            acc = acc + g * g
        return np.sqrt(acc)
