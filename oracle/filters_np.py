"""TEST INFRASTRUCTURE ONLY -- numpy restatements of the two third-party pre-filters the reference
calls and that are NOT vendored under /root/reference (SURVEY.md section 8c, Appendix D):

  * pywt.swtn(level=1) -- PyWavelets >= 1.6.0 (pyproject.toml:36), called at
    radiomics/imageoperations.py:935: periodic, undecimated convolution with the decomposition
    filters, out[n] = sum_j h[j] x[(n + F/2 - j) mod N], axes processed in the order given; odd
    lengths are wrap-padded by one sample and cropped (imageoperations.py:914-919,947-951).
  * ITK LaplacianRecursiveGaussianImageFilter -- SimpleITK >= 2.4.0 (pyproject.toml:35), called at
    radiomics/imageoperations.py:824-830: 4th-order Deriche-type recursive Gaussian (zero order
    along two axes, second order along the third), causal + anti-causal, sigma^2-normalised, summed
    over the three axes, float32 output.

PARITY UNPINNED: neither library is installed offline and the reference's tests hold no golden
vector for them (tests/test_wavelet.py compares the unfiltered image, SURVEY.md section 4).  These
restatements are checked by mathematical properties only (tests/test_filters_*.py): perfect
reconstruction / Parseval for the wavelet, agreement with an analytic Gaussian-Laplacian for LoG.
"""
from __future__ import annotations


import numpy as np


def swt_axis(x, h, axis):
    x = np.asarray(x, float)
    N = x.shape[axis]
    xp = x
    if N % 2:
        first = np.take(x, [0], axis=axis)
        xp = np.concatenate([x, first], axis=axis)
    F = len(h)
    out = np.zeros_like(xp)
    for j in range(F):
        out += h[j] * np.roll(xp, j - F // 2, axis=axis)     # roll by s: out[n] = x[n - s]
    if N % 2:
        out = np.take(out, range(N), axis=axis)
    return out


def swtn_level1(x, lo, hi, axes):
    """dict like pywt.swtn(..., level=1)[0]: keys of 'a'/'d', one letter per axis in `axes` order.
    (Padding of odd dimensions is applied per axis, which equals padding all axes first.)"""
    cur = {"": np.asarray(x, float)}
    for ax in axes:
        nxt = {}
        for k, v in cur.items():
            nxt[k + "a"] = swt_axis(v, lo, ax)
            nxt[k + "d"] = swt_axis(v, hi, ax)
        cur = nxt
    return cur


def recursive_gaussian_axis(x, coef, axis):
    """causal + anti-causal 4th-order recursion with 'edge value extends to infinity' boundaries;
    coef = N0..3, D1..4, M1..4 (+ unused boundary terms), float64 arithmetic."""
    N0, N1, N2, N3, D1, D2, D3, D4, M1, M2, M3, M4 = coef[:12]
    x = np.moveaxis(np.asarray(x, float), axis, 0)
    n = x.shape[0]
    SD = 1 + D1 + D2 + D3 + D4
    causal = np.zeros_like(x)
    x1 = x2 = x3 = x[0]
    y1 = y2 = y3 = y4 = x[0] * (N0 + N1 + N2 + N3) / SD
    for i in range(n):
        y = N0 * x[i] + N1 * x1 + N2 * x2 + N3 * x3 - D1 * y1 - D2 * y2 - D3 * y3 - D4 * y4
        causal[i] = y
        x3, x2, x1 = x2, x1, x[i]
        y4, y3, y2, y1 = y3, y2, y1, y
    out = np.zeros_like(x)
    a1 = a2 = a3 = a4 = x[n - 1]
    b1 = b2 = b3 = b4 = x[n - 1] * (M1 + M2 + M3 + M4) / SD
    for i in range(n - 1, -1, -1):
        y = M1 * a1 + M2 * a2 + M3 * a3 + M4 * a4 - D1 * b1 - D2 * b2 - D3 * b3 - D4 * b4
        out[i] = causal[i] + y
        a4, a3, a2, a1 = a3, a2, a1, x[i]
        b4, b3, b2, b1 = b3, b2, b1, y
    return np.moveaxis(out, 0, axis)


def log_restatement(x, sigma_mm, spacing_zyx, in_dtype=None, coefficients=None, return_terms=False):
    """sigma^2-normalised LoG exactly as the CUDA path computes it (imageoperations.log_filter_device): a float64 input
    stays float64 for the first pass, every other input is rounded to float32.  Every pass is the float64 recursion
    (causal + anti-causal) times its scale, rounded to float32; per direction d the two smoothing passes run in the
    kernel's order (d = z: y then x; d = y: z then x; d = x: z then y), the derivative pass is scaled by sigma_d^2, and
    the three terms are added in float32 in the order z, y, x.  `coefficients(sigma_vox, order)` defaults to the host's
    recursive_gaussian_coefficients.  Returns the float32 image (and the terms T_z, T_y, T_x when asked)."""
    if coefficients is None:
        from pyradiomics_b200.imageoperations import recursive_gaussian_coefficients as coefficients
    in_dtype = np.dtype(in_dtype if in_dtype is not None else np.asarray(x).dtype)
    src = np.asarray(x).astype(np.float64 if in_dtype == np.float64 else np.float32).astype(np.float64)
    s = [sigma_mm / float(v) for v in spacing_zyx]

    def rg(v, axis, order, scale=1.0):
        return (recursive_gaussian_axis(v, coefficients(s[axis], order), axis) * scale).astype(np.float32)

    def f64(v):
        return v.astype(np.float64)

    gz = f64(rg(src, 0, 0))
    terms = [rg(f64(rg(f64(rg(src, 1, 0)), 2, 0)), 0, 2, s[0] * s[0]),
             rg(f64(rg(gz, 2, 0)), 1, 2, s[1] * s[1]),
             rg(f64(rg(gz, 1, 0)), 2, 2, s[2] * s[2])]
    out = terms[0] + terms[1]
    out = out + terms[2]
    return (out, terms) if return_terms else out


def swt3_levels(x, lo, hi, axes, level=1, start_level=0):
    """restatement of the reference's _swt3 (radiomics/imageoperations.py:899-970) around swtn_level1: the odd axes are
    wrap-padded by one sample ONCE (:914-919), every level is a level-1 transform of the previous (still padded)
    approximation (:924-937), start_level discards the first levels, and only what is handed out is cropped (:947-963).
    Returns (approximation, [ {band: array} per kept level ])."""
    x = np.asarray(x, float)
    orig = x.shape
    pad = [(0, 1 if (d in axes and x.shape[d] % 2) else 0) for d in range(x.ndim)]
    data = np.pad(x, pad, "wrap")
    crop = tuple(slice(0, n) for n in orig)
    key_a = "a" * len(axes)

    def one(d):
        cur = {"": d}
        for ax in axes:                       # plain periodic convolution on the even-sized padded array
            nxt = {}
            for k, v in cur.items():
                nxt[k + "a"] = swt_axis(v, lo, ax)
                nxt[k + "d"] = swt_axis(v, hi, ax)
            cur = nxt
        return cur

    for _ in range(start_level):
        data = one(data)[key_a]
    out = []
    for _ in range(start_level, start_level + level):
        dec = one(data)
        data = dec[key_a]
        out.append({k: v[crop] for k, v in dec.items() if k != key_a})
    return data[crop], out
