"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's resampling step (radiomics/imageoperations.py:448-612):
the grid arithmetic of resampleImage (:493-566) in numpy, and SimpleITK's ResampleImageFilter(sitkBSpline) /
(sitkNearestNeighbor) restated with SciPy's cubic B-spline machinery (spline_filter + map_coordinates, mirror boundaries --
the same Unser recursive filter ITK's BSplineDecompositionImageFilter implements; SimpleITK is not installed here).

PINNED on the reference's own baseline: with the value cast done by clamping + TRUNCATION (ITK's ResampleImageFilter), the
first-order features of the `breast1_resampling` column of data/baseline/baseline_firstorder.csv (23 ROI voxels after
resampling to 2 mm) are reproduced exactly -- Mean 126.17391304347827, Energy 375154 (tests/test_resample_cpu.py); with
rounding instead they are not.  Only tests/ may import this.
"""
from __future__ import annotations

import numpy as np


def grid(mask, spacing_xyz, new_spacing_xyz, padDistance=5, label=1, offset_xyz=(0, 0, 0), full_size_xyz=None):
    """(newSize xyz, start xyz, step xyz, newSpacing): output voxel k samples the input at continuous index start + k*step.
    `offset_xyz` / `full_size_xyz`: the arrays are a crop of a larger image starting at that index -- the output grid is
    anchored at the FULL image's index 0 (imageoperations.py:520-548), so a committed crop must say where it sat."""
    sp = np.array(spacing_xyz, float)
    new = np.array(new_spacing_xyz, float)
    new = np.where(new == 0, sp, new)
    idx = np.array(np.where(np.asarray(mask) == label))
    lo, hi = idx.min(1)[::-1], idx.max(1)[::-1]
    off = np.array(offset_xyz, float)
    bb = np.concatenate([lo + off, hi - lo + 1]).astype(float)
    nd = len(sp)
    size = np.array(np.asarray(mask).shape[::-1] if full_size_xyz is None else full_size_xyz, float)
    new = np.where(bb[nd:] != 1, new, sp)
    ratio = sp / new
    L = np.floor((bb[:nd] - 0.5) * ratio - padDistance)
    U = np.ceil((bb[:nd] + bb[nd:] - 0.5) * ratio + padDistance)
    maxU = np.ceil(size * ratio) - 1
    L = np.where(L < 0, 0, L)
    U = np.where(U > maxU, maxU, U)
    return (U - L + 1).astype(int), 0.5 * (new - sp) / sp + L / ratio - off, new / sp, new


def resample(image, mask, spacing_xyz, new_spacing_xyz, padDistance=5, label=1, order=3, offset_xyz=(0, 0, 0), full_size_xyz=None):
    import scipy.ndimage as ndi
    image, mask = np.asarray(image), np.asarray(mask)
    newSize, start, step, new = grid(mask, spacing_xyz, new_spacing_xyz, padDistance, label, offset_xyz, full_size_xyz)
    g = [start[d] + step[d] * np.arange(newSize[d]) for d in range(3)]          # x, y, z
    zz, yy, xx = np.meshgrid(g[2], g[1], g[0], indexing="ij")
    if order == 3:
        coef = ndi.spline_filter(image.astype(np.float64), order=3, mode="mirror")
        val = ndi.map_coordinates(coef, [zz, yy, xx], order=3, mode="mirror", prefilter=False)
    else:
        val = ndi.map_coordinates(image.astype(np.float64), [zz, yy, xx], order=order, mode="nearest")
    inside = np.ones(val.shape, bool)
    for c, n in ((zz, image.shape[0]), (yy, image.shape[1]), (xx, image.shape[2])):
        inside &= (c >= -0.5) & (c < n - 0.5)
    val = np.where(inside, val, 0.0)
    if np.issubdtype(image.dtype, np.integer):
        info = np.iinfo(image.dtype)
        val = np.trunc(np.clip(val, info.min, info.max))
    out = val.astype(image.dtype)
    nn = [np.floor(c + 0.5).astype(int) for c in g]
    ins = [(c >= -0.5) & (c < n - 0.5) for c, n in zip(g, mask.shape[::-1])]
    mz, my, mx = np.meshgrid(nn[2], nn[1], nn[0], indexing="ij")
    iz, iy, ix = np.meshgrid(ins[2], ins[1], ins[0], indexing="ij")
    m = np.where(iz & iy & ix, mask[np.clip(mz, 0, mask.shape[0] - 1), np.clip(my, 0, mask.shape[1] - 1), np.clip(mx, 0, mask.shape[2] - 1)], 0)
    return out, m.astype(mask.dtype), new


# ---------------------------------------------------------------------------------------------------------------------
# ITK's own B-spline machinery, restated line for line (the SciPy path above pins the baseline; this one is what the CUDA
# resampler computes, so a kernel test can compare at rounding level instead of allowing off-by-one integers).
POLE = np.sqrt(3.0) - 2.0
HORIZON = 18                      # ceil(log(1e-10) / log|pole|): ITK's truncated causal start


def _bspline_lines(c, exact):
    """in place on c (lines, N): gain 6, causal start, causal recursion, ITK's anti-causal start, anti-causal recursion"""
    N = c.shape[1]
    if N == 1:
        return
    z = POLE
    c *= 6.0
    if not exact and HORIZON < N:
        zn, s = z, c[:, 0].copy()
        for n in range(1, HORIZON):
            s += zn * c[:, n]
            zn *= z
        c[:, 0] = s
    else:                                      # closed-form mirror sum (every length when exact, short lines otherwise)
        iz = 1.0 / z
        zn, z2n = z, z ** (N - 1)
        s = c[:, 0] + z2n * c[:, N - 1]
        z2n *= z2n * iz
        for n in range(1, N - 1):
            s += (zn + z2n) * c[:, n]
            zn *= z
            z2n *= iz
        c[:, 0] = s / (1.0 - zn * zn)
    for n in range(1, N):
        c[:, n] += z * c[:, n - 1]
    c[:, N - 1] = (z / (z * z - 1.0)) * (z * c[:, N - 2] + c[:, N - 1])
    for n in range(N - 2, -1, -1):
        c[:, n] = z * (c[:, n + 1] - c[:, n])


def bspline_coefficients(x, exact=False):
    """cubic B-spline coefficients of a (Z, Y, X) volume, mirror boundaries, like ITK's BSplineDecompositionImageFilter:
    x first, then y, then z.  exact=False: ITK's causal start, summed over HORIZON samples once a line is longer;
    exact=True: the closed-form mirror sum for every length (= scipy.ndimage.spline_filter(mode="mirror"))."""
    c = np.array(x, dtype=np.float64)
    for ax in (2, 1, 0):
        v = np.moveaxis(c, ax, -1)
        lines = np.ascontiguousarray(v).reshape(-1, v.shape[-1])
        _bspline_lines(lines, exact)
        c = np.moveaxis(lines.reshape(v.shape), -1, ax)
    return np.ascontiguousarray(c)


def _mirror(i, n):
    if n == 1:
        return np.zeros_like(i)
    period = 2 * n - 2
    i = np.abs(i) % period
    return np.where(i >= n, period - i, i)


def _axis_taps(coord, n, interp, dtype):
    """(indices (m, K), weights (m, K)) of one axis for the output coordinates `coord` (m,)"""
    c = coord.astype(dtype)
    f = np.floor(c)
    w = c - f
    fi = f.astype(np.int64)
    if interp == 0:                           # ITK's RoundHalfIntegerUp, clamped to the buffer
        return np.clip(np.floor(c + 0.5).astype(np.int64), 0, n - 1)[:, None], np.ones((c.size, 1), dtype)
    if interp == 1:
        return np.clip(np.stack([fi, fi + 1], 1), 0, n - 1), np.stack([1 - w, w], 1)
    w3 = w * w * w / 6
    w0 = 1 / dtype(6) + w * (w - 1) / 2 - w3
    w2 = w + w0 - 2 * w3
    w1 = 1 - w0 - w2 - w3
    return _mirror(fi[:, None] - 1 + np.arange(4), n), np.stack([w0, w1, w2, w3], 1)


def evaluate(src, out_size_zyx, start_zyx, step_zyx, interp, default_value=0.0, dtype=np.float64):
    """the resampler's value at every output voxel, before the cast: continuous input index start + k * step per axis,
    ITK's IsInsideBuffer ([-0.5, n - 0.5) on every axis, else `default_value`); `src` = the B-spline coefficients for
    interp 3, the image for 1 (linear, neighbours clamped) and 0 (nearest, round half up).  `dtype` = the arithmetic
    (np.longdouble bounds the rounding of the float64 one)."""
    src = np.asarray(src).astype(dtype)
    taps = []
    inside = []
    for d in range(3):
        coord = start_zyx[d] + step_zyx[d] * np.arange(out_size_zyx[d], dtype=np.float64)
        taps.append(_axis_taps(coord, src.shape[d], interp, dtype))
        inside.append((coord >= -0.5) & (coord < src.shape[d] - 0.5))
    (iz, wz), (iy, wy), (ix, wx) = taps
    t = (src[:, :, ix] * wx).sum(-1)                                    # (Z, Y, ox)
    t = (t[:, iy] * wy[None, :, :, None]).sum(2)                        # (Z, oy, ox)
    t = (t[iz] * wz[:, :, None, None]).sum(1)                           # (oz, oy, ox)
    keep = inside[0][:, None, None] & inside[1][None, :, None] & inside[2][None, None, :]
    return np.where(keep, t, dtype(default_value))


def cast(v, dtype):
    """ITK's CastPixelWithBoundsChecking: clamp to the pixel type's range, then truncate; floats are rounded"""
    dtype = np.dtype(dtype)
    if not np.issubdtype(dtype, np.integer):
        return np.asarray(v).astype(dtype)
    info = np.iinfo(dtype)
    hi = float(info.max)
    if hi > info.max:                         # 64-bit types: 2^63 / 2^64 do not fit, clamp to the largest double below
        hi = np.nextafter(hi, 0.0)
    return np.trunc(np.clip(v, float(info.min), hi)).astype(dtype)


def resample_itk(image, mask, spacing_xyz, new_spacing_xyz, padDistance=5, label=1, order=3):
    """`resample` with ITK's truncated causal start and the kernel's own evaluation: (image values before the cast,
    image cast to its dtype, mask, new spacing).  Nearest-neighbour for the mask, as above."""
    image = np.asarray(image)
    newSize, start, step, new = grid(mask, spacing_xyz, new_spacing_xyz, padDistance, label)
    osz, st, sp = tuple(newSize[::-1]), tuple(start[::-1]), tuple(step[::-1])
    src = bspline_coefficients(image) if order == 3 else image.astype(np.float64)
    val = evaluate(src, osz, st, sp, order)
    m = evaluate(np.asarray(mask), osz, st, sp, 0).astype(np.asarray(mask).dtype)
    return val, cast(val, image.dtype), m, new
