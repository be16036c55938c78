"""Drop-in replacement of ``radiomics.cShape`` (the reference's ``_cshape`` C extension) for the 3-D
path: ``calculate_coefficients(mask, pixelSpacing)`` with the reference's coercions and return value
(radiomics/src/_cshape.c:75-113), executed by the CUDA kernels of csrc/shape.cu behind the C ABI
(``rb_calculate_coefficients``).  ``moments`` exposes the exact integer voxel moments the shape class
builds its covariance from.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import check, lib, ptr, stream

_fallback = None        # the reference's _cshape module, set by featureclasses.install()


def __getattr__(name):
    """names this module does not implement are served by the reference's own extension when install() found one"""
    if _fallback is not None and hasattr(_fallback, name):
        return getattr(_fallback, name)
    raise AttributeError(f"module 'pyradiomics_b200.cshape' has no attribute {name!r}")


def calculate_coefficients(mask, pixelSpacing):
    """(SurfaceArea, Volume, (Maximum2DDiameterSlice, ...Column, ...Row, Maximum3DDiameter))"""
    msk = np.ascontiguousarray(np.asarray(mask).astype(np.int8, copy=False))       # NPY_BYTE | FORCECAST
    sp = np.ascontiguousarray(np.asarray(pixelSpacing).astype(np.float64, copy=False))
    if msk.ndim != 3:
        raise ValueError("Expected a 3D array for mask")                           # check_arrays, _cshape.c:163
    if sp.ndim != 1 or sp.shape[0] != 3:
        raise ValueError("Expecting spacing array to have shape (3,)")
    size = np.array(msk.shape, dtype=np.int32)
    strides = np.array([s // msk.itemsize for s in msk.strides], dtype=np.int32)
    sa, vol = C.c_double(), C.c_double()
    dia = (C.c_double * 4)()
    rc = lib().rb_calculate_coefficients(ptr(msk), ptr(size), ptr(strides), ptr(sp), C.byref(sa), C.byref(vol), dia)
    if rc:
        check(rc, "Calculation of Shape coefficients failed.")
    return sa.value, vol.value, tuple(dia)


def calculate_coefficients2D(mask, pixelSpacing):
    """(Perimeter, Surface, MaximumDiameter) of a 2-D mask: drop-in for the reference's
    ``cShape.calculate_coefficients2D`` (radiomics/src/_cshape.c:33-39, cshape.c:420-595; called at shape2D.py:99)"""
    msk = np.ascontiguousarray(np.asarray(mask).astype(np.int8, copy=False))
    sp = np.ascontiguousarray(np.asarray(pixelSpacing).astype(np.float64, copy=False))
    if msk.ndim != 2:
        raise ValueError("Expected a 2D array for mask")
    if sp.ndim != 1 or sp.shape[0] != 2:
        raise ValueError("Expecting spacing array to have shape (2,)")
    size = np.array(msk.shape, dtype=np.int32)
    strides = np.array([s // msk.itemsize for s in msk.strides], dtype=np.int32)
    per, sur, dia = C.c_double(), C.c_double(), C.c_double()
    rc = lib().rb_calculate_coefficients2D(ptr(msk), ptr(size), ptr(strides), ptr(sp), C.byref(per), C.byref(sur),
                                           C.byref(dia))
    if rc:
        check(rc, "Calculation of Shape coefficients failed.")
    return per.value, sur.value, dia.value


def coefficients_device(mask_t, spacing_zyx):
    """same for a contiguous uint8 CUDA tensor [Z, Y, X]; returns (area, volume, diameters, n_vertices)"""
    sp = (C.c_double * 3)(*[float(s) for s in spacing_zyx])
    out = (C.c_double * 7)()
    Z, Y, X = mask_t.shape
    check(lib().rb_shape_coefficients_dev(ptr(mask_t), Z, Y, X, sp, out, stream()), "shape coefficients")
    return out[0], out[1], tuple(out[2:6]), int(out[6])


def moments_device(mask_t):
    """exact integer sums {N, z, y, x, zz, zy, zx, yy, yx, xx} over the ROI voxels (Python ints)"""
    out = (C.c_ulonglong * 10)()
    Z, Y, X = mask_t.shape
    check(lib().rb_shape_moments_dev(ptr(mask_t), Z, Y, X, out, stream()), "shape moments")
    return [int(v) for v in out]


def covariance_eigenvalues(m, spacing_zyx):
    """eigenvalues (ascending) of the physical-coordinate covariance of the ROI voxels (shape.py:86-106),
    from exact integer moments: cov_ij = (N * S_ij - S_i * S_j) / N^2 * s_i * s_j, numerator exact."""
    n = m[0]
    s1 = m[1:4]
    s2 = {(0, 0): m[4], (0, 1): m[5], (0, 2): m[6], (1, 1): m[7], (1, 2): m[8], (2, 2): m[9]}
    cov = np.zeros((3, 3))
    for i in range(3):
        for j in range(i, 3):
            num = n * s2[(i, j)] - s1[i] * s1[j]                      # Python ints: exact
            cov[i, j] = cov[j, i] = (num / (n * n)) * float(spacing_zyx[i]) * float(spacing_zyx[j])
    ev = np.linalg.eigvals(cov).real
    ev[(ev < 0) & (ev > -1e-10)] = 0
    return np.sort(ev)
