"""Drop-in replacement of ``radiomics.cMatrices`` (the reference's ``_cmatrices`` C extension):
the same six positional signatures, return shapes / dtypes / angle order and exception types
(reference radiomics/src/_cmatrices.c:41-50, 104, 255, 450, 601, 749, 892), executed by the CUDA
kernels behind the C ABI of include/b200radiomics.h.  Install with
``pyradiomics_b200.install()`` or assign it to ``radiomics.<class module>.cMatrices``.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import check, lib, ptr, stream


def _arrays(image, mask):
    # same coercions as try_parse_arrays (_cmatrices.c:1023-1085): FORCECAST to int32 / bool
    img = np.ascontiguousarray(np.asarray(image).astype(np.int32, copy=False))
    msk = np.ascontiguousarray(np.asarray(mask).astype(np.bool_, copy=False)).view(np.uint8)
    if img.ndim != msk.ndim:
        raise ValueError("Expected image and mask to have equal number of dimensions.")
    if img.shape != msk.shape:
        raise ValueError("Dimensions of image and mask do not match.")
    if img.ndim not in (2, 3):
        raise ValueError("pyradiomics_b200 handles 2-D and 3-D arrays")
    return img, msk, np.array(img.shape, dtype=np.int32)


def _voxels(voxels, nd, kernelRadius):
    if voxels is None:
        return None, 1
    if kernelRadius <= 0:
        raise RuntimeError("Expecting kernelRadius > 0")
    v = np.ascontiguousarray(np.asarray(voxels).astype(np.int32, copy=False))
    if v.ndim != 2 or v.shape[0] != nd:
        raise RuntimeError("Expecting voxel indices array to be 2-dimensional")
    return v, int(v.shape[1])


def _distances(distances):
    d = np.ascontiguousarray(np.asarray(distances).astype(np.int32, copy=False))
    if d.ndim != 1:
        raise ValueError("Expecting distances array to be 1-dimensional.")
    return d


def generate_angles(size, distances, bidirectional, force2D, force2Ddimension):
    size = np.ascontiguousarray(np.asarray(size).astype(np.int32, copy=False))
    if size.ndim != 1:
        raise ValueError("Expected a 1D array for size")
    d = _distances(distances)
    nd = int(size.shape[0])
    cap = max(1, (2 * int(d.max()) + 1) ** nd) if d.size else 1
    buf = np.empty((cap, nd), dtype=np.int32)
    na = lib().rb_generate_angles(ptr(size), nd, ptr(d), int(d.size), int(bool(bidirectional)), int(bool(force2D)),
                                  int(force2Ddimension), ptr(buf), cap)
    if na <= 0:
        raise RuntimeError("Error getting angle count.")
    return buf[:na].copy()


def calculate_glcm(image, mask, distances, Ng, force2D, force2Ddimension, kernelRadius=0, voxels=None):
    img, msk, size = _arrays(image, mask)
    d = _distances(distances)
    ang = generate_angles(size, d, 0, force2D, force2Ddimension)
    v, nvox = _voxels(voxels, img.ndim, kernelRadius)
    out = np.empty((nvox, Ng, Ng, ang.shape[0]), dtype=np.float64)
    check(lib().rb_calculate_glcm(ptr(img), ptr(msk), ptr(size), img.ndim, ptr(d), int(d.size), int(Ng), int(bool(force2D)),
                                  int(force2Ddimension), int(kernelRadius), ptr(v), nvox, ptr(out), None), "GLCM")
    return out, ang


def calculate_glrlm(image, mask, Ng, Nr, force2D, force2Ddimension, kernelRadius=0, voxels=None):
    img, msk, size = _arrays(image, mask)
    ang = generate_angles(size, [1], 0, force2D, force2Ddimension)
    v, nvox = _voxels(voxels, img.ndim, kernelRadius)
    out = np.empty((nvox, Ng, int(Nr), ang.shape[0]), dtype=np.float64)
    check(lib().rb_calculate_glrlm(ptr(img), ptr(msk), ptr(size), img.ndim, int(Ng), int(Nr), int(bool(force2D)),
                                   int(force2Ddimension), int(kernelRadius), ptr(v), nvox, ptr(out), None), "GLRLM")
    return out, ang


def calculate_glszm(image, mask, Ng, Ns, force2D, force2Ddimension, kernelRadius=0, voxels=None):
    img, msk, size = _arrays(image, mask)
    generate_angles(size, [1], 1, force2D, force2Ddimension)   # same RuntimeError as the reference when none
    v, nvox = _voxels(voxels, img.ndim, kernelRadius)
    mx = C.c_int(0)
    handle = C.c_void_p()
    check(lib().rb_calculate_glszm(ptr(img), ptr(msk), ptr(size), img.ndim, int(Ng), int(bool(force2D)),
                                   int(force2Ddimension), int(kernelRadius), ptr(v), nvox, C.byref(mx), C.byref(handle)),
          "GLSZM")
    max_region = max(1, mx.value)
    out = np.empty((nvox, Ng, max_region), dtype=np.float64)
    check(lib().rb_fill_glszm(handle, int(Ng), max_region, ptr(out)), "GLSZM")
    return out


def calculate_ngtdm(image, mask, distances, Ng, force2D, force2Ddimension, kernelRadius=0, voxels=None):
    img, msk, size = _arrays(image, mask)
    d = _distances(distances)
    generate_angles(size, d, 1, force2D, force2Ddimension)
    v, nvox = _voxels(voxels, img.ndim, kernelRadius)
    out = np.empty((nvox, Ng, 3), dtype=np.float64)
    check(lib().rb_calculate_ngtdm(ptr(img), ptr(msk), ptr(size), img.ndim, ptr(d), int(d.size), int(Ng), int(bool(force2D)),
                                   int(force2Ddimension), int(kernelRadius), ptr(v), nvox, ptr(out)), "NGTDM")
    return out


def calculate_gldm(image, mask, distances, Ng, alpha, force2D, force2Ddimension, kernelRadius=0, voxels=None):
    img, msk, size = _arrays(image, mask)
    d = _distances(distances)
    ang = generate_angles(size, d, 1, force2D, force2Ddimension)
    v, nvox = _voxels(voxels, img.ndim, kernelRadius)
    out = np.empty((nvox, Ng, 2 * ang.shape[0] + 1), dtype=np.float64)
    check(lib().rb_calculate_gldm(ptr(img), ptr(msk), ptr(size), img.ndim, ptr(d), int(d.size), int(Ng), int(alpha),
                                  int(bool(force2D)), int(force2Ddimension), int(kernelRadius), ptr(v), nvox, ptr(out)),
          "GLDM")
    return out


# ---------------------------------------------------------------------------------------------------------------------
# Device-resident variants: the same matrices from a packed level volume that is already on the GPU (a CUDA tensor from
# rb_pack_levels_dev) -- what the plugin classes use in segment-based mode, so the discretised image never returns to
# the host (the reference hands cMatrices the host array it binned in Python, radiomics/glcm.py:145 etc.).  They run on
# torch's current stream, the one the levels were written on.
def _dev_args(levels):
    import torch
    assert isinstance(levels, torch.Tensor) and levels.is_cuda and levels.is_contiguous() and levels.ndim in (2, 3)
    size = np.array(levels.shape, dtype=np.int32)
    lb = 1 if levels.dtype == torch.uint8 else 2
    return levels.data_ptr(), lb, size


def segment_texture_device(levels, distances, Ng, alpha, force2D, force2Ddimension, glcm=True, gldm=True, ngtdm=True):
    """GLCM, GLDM and NGTDM of one ROI in ONE pass over the device-resident level volume (rb_segment_texture_dev):
    {"glcm": (P [1,Ng,Ng,Na], angles), "gldm": P [1,Ng,2*Na_bi+1], "ngtdm": P [1,Ng,3]} for the requested ones"""
    lev, lb, size = _dev_args(levels)
    d = _distances(distances)
    ang = generate_angles(size, d, 0, force2D, force2Ddimension)
    ang_bi = generate_angles(size, d, 1, force2D, force2Ddimension)
    out = {}
    P_glcm = np.empty((1, Ng, Ng, ang.shape[0]), dtype=np.float64) if glcm else None
    P_gldm = np.empty((1, Ng, 2 * ang_bi.shape[0] + 1), dtype=np.float64) if gldm else None
    P_ngtdm = np.empty((1, Ng, 3), dtype=np.float64) if ngtdm else None
    check(lib().rb_segment_texture_dev(lev, lb, ptr(size), int(size.size), ptr(d), int(d.size), int(Ng), int(alpha), int(bool(force2D)),
                                       int(force2Ddimension), ptr(P_glcm), ptr(P_gldm), ptr(P_ngtdm), None, stream()),
          "GLCM/GLDM/NGTDM")
    if glcm:
        out["glcm"] = (P_glcm, ang)
    if gldm:
        out["gldm"] = P_gldm
    if ngtdm:
        out["ngtdm"] = P_ngtdm
    return out


def calculate_glrlm_device(levels, Ng, Nr, force2D, force2Ddimension):
    lev, lb, size = _dev_args(levels)
    ang = generate_angles(size, [1], 0, force2D, force2Ddimension)
    out = np.empty((1, Ng, int(Nr), ang.shape[0]), dtype=np.float64)
    check(lib().rb_segment_glrlm_dev(lev, lb, ptr(size), int(size.size), int(Ng), int(Nr), int(bool(force2D)), int(force2Ddimension),
                                     ptr(out), None, stream()), "GLRLM")
    return out, ang


def calculate_glszm_device(levels, Ng, force2D, force2Ddimension):
    lev, lb, size = _dev_args(levels)
    generate_angles(size, [1], 1, force2D, force2Ddimension)
    mx = C.c_int(0)
    handle = C.c_void_p()
    check(lib().rb_segment_glszm_dev(lev, lb, ptr(size), int(size.size), int(Ng), int(bool(force2D)), int(force2Ddimension),
                                     C.byref(mx), C.byref(handle), stream()), "GLSZM")
    max_region = max(1, mx.value)
    out = np.empty((1, Ng, max_region), dtype=np.float64)
    check(lib().rb_fill_glszm(handle, int(Ng), max_region, ptr(out)), "GLSZM")
    return out
