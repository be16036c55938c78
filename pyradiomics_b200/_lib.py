"""ctypes binding of libb200radiomics.so (include/b200radiomics.h).  There is no fallback: if the
library is missing or a call fails, an exception is raised.

Every function of the header gets its prototype from PROTOTYPES, so ctypes converts each argument to the C type the
header declares (a Python int reaches a `long long` whole, not cut to an `int`) and refuses a value of the wrong kind
with ctypes.ArgumentError.  Callers pass plain ints, floats, ptr(...) and stream()."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
# B200_RADIOMICS_LIB: developer override to A/B a differently-compiled build of the same library
LIB_PATH = os.environ.get("B200_RADIOMICS_LIB") or os.path.join(HERE, "libb200radiomics.so")

RB_OK, RB_ERR_CUDA, RB_ERR_LEVEL_RANGE, RB_ERR_ARG, RB_ERR_NOMEM, RB_ERR_UNSUPPORTED = 0, -1, -2, -3, -4, -5
CLASSES = ("glcm", "glrlm", "glszm", "gldm", "ngtdm")
CLASS_ID = {n: i for i, n in enumerate(CLASSES)}
WEIGHTING = {None: 0, "infinity": 1, "euclidean": 2, "manhattan": 3, "no_weighting": 4}
ALIVE_WORDS = 6


class VoxelSettings(C.Structure):
    _fields_ = [
        ("kernelRadius", C.c_int), ("force2D", C.c_int), ("force2Ddimension", C.c_int),
        ("ndist", C.c_int), ("distances", C.c_int * 8), ("symmetricalGLCM", C.c_int),
        ("weighting", C.c_int), ("spacing_zyx", C.c_double * 3), ("gldm_a", C.c_int),
        ("initValue", C.c_double), ("Ng", C.c_int), ("n_roi_levels", C.c_int),
    ]


class B200Error(RuntimeError):
    pass


# rb_dtype: the pixel types the device code reads, code = position in this tuple
DTYPE_CODE = {np.dtype(n): code for code, n in enumerate(("int16", "int32", "float32", "float64", "uint8", "uint16", "int64"))}
# the torch dtypes the device path takes (a uint16 image travels as int32) and their NumPy scalar types
NP_OF_TORCH = {torch.int16: np.int16, torch.int32: np.int32, torch.float32: np.float32, torch.float64: np.float64,
               torch.uint8: np.uint8, torch.int64: np.int64}
TORCH_OF_NP = {n: t for t, n in NP_OF_TORCH.items()}
TORCH_DTYPE_CODE = {t: DTYPE_CODE[np.dtype(n)] for t, n in NP_OF_TORCH.items()}


def ptr(x):
    """data address of a torch tensor or an ndarray, None for None (NULL)"""
    if x is None:
        return None
    return x.data_ptr() if isinstance(x, torch.Tensor) else x.ctypes.data


def stream():
    """the current CUDA stream, as the `void *stream` argument"""
    return torch.cuda.current_stream().cuda_stream


# (restype, argtypes) of every function of include/b200radiomics.h: every data pointer is c_void_p, a settings pointer
# POINTER(VoxelSettings), a `const char *` result c_char_p
_i, _ll, _ull, _d, _p, _s = C.c_int, C.c_longlong, C.c_ulonglong, C.c_double, C.c_void_p, C.c_char_p
_SET = C.POINTER(VoxelSettings)
PROTOTYPES = {
    "rb_last_error": (_s, []),
    "rb_version": (_s, []),
    "rb_device_count": (_i, []),
    "rb_num_features": (_i, [_i]),
    "rb_release_device_caches": (_i, []),
    "rb_feature_name": (_s, [_i, _i]),
    "rb_generate_angles": (_i, [_p, _i, _p, _i, _i, _i, _i, _p, _i]),
    "rb_level_bytes": (_i, [_i]),
    "rb_pack_levels_dev": (_i, [_p, _p, _ll, _i, _p, _p, _p, _p]),
    "rb_glcm_alive_angles_dev": (_i, [_p, _i, _p, _i, _i, _i, _SET, _p, _p]),
    "rb_voxel_features_dev": (_i, [_i, _p, _i, _p, _i, _i, _i, _i, _i, _SET, _p, _p, _i, _ll, _i, _p, _p]),
    "rb_memcpy2d_async": (_i, [_p, _ull, _p, _ull, _ull, _ull, _i, _p]),
    "rb_maps_to_f32_dev": (_i, [_p, _ll, _p, _ll, _ll, _ll, _p]),
    "rb_voxel_features_host": (_i, [_i, _p, _p, _i, _i, _i, _SET, _p]),
    "rb_calculate_glcm": (_i, [_p, _p, _p, _i, _p, _i, _i, _i, _i, _i, _p, _i, _p, _p]),
    "rb_calculate_glrlm": (_i, [_p, _p, _p, _i, _i, _i, _i, _i, _i, _p, _i, _p, _p]),
    "rb_calculate_gldm": (_i, [_p, _p, _p, _i, _p, _i, _i, _i, _i, _i, _i, _p, _i, _p]),
    "rb_calculate_ngtdm": (_i, [_p, _p, _p, _i, _p, _i, _i, _i, _i, _i, _p, _i, _p]),
    "rb_calculate_glszm": (_i, [_p, _p, _p, _i, _i, _i, _i, _i, _p, _i, _p, _p]),
    "rb_fill_glszm": (_i, [_p, _i, _i, _p]),
    "rb_glszm_release": (None, [_p]),
    "rb_segment_texture_dev": (_i, [_p, _i, _p, _i, _p, _i, _i, _i, _i, _i, _p, _p, _p, _p, _p]),
    "rb_segment_glrlm_dev": (_i, [_p, _i, _p, _i, _i, _i, _i, _i, _p, _p, _p]),
    "rb_segment_glszm_dev": (_i, [_p, _i, _p, _i, _i, _i, _i, _p, _p, _p]),
    "rb_minmax_dev": (_i, [_p, _i, _p, _ll, _p, _p]),
    "rb_digitize_dev": (_i, [_p, _i, _p, _ll, _p, _i, _p, _p]),
    "rb_swt_axis_dev": (_i, [_p, _i, _i, _i, _i, _p, _p, _i, _p, _p, _p]),
    "rb_swt3d_dev": (_i, [_p, _i, _i, _i, _p, _p, _i, _p, _ll, _i, _i, _p]),
    "rb_recursive_gaussian_axis_dev": (_i, [_p, _i, _i, _i, _i, _i, _p, _p, _p, _d, _i, _p]),
    "rb_bspline_prefilter_dev": (_i, [_p, _i, _i, _i, _p]),
    "rb_resample_dev": (_i, [_p, _i, _p, _p, _i, _p, _p, _p, _i, _d, _p]),
    "rb_lbp3d_dev": (_i, [_p, _i, _i, _p, _i, _i, _i, _p, _i, _p, _i, _p, _p, _p]),
    "rb_lbp2d_dev": (_i, [_p, _i, _i, _i, _i, _i, _i, _p, _p, _i, _p, _p]),
    "rb_lbp2d_cast_dev": (_i, [_p, _i, _i, _i, _i, _i, _i, _p, _p, _i, _p, _p]),
    "rb_pointwise_image_dev": (_i, [_p, _i, _ll, _i, _d, _p, _p]),
    "rb_gradient_magnitude_dev": (_i, [_p, _i, _i, _i, _i, _p, _p, _p]),
    "rb_roi_moments_dev": (_i, [_p, _i, _p, _ll, _i, _p, _p, _p]),
    "rb_normalize_dev": (_i, [_p, _i, _ll, _d, _d, _i, _d, _d, _p, _p]),
    "rb_resegment_dev": (_i, [_p, _i, _p, _ll, _d, _d, _i, _p, _p, _p]),
    "rb_calculate_coefficients": (_i, [_p, _p, _p, _p, _p, _p, _p]),
    "rb_shape_coefficients_dev": (_i, [_p, _i, _i, _i, _p, _p, _p]),
    "rb_shape_moments_dev": (_i, [_p, _i, _i, _i, _p, _p]),
    "rb_calculate_coefficients2D": (_i, [_p, _p, _p, _p, _p, _p, _p]),
    "rb_firstorder_num_features": (_i, []),
    "rb_firstorder_feature_name": (_s, [_i]),
    "rb_firstorder_voxel_dev": (_i, [_p, _i, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _d, _d, _d, _p, _ll, _i, _i, _i, _p]),
    "rb_firstorder_segment_dev": (_i, [_p, _i, _p, _p, _i, _i, _i, _i, _d, _d, _p, _p]),
}

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B200Error(
                f"{LIB_PATH} is not built -- run `python -m pyradiomics_b200.build` (needs nvcc); "
                "pyradiomics_b200 has no CPU fallback")
        L = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in PROTOTYPES.items():
            f = getattr(L, name)
            f.restype, f.argtypes = restype, argtypes
        _lib = L
    return _lib


def check(rc, what=""):
    """Map rb_status to the exception types the reference binding raises
    (reference radiomics/src/_cmatrices.c:159,219,1045,1079,1093)."""
    if rc >= 0:
        return rc
    msg = (lib().rb_last_error() or b"").decode()
    if rc == RB_ERR_LEVEL_RANGE:
        raise IndexError(f"Calculation of {what or 'matrix'} Failed. ({msg})")
    if rc == RB_ERR_ARG:
        raise ValueError(msg)
    if rc == RB_ERR_NOMEM:
        raise MemoryError(msg)
    raise B200Error(f"{what}: rb_status {rc}: {msg}")


def feature_names(cls):
    """the map order of a voxel class's kernel: one of CLASSES (or its id) or "firstorder\""""
    L = lib()
    if cls == "firstorder":
        return [L.rb_firstorder_feature_name(i).decode() for i in range(L.rb_firstorder_num_features())]
    cid = CLASS_ID[cls] if isinstance(cls, str) else cls
    return [L.rb_feature_name(cid, i).decode() for i in range(L.rb_num_features(cid))]


def make_settings(Ng, n_roi_levels, **kw):
    s = VoxelSettings()
    s.kernelRadius = int(kw.get("kernelRadius", 1))
    s.force2D = int(bool(kw.get("force2D", False)))
    s.force2Ddimension = int(kw.get("force2Ddimension", 0))
    d = [int(x) for x in kw.get("distances", [1])]
    if not 1 <= len(d) <= 8:
        raise ValueError("1..8 distances supported")
    s.ndist = len(d)
    for i, v in enumerate(d):
        s.distances[i] = v
    s.symmetricalGLCM = int(bool(kw.get("symmetricalGLCM", True)))
    wn = kw.get("weightingNorm")
    s.weighting = WEIGHTING.get(wn, 4)  # unknown names weigh 1 like the reference (glcm.py:176-181)
    sp = kw.get("spacing_zyx", (1.0, 1.0, 1.0))
    for i in range(3):
        s.spacing_zyx[i] = float(sp[i])
    s.gldm_a = int(kw.get("gldm_a", 0))
    s.initValue = float(kw.get("initValue", 0))
    s.Ng = int(Ng)
    s.n_roi_levels = int(n_roi_levels)
    return s
