"""No-GPU checks of the C-ABI library: it loads, exports every symbol include/b200radiomics.h
declares, and its host-only entry points (angles, names) agree with the oracle."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import cmatrices_oracle as O
from pyradiomics_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    build.build()
    return _lib.lib()


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "b200radiomics.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(rb_[a-z0-9_]+)\s*\(", hdr)))


def test_library_exports_every_declared_symbol(L):
    syms = declared_symbols()
    assert len(syms) >= 10
    for s in syms:
        assert hasattr(L, s), f"{s} declared in include/b200radiomics.h but not exported"


def test_settings_struct_layout_matches_header():
    # 4 ints + 8 ints + 2 ints (+pad) + 3 doubles + int (+pad) + double + 2 ints
    assert C.sizeof(_lib.VoxelSettings) == 104


def test_feature_names(L):
    from pyradiomics_b200 import _matrix_features as MF, featureclasses as FC
    assert [L.rb_num_features(i) for i in range(5)] == [24, 16, 16, 14, 5]
    assert _lib.feature_names("glcm")[19] == "MCC"
    assert _lib.feature_names("ngtdm") == ["Busyness", "Coarseness", "Complexity", "Contrast", "Strength"]
    # every Python name table lists the features in the order of the library's maps
    tables = {"glcm": MF.GLCM_NAMES, "glrlm": MF.GLRLM_NAMES, "glszm": sorted(MF.GLSZM_NAMES.values()),
              "gldm": sorted(MF.GLDM_NAMES.values()), "ngtdm": MF.NGTDM_NAMES, "firstorder": FC.RadiomicsFirstOrder.NAMES}
    for cls, names in tables.items():
        assert list(names) == _lib.feature_names(cls), cls


@pytest.mark.parametrize("size", [(5, 5, 5), (1, 6, 7), (2, 2, 9), (3, 1, 4), (6, 7), (1, 5)])
@pytest.mark.parametrize("dist", [[1], [1, 2], [2, 3], [3]])
@pytest.mark.parametrize("bidir", [0, 1])
@pytest.mark.parametrize("f2", [(0, 0), (1, 0), (1, 1)])
def test_generate_angles_matches_oracle(L, size, dist, bidir, f2):
    nd = len(size)
    if f2[0] and f2[1] >= nd:
        pytest.skip("dimension out of range")
    sz = np.array(size, np.int32)
    d = np.array(dist, np.int32)
    buf = np.zeros((400, nd), np.int32)
    na = L.rb_generate_angles(sz.ctypes.data_as(C.c_void_p), nd, d.ctypes.data_as(C.c_void_p), len(dist), bidir,
                              f2[0], f2[1], buf.ctypes.data_as(C.c_void_p), 400)
    try:
        ref = O.generate_angles(size, dist, bidir, f2[0], f2[1])
    except RuntimeError:
        assert na == _lib.RB_ERR_ARG
        return
    assert na == ref.shape[0]
    assert np.array_equal(buf[:na], ref)


def test_no_cpu_fallback_without_device(L):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    img = np.ones((3, 3, 3), np.int32)
    msk = np.ones((3, 3, 3), np.uint8)
    out = np.zeros((5, 3, 3, 3))
    s = _lib.make_settings(1, 1)
    rc = L.rb_voxel_features_host(4, img.ctypes.data_as(C.c_void_p), msk.ctypes.data_as(C.c_void_p), 3, 3, 3,
                                  C.byref(s), out.ctypes.data_as(C.c_void_p))
    assert rc in (_lib.RB_ERR_CUDA, _lib.RB_ERR_NOMEM)
