"""CPU checks of the generic voxel kernel at its capacity limits, through the host-compiled device math
(tests/host_emul/emul.cpp compiles pyradiomics_b200/csrc/vox_features.cuh, the header the CUDA kernel runs, with g++).

* MCC: the dense eigen-solve holds 32 row levels (NJCAP).  r = 2 and r = 3 windows of i.i.d. levels hold more; the MCC
  of such a voxel is NaN and the run's status has bit 0 set -- never the mean over its remaining angles.
* Weighted GLCM: every angle pools into one entry list of 2048 entries; a window with more distinct pairs fails the run
  (status bit 1)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cmatrices_oracle as O
import pipeline as PL
from helpers import alive_mask_bruteforce, assert_maps_close, envelope_volume, mcc_over_capacity
from pyradiomics_b200 import _lib
from test_host_emul import NAMES

HERE = os.path.dirname(os.path.abspath(__file__))
SPACING_ZYX = (2.0, 0.7, 1.0)
CASES = [(r, n, False) for r in (2, 3) for n in (24, 36, 48, 64)] + [(2, 48, True), (3, 48, True)]


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(HERE, "host_emul", "libemul_envelope.so")
    src = os.path.join(HERE, "host_emul", "emul.cpp")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so + ".%d" % os.getpid(), src])
    os.replace(so + ".%d" % os.getpid(), so)
    return C.CDLL(so)


def _emul_maps(emul, cname, lev, s, alive=None):
    """(maps [F, Z, Y, X], status word) of one class; the ROI is lev != 0"""
    lev16 = np.ascontiguousarray(lev, dtype=np.uint16)
    out = np.zeros((len(NAMES[cname]),) + lev.shape)
    rc = emul.emul_voxel_features(_lib.CLASS_ID[cname], lev16.ctypes.data_as(C.c_void_p), None, *lev.shape, C.byref(s),
                                  None if alive is None else alive.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
    assert rc >= 0, rc
    return out, rc


def _check_mcc(got, ref, over, what):
    """NaN exactly on the over-capacity voxels, the oracle's value everywhere else"""
    finite_wrong = int(np.sum(over & np.isfinite(got)))
    assert finite_wrong == 0, f"{what}: {finite_wrong} over-capacity voxels hold a finite MCC"
    assert not np.isnan(got[~over]).any(), f"{what}: NaN MCC outside the over-capacity voxels"
    assert_maps_close(got, np.where(over, np.nan, ref), what, rtol=1e-7, atol=1e-9)


@pytest.mark.parametrize("r,n_levels,holes", CASES, ids=[f"r{r}-L{n}" + ("-holes" if h else "") for r, n, h in CASES])
def test_generic_math_beyond_the_mcc_capacity(emul, r, n_levels, holes):
    lev = envelope_volume(n_levels, holes)
    mask = lev != 0
    s = _lib.make_settings(n_levels, n_levels, kernelRadius=r)
    alive = alive_mask_bruteforce(lev, mask, O.generate_angles(lev.shape, [1], 0, False, 0), [r] * 3)
    over = mcc_over_capacity(lev, mask, r)
    assert over.any() == (n_levels > 32), "the volume does not probe the limit it is meant to"
    for cname in _lib.CLASSES:
        out, st = _emul_maps(emul, cname, lev, s, alive if cname == "glcm" else None)
        ref = PL.extract(cname, lev, mask, voxelBased=True, binWidth=1, kernelRadius=r)
        assert st == (int(over.any()) if cname == "glcm" else 0), st
        for k, f in enumerate(NAMES[cname]):
            what = f"r{r}/L{n_levels}/{cname}/{f}"
            if f == "MCC":
                _check_mcc(out[k][mask], ref[f], over, what)
            else:
                assert_maps_close(out[k][mask], ref[f], what, rtol=1e-7, atol=1e-9)


@pytest.mark.parametrize("r,n_levels", [(3, 32), (2, 64), (3, 64)])
def test_weighted_glcm_pooled_matrix_limits(emul, r, n_levels):
    """euclidean weights on anisotropic spacing: r = 3 with 32 levels fits (MCC included); r = 2 with 64 levels fits
    the entry list but not the MCC solve (NaN where the pooled matrix is over capacity); r = 3 with 64 levels has windows
    with more than 2048 distinct pairs and fails loudly"""
    lev = envelope_volume(n_levels)
    mask = lev != 0
    kw = dict(kernelRadius=r, weightingNorm="euclidean")
    out, st = _emul_maps(emul, "glcm", lev, _lib.make_settings(n_levels, n_levels, spacing_zyx=SPACING_ZYX, **kw))
    if (r, n_levels) == (3, 64):
        assert st & 2, st
        return
    over = mcc_over_capacity(lev, mask, r, spacing_zyx=SPACING_ZYX, weightingNorm="euclidean")
    assert over.any() == (n_levels > 32)
    assert st == int(over.any()), st
    ref = PL.extract("glcm", lev, mask, voxelBased=True, binWidth=1, spacing_zyx=SPACING_ZYX, **kw)
    for k, f in enumerate(NAMES["glcm"]):
        what = f"weighted/r{r}/L{n_levels}/{f}"
        if f == "MCC":
            _check_mcc(out[k][mask], ref[f], over, what)
        else:
            assert_maps_close(out[k][mask], ref[f], what, rtol=1e-7, atol=1e-9)
