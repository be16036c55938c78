"""CPU check of GLCM phase A's full-window body (every window level non-zero: no validity logic, constant
denominators) against its general body on the same windows, compiled for the host from the device headers.
Per angle, the quantities that come from integers (the sums, the pair multiplicities behind JointEnergy and
MaximumProbability, the task bit and size class) must be bit-identical; per voxel, every feature agrees to rounding."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from pyradiomics_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
# features that are an integer over a power of S within one angle
EXACT = ("Autocorrelation", "JointAverage", "ClusterTendency", "Contrast", "DifferenceAverage", "DifferenceVariance",
         "JointEnergy", "MaximumProbability", "SumAverage", "SumSquares", "MCC")
NAMES = ["Autocorrelation", "ClusterProminence", "ClusterShade", "ClusterTendency", "Contrast", "Correlation",
         "DifferenceAverage", "DifferenceEntropy", "DifferenceVariance", "Id", "Idm", "Idmn", "Idn", "Imc1", "Imc2",
         "InverseVariance", "JointAverage", "JointEnergy", "JointEntropy", "MCC", "MaximumProbability", "SumAverage",
         "SumEntropy", "SumSquares"]


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(HERE, "host_emul", "libglcm_full_emul.so")
    src = os.path.join(HERE, "host_emul", "glcm_full_emul.cpp")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so + ".%d" % os.getpid(), src])
    os.replace(so + ".%d" % os.getpid(), so)
    lib = C.CDLL(so)
    lib.emul_glcm_angle.restype = C.c_longlong
    lib.emul_glcm_phaseA.restype = C.c_longlong
    return lib


def _full_windows(rng, kind, ng, count):
    if kind == "uniform":
        return rng.integers(1, ng + 1, (count, 27)).astype(np.uint8)
    # smooth: a random linear ramp over the 3x3x3 window plus a little noise, quantised to 1..ng
    zz, yy, xx = np.meshgrid(*[np.arange(3)] * 3, indexing="ij")
    pos = np.stack([zz.ravel(), yy.ravel(), xx.ravel()], 1).astype(float)
    g = rng.normal(size=(count, 3)) * rng.uniform(0.1, 1.5, (count, 1))
    f = g @ pos.T + 0.3 * rng.normal(size=(count, 27)) + rng.uniform(0, ng, (count, 1))
    return np.clip(np.rint(f), 1, ng).astype(np.uint8)


@pytest.mark.parametrize("kind", ["uniform", "smooth"])
@pytest.mark.parametrize("ng", [2, 3, 5, 8, 16, 32])
def test_full_window_body_equals_general_body(emul, kind, ng):
    rng = np.random.default_rng(100 + ng)
    s = _lib.make_settings(ng, ng)
    exact = [NAMES.index(f) for f in EXACT]
    for w in _full_windows(rng, kind, ng, 300):
        wp = np.ascontiguousarray(w).ctypes.data_as(C.c_void_p)
        for slot in range(13):
            a, b = np.zeros(24), np.zeros(24)
            ta, tb = C.c_ulonglong(0), C.c_ulonglong(0)
            ma = emul.emul_glcm_angle(wp, slot, 1, C.byref(s), a.ctypes.data_as(C.c_void_p), C.byref(ta))
            mb = emul.emul_glcm_angle(wp, slot, 0, C.byref(s), b.ctypes.data_as(C.c_void_p), C.byref(tb))
            assert ma >= 0 and (ma, ta.value) == (mb, tb.value), (w, slot)
            assert np.array_equal(a[exact], b[exact]), (w, slot)
            assert np.allclose(a, b, rtol=1e-12, atol=1e-12), (w, slot)
        fa, fb = np.zeros(24), np.zeros(24)
        na, nb = C.c_int(0), C.c_int(0)
        ca, cb = C.c_ulonglong(0), C.c_ulonglong(0)
        ma = emul.emul_glcm_phaseA(wp, 1, C.byref(s), fa.ctypes.data_as(C.c_void_p), C.byref(na), C.byref(ca))
        mb = emul.emul_glcm_phaseA(wp, 0, C.byref(s), fb.ctypes.data_as(C.c_void_p), C.byref(nb), C.byref(cb))
        assert ma >= 0 and (ma, na.value, ca.value) == (mb, nb.value, cb.value) and na.value == 13
        for k, f in enumerate(NAMES):
            atol = 1e-6 if f in ("Imc1", "Imc2") else 1e-9
            assert np.isclose(fa[k], fb[k], rtol=1e-7, atol=atol), (f, w)
