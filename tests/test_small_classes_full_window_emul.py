"""CPU check of the GLSZM and GLDM fast paths' two bodies -- the full-window body (every window level non-zero:
constant counts, no sentinels) and the general one -- against each other and against the generic
per-voxel math on the same windows, compiled for the host from the device headers."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from pyradiomics_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
CLASSES = {"glszm": 16, "gldm": 14}


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(HERE, "host_emul", "libsmall_classes_full_emul.so")
    src = os.path.join(HERE, "host_emul", "small_classes_full_emul.cpp")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so + ".%d" % os.getpid(), src])
    os.replace(so + ".%d" % os.getpid(), so)
    return C.CDLL(so)


def _run(emul, cname, w, body, s):
    out = np.zeros(CLASSES[cname])
    w = np.ascontiguousarray(w, dtype=np.uint8)
    rc = emul.emul_small_class_window(_lib.CLASS_ID[cname], w.ctypes.data_as(C.c_void_p), body, C.byref(s),
                                      out.ctypes.data_as(C.c_void_p))
    assert rc == 0, rc
    return out


def _full_windows(rng, ng):
    wins = [rng.integers(1, ng + 1, 27) for _ in range(300)]
    wins += [rng.integers(1, min(ng, 3) + 1, 27) for _ in range(100)]       # few large classes, large zones
    wins += [np.full(27, ng), np.full(27, 1), np.arange(27) % ng + 1]
    zz, yy, xx = np.meshgrid(range(3), range(3), range(3), indexing="ij")
    wins.append(np.where((zz + yy + xx) % 2 == 0, 1, ng).reshape(27))        # checkerboard: 13 + 14 positions
    for axis in (zz, yy, xx):                                                 # planes: zones of 9
        wins.append((axis.reshape(27) % ng) + 1)
    return [np.clip(w, 1, ng) for w in wins]


@pytest.mark.parametrize("cname", list(CLASSES))
@pytest.mark.parametrize("ng", [2, 5, 32, 255])
def test_full_body_equals_general_body_and_generic_math(emul, cname, ng):
    rng = np.random.default_rng(400 + ng)
    for a in ((0, 1, 3, 255) if cname == "gldm" else (0,)):
        s = _lib.make_settings(ng, ng, gldm_a=a)
        for w in _full_windows(rng, ng):
            full, general, generic = (_run(emul, cname, w, b, s) for b in (1, 0, 2))
            assert np.allclose(full, general, rtol=1e-12, atol=1e-13), (cname, a, w, full, general)
            assert np.allclose(full, generic, rtol=1e-10, atol=1e-12), (cname, a, w, full, generic)


@pytest.mark.parametrize("cname", list(CLASSES))
def test_general_body_with_one_zero_at_each_position_and_with_holes(emul, cname):
    """a single unmasked position at each of the 27 places (the centre stays), then windows with more and more holes
    down to a lone centre, against the generic math"""
    rng = np.random.default_rng(401)
    for a in ((0, 3) if cname == "gldm" else (0,)):
        s = _lib.make_settings(32, 32, gldm_a=a)
        wins = []
        for pos in range(27):
            for _ in range(6):
                w = rng.integers(1, 33 if _ % 2 else 4, 27)
                w[pos] = 0
                w[13] = max(int(w[13]), 1)
                wins.append(w)
        for it in range(300):
            w = rng.integers(1, 33 if it % 2 else 4, 27)
            w[rng.random(27) < (it % 10) / 10] = 0
            w[13] = max(int(w[13]), 1)
            wins.append(w)
        lone = np.zeros(27, int)
        lone[13] = 5
        wins.append(lone)
        for w in wins:
            general, generic = _run(emul, cname, w, 0, s), _run(emul, cname, w, 2, s)
            assert np.array_equal(np.isnan(general), np.isnan(generic)), (cname, w, general, generic)
            ok = ~np.isnan(generic)
            assert np.allclose(general[ok], generic[ok], rtol=1e-10, atol=1e-12), (cname, a, w, general, generic)

