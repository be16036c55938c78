"""CPU check of the NGTDM fast path's full-window body (every window level non-zero: constant neighbour counts, exact
integer differences, Busyness from one sort) against its general body and the generic per-voxel math on the same
windows, compiled for the host from the device headers."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from pyradiomics_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
NAMES = ["Busyness", "Coarseness", "Complexity", "Contrast", "Strength"]


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(HERE, "host_emul", "libngtdm_full_emul.so")
    src = os.path.join(HERE, "host_emul", "ngtdm_full_emul.cpp")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so + ".%d" % os.getpid(), src])
    os.replace(so + ".%d" % os.getpid(), so)
    return C.CDLL(so)


def _run(emul, w, body, s):
    out = np.zeros(5)
    w = np.ascontiguousarray(w, dtype=np.uint8)
    assert emul.emul_ngtdm_window(w.ctypes.data_as(C.c_void_p), body, C.byref(s), out.ctypes.data_as(C.c_void_p)) == 0
    return out


def _special_windows(ng):
    out = [np.full(27, ng), np.full(27, 1)]                       # a single level
    for pos in (0, 1, 4, 13):                                      # the largest numerators: 255 beside 1s
        w = np.ones(27, int)
        w[pos] = ng
        out.append(w)
        out.append(ng + 1 - w)                                     # and 1 beside 255s
    if ng >= 27:
        out.append(np.arange(1, 28))                               # all distinct
        out.append(ng - np.arange(27))
        out.append(np.random.default_rng(ng).permutation(np.arange(ng - 26, ng + 1)))
    for split in (13, 14, 20):                                     # two large classes
        w = np.full(27, ng)
        w[np.random.default_rng(split).permutation(27)[:split]] = 1 + ng // 3
        out.append(w)
    zz, yy, xx = np.meshgrid(range(3), range(3), range(3), indexing="ij")
    out.append(np.where((zz + yy + xx) % 2 == 0, 1, ng).reshape(27))     # checkerboard of extremes
    return [np.clip(w, 1, ng) for w in out]


@pytest.mark.parametrize("ng", [2, 5, 32, 255])
def test_full_window_body_equals_general_body_and_generic_math(emul, ng):
    rng = np.random.default_rng(300 + ng)
    s = _lib.make_settings(ng, ng)
    wins = [rng.integers(1, ng + 1, 27) for _ in range(400)]
    wins += [rng.integers(1, min(ng, 4) + 1, 27) for _ in range(100)]           # few large classes
    wins += _special_windows(ng)
    for w in wins:
        full = _run(emul, w, 1, s)
        general = _run(emul, w, 0, s)
        generic = _run(emul, w, 2, s)
        for k, f in enumerate(NAMES):
            assert np.isclose(full[k], general[k], rtol=1e-12, atol=1e-13), (f, w, full[k], general[k])
            assert np.isclose(full[k], generic[k], rtol=1e-10, atol=1e-12), (f, w, full[k], generic[k])


def test_full_window_conventions(emul):
    """a single-level window: Coarseness 1e6 (sum p s = 0), Busyness and Contrast 0, Strength 0 (sum s = 0)"""
    s = _lib.make_settings(32, 32)
    out = _run(emul, np.full(27, 7), 1, s)
    assert out.tolist() == [0.0, 1e6, 0.0, 0.0, 0.0]


def test_general_body_on_windows_with_holes(emul):
    """the general body (zeros unmasked, counts from the mask) against the generic math, down to a lone centre"""
    rng = np.random.default_rng(301)
    s = _lib.make_settings(32, 32)
    for it in range(600):
        w = rng.integers(1, 33, 27)
        w[rng.random(27) < (it % 10) / 10] = 0
        w[13] = max(int(w[13]), 1)
        general, generic = _run(emul, w, 0, s), _run(emul, w, 2, s)
        assert np.allclose(general, generic, rtol=1e-10, atol=1e-12), (w, general, generic)
    lone = np.zeros(27, int)
    lone[13] = 5
    assert _run(emul, lone, 0, s).tolist() == _run(emul, lone, 2, s).tolist() == [0.0, 1e6, 0.0, 0.0, 0.0]
