"""CPU check of the first-order full-window body (stable ranks from pair compares, a scatter into strided scratch, level
classes from the equality masks) against the generic per-voxel math firstorder_voxel<27> (insertion sort, first-
occurrence level compaction) on the same 27-voxel windows, both compiled for the host from csrc/firstorder.cuh with the
same flags: every feature bit for bit, the sign of zero included."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
INT_RANGES = {"int16": (-32768, 32767), "int32": (-2**31, 2**31 - 1), "uint8": (0, 255), "uint16": (0, 65535),
              "int64": (-2**63, 2**63 - 1)}


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(HERE, "host_emul", "libfirstorder_full_emul.so")
    src = os.path.join(HERE, "host_emul", "firstorder_full_emul.cpp")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so + ".%d" % os.getpid(), src])
    os.replace(so + ".%d" % os.getpid(), so)
    return C.CDLL(so)


def _run(emul, x, w, body, shift, vv):
    out = np.zeros(18)
    x = np.ascontiguousarray(x, dtype=np.float64)
    w = np.ascontiguousarray(w, dtype=np.uint16)
    assert emul.emul_firstorder_window(x.ctypes.data_as(C.c_void_p), w.ctypes.data_as(C.c_void_p), body,
                                       C.c_double(shift), C.c_double(vv), out.ctypes.data_as(C.c_void_p)) == 0
    return out


def signed_zero_windows(rng):
    """-0.0 and +0.0 in both orders, with k values below and m above them so that the minimum, a percentile (sorted
    positions 2-3, 6-7, 13, 19-20, 23-24) or the maximum falls on a zero"""
    out = []
    for below in (0, 2, 3, 6, 7, 13, 19, 20, 23, 24, 25):
        for nz in (2, 3, 27 - below):
            nz = min(nz, 27 - below)
            if nz < 2:
                continue
            for first_neg in (True, False):
                z = np.where(np.arange(nz) % 2 == (0 if first_neg else 1), -0.0, 0.0)
                v = np.concatenate([-rng.integers(1, 50, below).astype(float), z, rng.integers(1, 50, 27 - below - nz) * 1.0])
                out.append(v)
                out.append(v[rng.permutation(27)])
    out.append(np.full(27, -0.0))
    out.append(np.full(27, 0.0))
    return out


def special_windows(rng):
    out = [np.full(27, 7.0), np.full(27, -3.25), np.full(27, 1e300), np.arange(27.0), -np.arange(27.0)[::-1],
           rng.permutation(np.arange(27.0)), rng.normal(size=27)]
    out += [rng.integers(0, 3, 27).astype(float) for _ in range(20)]              # many ties
    out += [rng.choice([-1.0, 1.0, 5.0], 27) for _ in range(10)]
    # large magnitudes that cancel in the sums and moments
    for big in (1e17, 1e154, 1e300):
        v = np.concatenate([np.full(13, big), np.full(13, -big), [1.0]])
        out += [v, v[rng.permutation(27)], v + rng.normal(size=27)]
    out.append(np.concatenate([np.full(26, 1e16), [1.0]]))
    out.append(np.array([np.inf, -np.inf] + [0.0] * 25))                            # infinities (not NaN: full windows)
    out.append(np.array([np.inf] * 27))
    for lo, hi in INT_RANGES.values():
        out.append(rng.integers(lo, hi, 27, endpoint=True).astype(np.float64))
        out.append(np.array([lo, hi] * 13 + [lo], dtype=np.float64))
        out.append(np.where(rng.random(27) < 0.5, lo, hi).astype(np.float64))
    return out + signed_zero_windows(rng)


def level_windows(rng, x):
    """levels for the intensities x: 1 to 27 distinct classes, in shuffled and in sorted-by-value order"""
    out = []
    for k in range(1, 28):
        w = np.concatenate([np.arange(1, k + 1), rng.integers(1, k + 1, 27 - k)])
        out.append(rng.permutation(w))
    ranks = np.argsort(np.argsort(x, kind="stable"), kind="stable")
    out.append(1 + ranks // 3)                                                       # binned like an image
    out.append(np.full(27, 255))
    out.append(np.full(27, 65535))
    return out


def _equal(a, b):
    return np.array_equal(a.view(np.uint64), b.view(np.uint64))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_full_window_body_equals_generic_math_bit_for_bit(emul, seed):
    rng = np.random.default_rng(900 + seed)
    wins = special_windows(rng) + [rng.normal(0, 10.0 ** rng.integers(-3, 6), 27) for _ in range(150)]
    wins += [np.round(rng.normal(0, 4, 27)) for _ in range(150)]                     # integer images: ties
    n = 0
    for i, x in enumerate(wins):
        for w in level_windows(rng, x)[i % 5::5]:
            for shift, vv in ((0.0, 1.0), (1000.0, 0.3), (-2.5, 8.0)):
                gen = _run(emul, x, w, 0, shift, vv)
                full = _run(emul, x, w, 1, shift, vv)
                assert _equal(gen, full), (i, x.tolist(), w.tolist(), shift, gen, full)
                n += 1
    assert n > 3000


def test_signed_zero_lands_where_the_stable_order_puts_it(emul):
    """the generic sort keeps window order among equal values: a window starting -0.0, +0.0 has Minimum -0.0, one
    starting +0.0, -0.0 has Minimum +0.0 -- the full-window body reproduces both"""
    w = np.arange(1, 28)
    for first, sign in ((-0.0, True), (0.0, False)):
        x = np.concatenate([[first, -first], np.arange(1.0, 26.0)])
        for body in (0, 1):
            out = _run(emul, x, w, body, 0.0, 1.0)
            assert out[10] == 0 and np.signbit(out[10]) == sign
