"""2-D LBP (getLBP2DImage) without a GPU: the NumPy oracle against the reference's goldens, exact properties of the
restated local_binary_pattern, the CUDA kernel's per-pixel arithmetic (csrc/lbp2d.cuh, compiled with g++ by
tests/host_emul/lbp2d_emul.cpp) against the oracle bit for bit, and the generator's guards."""
import ctypes as C
import glob
import json
import logging
import os
import subprocess
import warnings

import numpy as np
import pytest

import lbp2d_np
from pyradiomics_b200 import _lib, imageoperations as IO

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "lbp2d_*.npz")))
NAMES = [os.path.basename(f)[6:-4] for f in GOLDEN]
WARN_3D = "Calculating Local Binary Pattern in 2D, but extracting features in 3D. Use with caution!"


def load(name):
    """golden npz, its settings, and (P, R, method, axis) with the reference's defaults"""
    z = np.load(os.path.join(HERE, "golden", f"lbp2d_{name}.npz"))
    kw = json.loads(str(z["settings"]))
    return z, kw, (kw.get("lbp2DSamples", 8), kw.get("lbp2DRadius", 1), kw.get("lbp2DMethod", "uniform"),
                   kw.get("force2Ddimension", 0))


def reference_cast(img, out, axis):
    """the reference wrapper's result from float64 per-slice LBPs `out`: a 3-D image keeps its dtype through NumPy's
    slice assignment, a 2-D image stays float64"""
    if img.ndim == 2:
        return out
    im_arr = np.array(img).swapaxes(0, axis)
    o = out.swapaxes(0, axis)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        for i in range(im_arr.shape[0]):
            im_arr[i, ...] = np.ascontiguousarray(o[i])
    return im_arr.swapaxes(0, axis)


def assert_bits_equal(got, ref, what=""):
    """identical dtype, shape, NaN positions and bits everywhere else (signed zeros included)"""
    assert got.dtype == ref.dtype and got.shape == ref.shape, (what, got.dtype, ref.dtype, got.shape, ref.shape)
    if got.dtype.kind == "f":
        nan_g, nan_r = np.isnan(got), np.isnan(ref)
        np.testing.assert_array_equal(nan_g, nan_r, err_msg=f"{what}: NaN positions")
        got, ref = np.where(nan_g, 0, got), np.where(nan_r, 0, ref)
    bad = got.view(np.uint8).reshape(got.shape + (-1,)) != ref.view(np.uint8).reshape(ref.shape + (-1,))
    assert not bad.any(), f"{what}: {int(bad.any(axis=-1).sum())} elements differ"


@pytest.fixture(scope="module")
def oracle_runs():
    out = {}
    for name in NAMES:
        z, kw, (P, R, method, axis) = load(name)
        out[name] = lbp2d_np.lbp2d_volume(z["image"], P, R, method, axis)
    return out


def test_goldens_present():
    assert set(NAMES) == {"brain1_a0", "brain1_a1", "brain1_a2", "u8_2d", "f32_naninf", "f64_naninf", "f64_naninf_var",
                          "const_var_i16", "var_i16", "u8_default_p9", "p24_r3", "p24_r3_default_f64", "r05_ror"}
    methods = {load(n)[2][2] for n in NAMES}
    assert methods == set(IO.LBP2D_METHODS)
    for f in GOLDEN:
        assert os.path.getsize(f) < 1 << 20


@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_golden(name, oracle_runs):
    z, kw, (P, R, method, axis) = load(name)
    assert_bits_equal(reference_cast(z["image"], oracle_runs[name], axis), z["out"], name)


@pytest.mark.parametrize("name", NAMES)
def test_golden_warnings(name):
    z, kw, _ = load(name)
    expect = [WARN_3D] if z["image"].ndim == 3 and not kw.get("force2D", False) else []
    assert json.loads(str(z["warnings"])) == expect


def test_goldens_cover_the_cast():
    """NaN cast to int16 (constant image, var), truncation (var on int16) and out-of-range codes cast to uint8"""
    z, *_ = load("const_var_i16")
    o = lbp2d_np.lbp2d_volume(z["image"], 8, 1, "var", 0)
    assert np.isnan(o).any() and z["out"].dtype == np.int16
    z, *_ = load("var_i16")
    o = lbp2d_np.lbp2d_volume(z["image"], 8, 1.5, "var", 0)
    assert (o != np.trunc(o)).any() and (z["out"] == np.trunc(o)).all()
    z, *_ = load("u8_default_p9")
    o = lbp2d_np.lbp2d_volume(z["image"], 9, 1, "default", 0)
    assert (o > 255).any() and z["out"].dtype == np.uint8


@pytest.mark.parametrize("P,R", [(8, 1), (9, 1), (24, 3), (4, 1), (1, 2.5), (31, 0.5)])
def test_offsets_are_the_librarys(P, R):
    rp, cp = lbp2d_np.offsets(P, R)
    _, _, rp2, cp2 = IO._lbp2d_params(P, R, "default")
    assert rp.tobytes() == rp2.tobytes() and cp.tobytes() == cp2.tobytes()
    ang = 2 * np.pi * np.arange(P) / P
    np.testing.assert_allclose(rp, -R * np.sin(ang), atol=5e-6)
    np.testing.assert_allclose(cp, R * np.cos(ang), atol=5e-6)


# ---------------------------------------------------------------------------------------------- exact properties
def _img(shape=(11, 13), seed=0, hi=6):
    return np.random.default_rng(seed).integers(0, hi, shape).astype(np.int16)


def test_p4_r1_is_the_four_zero_padded_neighbours():
    img = _img()
    rp, cp = lbp2d_np.offsets(4, 1)
    assert (rp == np.round(rp)).all() and (cp == np.round(cp)).all()
    p = np.pad(img.astype(np.float64), 1)
    ctr = p[1:-1, 1:-1]
    nb = [p[1:-1, 2:], p[:-2, 1:-1], p[1:-1, :-2], p[2:, 1:-1]]          # k = 0..3: east, north, west, south
    bits = np.stack([(n - ctr >= 0) for n in nb]).astype(np.int64)
    code = sum(bits[k] << k for k in range(4))
    np.testing.assert_array_equal(lbp2d_np.local_binary_pattern(img, 4, 1, "default"), code)
    np.testing.assert_array_equal(lbp2d_np.local_binary_pattern(img, 4, 1, "uniform"),
                                  np.where((bits[:-1] != bits[1:]).sum(0) <= 2, bits.sum(0), 5))


def _rotations(code, P):
    rots, v = [code], code.astype(np.int64)
    for _ in range(P - 1):
        v = (v >> 1) | ((v & 1) << (P - 1))
        rots.append(v)
    return np.stack(rots)


@pytest.mark.parametrize("P,R", [(8, 1), (6, 1.7), (12, 2)])
def test_ror_is_the_minimum_rotation_of_default(P, R):
    img = _img((14, 12), 1)
    d = lbp2d_np.local_binary_pattern(img, P, R, "default").astype(np.int64)
    np.testing.assert_array_equal(lbp2d_np.local_binary_pattern(img, P, R, "ror"), _rotations(d, P).min(0))


@pytest.mark.parametrize("P,R", [(8, 1), (16, 2), (5, 1.3)])
def test_uniform_range_and_popcount(P, R):
    img = _img((15, 16), 2)
    d = lbp2d_np.local_binary_pattern(img, P, R, "default").astype(np.int64)
    u = lbp2d_np.local_binary_pattern(img, P, R, "uniform")
    assert u.min() >= 0 and u.max() <= P + 1
    bits = (d[None] >> np.arange(P)[:, None, None]) & 1
    changes = (bits[:-1] != bits[1:]).sum(0)
    np.testing.assert_array_equal(u[changes <= 2], bits.sum(0)[changes <= 2])
    assert (u[changes > 2] == P + 1).all() and (changes > 2).any()


def _patterns(P):
    v = np.arange(1 << P, dtype=np.int64)
    bits = (v[None] >> np.arange(P)[:, None]) & 1
    return v, bits, (bits[:-1] != bits[1:]).sum(0) if P > 1 else np.zeros(v.shape, np.int64)


@pytest.mark.parametrize("P", [1, 2, 3, 4, 8, 12])
def test_nri_uniform_is_one_to_one_on_uniform_patterns(P):
    v, bits, changes = _patterns(P)
    n = lbp2d_np.codes(bits, P, "nri_uniform")
    uni = changes <= 2
    assert uni.sum() == 2 + P * (P - 1)
    assert sorted(n[uni].astype(int)) == list(range(P * (P - 1) + 2))
    assert (n[~uni] == P * (P - 1) + 2).all()


def test_var_is_the_one_pass_formula_and_nan_when_flat():
    img = np.random.default_rng(3).normal(size=(9, 10)) * 40
    img[3:8, 3:8] = 5.0                                        # flat neighbourhoods inside
    P, R = 8, 1.0
    got = lbp2d_np.local_binary_pattern(img, P, R, "var")
    t, _ = lbp2d_np.textures(img, P, R)
    for r in range(img.shape[0]):
        for c in range(img.shape[1]):
            s = q = 0.0
            for k in range(P):
                s += float(t[k, r, c])
                q += float(t[k, r, c]) * float(t[k, r, c])
            v = (q - (s * s) / P) / P
            if v != 0:
                assert got[r, c] == v
            else:
                assert np.isnan(got[r, c])
    assert np.isnan(got[4:7, 4:7]).all()


def test_rotating_a_slice_rotates_default_codes_by_one_bit():
    """P = 4, R = 1 samples exact neighbours; a 90-degree turn (np.rot90) moves east to north, north to west, ...: the
    code of the turned image at the turned pixel is the code rotated left by one bit (zero padding turns along)"""
    img = _img((10, 13), 4)
    d = lbp2d_np.local_binary_pattern(img, 4, 1, "default").astype(np.int64)
    e = lbp2d_np.local_binary_pattern(np.rot90(img), 4, 1, "default").astype(np.int64)
    np.testing.assert_array_equal(np.rot90(((d << 1) | (d >> 3)) & 15), e)


# ---------------------------------------------------------------------------------------------- host-compiled device math
@pytest.fixture(scope="module")
def emul():
    so = os.path.join(HERE, "host_emul", "liblbp2d_emul.so")
    src = os.path.join(HERE, "host_emul", "lbp2d_emul.cpp")
    tmp = so + ".%d" % os.getpid()
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", tmp, src])
    os.replace(tmp, so)
    lib = C.CDLL(so)
    lib.lbp2d_emul.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                               C.c_int, C.c_void_p]
    lib.lbp2d_codes_emul.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_longlong, C.c_void_p]
    lib.lbp2d_codes_emul.restype = None
    return lib


def run_emul(lib, img, P, R, method, axis):
    img = np.ascontiguousarray(img)
    if img.dtype == np.uint16:
        img = img.astype(np.int32)
    P, code, rp, cp = IO._lbp2d_params(P, R, method)
    Z, Y, X = (1,) * (3 - img.ndim) + img.shape
    out = np.empty(img.shape, np.float64)
    rc = lib.lbp2d_emul(img.ctypes.data, _lib.DTYPE_CODE[img.dtype], Z, Y, X, axis % 3 if img.ndim == 3 else 0, P, rp.ctypes.data,
                        cp.ctypes.data, code, out.ctypes.data)
    assert rc == 0
    return out


@pytest.mark.parametrize("name", NAMES)
def test_device_math_matches_oracle(name, emul, oracle_runs):
    z, kw, (P, R, method, axis) = load(name)
    got = run_emul(emul, z["image"], P, R, method, axis)
    assert_bits_equal(got, oracle_runs[name], name)
    assert_bits_equal(reference_cast(z["image"], got, axis), z["out"], name + " (golden)")


@pytest.mark.parametrize("method", list(IO.LBP2D_METHODS))
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_device_math_every_method_and_axis(method, axis, emul):
    img = np.round(np.random.default_rng(axis).normal(size=(6, 9, 11)) * 30).astype(np.int16)
    img[2, 4, 5] = 0
    for P, R in [(8, 1), (5, 2.25)]:
        assert_bits_equal(run_emul(emul, img, P, R, method, axis), lbp2d_np.lbp2d_volume(img, P, R, method, axis),
                          f"{method} axis {axis} P {P}")


@pytest.mark.parametrize("P", [1, 2, 5, 8, 13])
@pytest.mark.parametrize("method", ["default", "ror", "uniform", "nri_uniform"])
def test_device_codes_match_oracle_on_every_pattern(P, method, emul):
    v, bits, _ = _patterns(P)
    out = np.empty(v.shape, np.float64)
    b32 = np.ascontiguousarray(v, dtype=np.uint32)
    emul.lbp2d_codes_emul(IO.LBP2D_METHODS[method], P, b32.ctypes.data, len(v), out.ctypes.data)
    np.testing.assert_array_equal(out, lbp2d_np.codes(bits, P, method))


def test_device_codes_at_31_samples(emul):
    rng = np.random.default_rng(9)
    v = np.concatenate([rng.integers(0, 1 << 31, 4096), [0, (1 << 31) - 1, 1, 1 << 30, (1 << 30) - 1]]).astype(np.int64)
    bits = (v[None] >> np.arange(31)[:, None]) & 1
    b32 = np.ascontiguousarray(v, dtype=np.uint32)
    for method in ["default", "ror", "uniform", "nri_uniform"]:
        out = np.empty(v.shape, np.float64)
        emul.lbp2d_codes_emul(IO.LBP2D_METHODS[method], 31, b32.ctypes.data, len(v), out.ctypes.data)
        np.testing.assert_array_equal(out, lbp2d_np.codes(bits, 31, method), err_msg=method)


# ---------------------------------------------------------------------------------------------- guards
def test_4d_image_yields_nothing_with_a_warning(caplog):
    img = np.zeros((2, 3, 4, 5), np.int16)
    with caplog.at_level(logging.WARNING, logger="radiomics.imageoperations"):
        assert list(IO.getLBP2DImage(img, None)) == []
    assert "LBP 2D is only available for 2D or 3D with forced 2D extraction" in caplog.text


@pytest.mark.parametrize("kw,exc", [({"lbp2DSamples": 0}, ValueError), ({"lbp2DSamples": 32}, ValueError),
                                    ({"lbp2DSamples": 8.0}, ValueError), ({"lbp2DRadius": 0}, ValueError),
                                    ({"lbp2DRadius": -1.0}, ValueError), ({"lbp2DRadius": float("nan")}, ValueError),
                                    ({"lbp2DMethod": "median"}, KeyError)])
@pytest.mark.parametrize("nd", [2, 3])
def test_outside_the_envelope_raises_before_the_device(kw, exc, nd):
    img = np.zeros((4,) * nd, np.int16)
    with pytest.raises(exc):
        next(IO.getLBP2DImage(img, None, **kw))


def test_method_names_are_case_insensitive():
    assert IO._lbp2d_params(8, 1, "NRI_Uniform")[1] == IO.LBP2D_METHODS["nri_uniform"]
    np.testing.assert_array_equal(lbp2d_np.local_binary_pattern(_img(), 8, 1, "Uniform"),
                                  lbp2d_np.local_binary_pattern(_img(), 8, 1, "uniform"))
