"""The 2-D LBP image of the device-resident suites without a GPU: the kernel's store in the image's own dtype
(numpy_cast in csrc/lbp2d.cuh, compiled with g++ by tests/host_emul/lbp2d_cast_emul.cpp) against NumPy's assignment cast
and against the reference's goldens, and pipeline.derived_images' settings checks, names, order and warning."""
import ctypes as C
import logging
import os
import subprocess
import warnings

import numpy as np
import pytest
import torch

import lbp2d_np
from pyradiomics_b200 import _lib, imageoperations as IO, pipeline
from test_lbp2d_cpu import NAMES, WARN_3D, assert_bits_equal, load, reference_cast

HERE = os.path.dirname(os.path.abspath(__file__))
DTYPES = [np.int16, np.int32, np.float32, np.float64, np.uint8, np.uint16, np.int64]
CORPUS = [0.0, -0.0, 0.5, 1.9999, 2.0 ** 7 - 1, 2.0 ** 7 + 1, 2.0 ** 8 - 1, 2.0 ** 8 + 1, 2.0 ** 15 - 1, 2.0 ** 15 + 1,
          2.0 ** 16 - 1, 2.0 ** 16 + 1, 2.0 ** 31 - 1, 2.0 ** 31, 2.0 ** 32 - 1, 2.0 ** 32 + 1, 2.0 ** 53, 2.0 ** 63,
          2.0 ** 64, 1e300, np.inf, -np.inf, np.nan,
          # what VAR gives beyond the codes: fractions, values between the integer ranges, and negatives from rounding
          70000.5, 3e9, 1e10 + 0.25, 2.0 ** 62 + 2.0 ** 40, -1e-12, -1.5, -129.0, -2.0 ** 31, -2.0 ** 31 - 1, -2.0 ** 63]


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(HERE, "host_emul", "liblbp2d_cast_emul.so")
    src = os.path.join(HERE, "host_emul", "lbp2d_cast_emul.cpp")
    tmp = so + ".%d" % os.getpid()
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", tmp, src])
    os.replace(tmp, so)
    lib = C.CDLL(so)
    lib.numpy_cast_emul.argtypes = [C.c_int, C.c_void_p, C.c_longlong, C.c_void_p]
    lib.lbp2d_cast_emul.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                    C.c_void_p, C.c_int, C.c_void_p]
    return lib


def numpy_assign(values, dtype):
    """what NumPy stores for float64 `values` assigned into an array of `dtype` (the reference's per-slice assignment)"""
    out = np.zeros(len(values), dtype)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        out[...] = values
    return out


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
def test_numpy_cast_matches_numpy_assignment(dtype, emul):
    # every value alone and in arrays of several lengths and offsets, so that NumPy's vector loops run as well as its
    # scalar tail; NumPy's result for one value must not depend on either
    for v in CORPUS:
        for n in (1, 3, 8, 17, 64, 257):
            for off in (0, 1, 3):
                vals = np.full(n + off, v)[off:]
                ref = numpy_assign(vals, dtype)
                assert len(np.unique(ref.view(f"u{ref.itemsize}"))) == 1, (dtype, v, n, off)
                got = np.empty(n, dtype)
                assert emul.numpy_cast_emul(_lib.DTYPE_CODE[np.dtype(dtype)], vals.ctypes.data, n, got.ctypes.data) == 0
                assert_bits_equal(got, ref, f"{np.dtype(dtype)} {v!r} n {n} offset {off}")


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
def test_numpy_cast_on_every_code(dtype, emul):
    # the integer codes of P <= 31 and the bit patterns around every power of two up to 2^31 - 1
    v = np.unique(np.concatenate([np.arange(0, 4096), ((2.0 ** np.arange(1, 32))[:, None] + np.arange(-2, 3)).ravel()]))
    v = v[(v >= 0) & (v <= 2.0 ** 31 - 1)]
    got = np.empty(len(v), dtype)
    emul.numpy_cast_emul(_lib.DTYPE_CODE[np.dtype(dtype)], v.ctypes.data, len(v), got.ctypes.data)
    assert_bits_equal(got, numpy_assign(v, dtype), np.dtype(dtype).name)


def cast_emul(lib, img, P, R, method, axis):
    img = np.ascontiguousarray(img)
    P, code, rp, cp = IO._lbp2d_params(P, R, method)
    out = np.empty(img.shape, img.dtype)
    assert lib.lbp2d_cast_emul(img.ctypes.data, _lib.DTYPE_CODE[img.dtype], *img.shape, axis % 3, P, rp.ctypes.data,
                               cp.ctypes.data, code, out.ctypes.data) == 0
    return out


@pytest.mark.parametrize("name", [n for n in NAMES if load(n)[0]["image"].ndim == 3])
def test_fused_store_matches_golden(name, emul):
    z, _, (P, R, method, axis) = load(name)
    assert_bits_equal(cast_emul(emul, z["image"], P, R, method, axis), z["out"], name)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("method", list(IO.LBP2D_METHODS))
def test_fused_store_matches_host_cast(dtype, method, emul):
    raw = np.round(np.random.default_rng(5).normal(size=(5, 9, 11)) * 70)
    if np.issubdtype(dtype, np.unsignedinteger):
        raw -= raw.min()
    img = raw.astype(dtype)
    if dtype == np.int32:
        img *= 40000                                            # VAR beyond the int32 range
    if np.issubdtype(dtype, np.floating):
        img[1, 2, 3], img[2, 4, 4], img[3, 6, 1] = np.nan, np.inf, -np.inf
    for axis, P, R in [(0, 8, 1), (1, 17, 2), (2, 5, 1.5)]:
        assert_bits_equal(cast_emul(emul, img, P, R, method, axis),
                          reference_cast(img, lbp2d_np.lbp2d_volume(img, P, R, method, axis), axis),
                          f"{np.dtype(dtype)} {method} axis {axis} P {P}")


def test_cast_entry_refuses_unknown_dtype_codes_before_the_device():
    L = _lib.lib()
    # placeholder device pointers must never reach a card: this runs only where there is none
    if torch.cuda.is_available() or L.rb_device_count() > 0:
        pytest.skip("GPU present")
    buf, rp = np.zeros(64), np.zeros(8)
    for code in (-1, 7):
        assert L.rb_lbp2d_cast_dev(_lib.ptr(buf), code, 2, 2, 2, 0, 8, _lib.ptr(rp), _lib.ptr(rp), 0, _lib.ptr(buf),
                                   None) == _lib.RB_ERR_ARG
        assert b"unknown dtype code" in L.rb_last_error()


# ---------------------------------------------------------------------------------------------- pipeline, without a GPU
BAD = [({"lbp2DSamples": 0}, ValueError), ({"lbp2DSamples": 32}, ValueError), ({"lbp2DSamples": 8.0}, ValueError),
       ({"lbp2DRadius": 0}, ValueError), ({"lbp2DRadius": float("nan")}, ValueError),
       ({"lbp2DMethod": "median"}, KeyError), ({"force2Ddimension": 3}, ValueError),
       ({"force2Ddimension": 1.0}, ValueError)]


@pytest.mark.parametrize("kw,exc", BAD)
def test_bad_settings_raise_before_the_device(kw, exc, monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("reached the device")
    for f in ("lbp2d_device", "normalize_image_device", "resegment_mask_device", "log_filter_device"):
        monkeypatch.setattr(IO, f, no_device)
    x = torch.zeros((4, 5, 6), dtype=torch.int16)                # a CPU tensor: any device work would fail
    m = torch.ones((4, 5, 6), dtype=torch.uint8)
    with pytest.raises(exc):
        next(pipeline.derived_images(x, wavelet=None, sigmas=(), lbp2d=kw))
    with pytest.raises(exc):
        pipeline.voxel_suite_with_filters(x, m, wavelet=None, sigmas=(), lbp2d=kw, normalize={})
    with pytest.raises(exc):
        pipeline.segment_suite_with_filters(x, m, wavelet=None, sigmas=(), lbp2d=kw, normalize={})


@pytest.fixture
def fake_device(monkeypatch):
    """the image-type steps of derived_images replaced by recorders, so that names and order show without a GPU"""
    calls = []

    def rec(name):
        def f(x, *a, **k):
            calls.append((name, a, k))
            return torch.zeros((3,) + tuple(x.shape)) if name == "lbp3d" else x
        return f
    for f, name in (("lbp2d_device", "lbp2d"), ("lbp3d_device", "lbp3d"), ("log_filter_device", "log"),
                    ("pointwise_image_device", "pointwise"), ("gradient_magnitude_device", "gradient")):
        monkeypatch.setattr(IO, f, rec(name))
    monkeypatch.setattr(IO, "image_max_abs", lambda x: 1.0)
    return calls


def names(**kw):
    x = torch.zeros((4, 5, 6), dtype=torch.int16)
    return [n for n, _ in pipeline.derived_images(x, wavelet=None, sigmas=(1.0,), image_types=("square", "gradient"),
                                                  lbp3d={}, mask=x, **kw)]


def test_names_and_order_with_and_without_lbp2d(fake_device):
    before = ["original", "log-sigma-1-0-mm-3D", "square", "gradient", "lbp-3D-m1", "lbp-3D-m2", "lbp-3D-k"]
    assert names() == before
    assert not [c for c in fake_device if c[0] == "lbp2d"]
    assert names(lbp2d={}) == before[:4] + ["lbp-2D"] + before[4:]
    (_, args, kw), = [c for c in fake_device if c[0] == "lbp2d"]
    assert args == (0, 8, 1, "uniform") and kw == {"out_dtype": torch.int16}       # getLBP2DImage's defaults
    fake_device.clear()
    names(lbp2d={"lbp2DRadius": 2, "lbp2DSamples": 12, "lbp2DMethod": "var", "force2D": True, "force2Ddimension": -1})
    (_, args, _), = [c for c in fake_device if c[0] == "lbp2d"]
    assert args == (2, 12, 2, "var")


def test_warning_when_force2d_is_off(fake_device, caplog):
    with caplog.at_level(logging.WARNING, logger="radiomics.imageoperations"):
        names(lbp2d={})
    assert WARN_3D in caplog.text
    caplog.clear()
    with caplog.at_level(logging.WARNING, logger="radiomics.imageoperations"):
        names(lbp2d={"force2D": True})
    assert WARN_3D not in caplog.text


def test_suites_fill_force2d_from_their_settings():
    assert pipeline._suite_lbp2d(None, {"force2D": True}) is None
    assert pipeline._suite_lbp2d({}, {}) == {"force2D": False, "force2Ddimension": 0}
    assert pipeline._suite_lbp2d({}, {"force2D": True, "force2Ddimension": 2}) == {"force2D": True, "force2Ddimension": 2}
    assert pipeline._suite_lbp2d({"force2D": False, "force2Ddimension": 1, "lbp2DSamples": 4},
                                 {"force2D": True, "force2Ddimension": 2}) == \
        {"force2D": False, "force2Ddimension": 1, "lbp2DSamples": 4}
