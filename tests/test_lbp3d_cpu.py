"""3-D LBP (getLBP3DImage) without a GPU: the NumPy/SciPy oracle against the reference's goldens, the host tables
(icosphere, harmonics) against SciPy, the CUDA kernel's per-voxel arithmetic (csrc/lbp3d.cuh, compiled with g++ by
tests/host_emul/lbp3d_emul.cpp) against the oracle, and the generator's guards."""
import ctypes as C
import glob
import json
import logging
import os
import subprocess

import numpy as np
import pytest
from scipy import ndimage
from scipy.special import sph_harm_y

import lbp3d_np
from pyradiomics_b200 import _lib, imageoperations as IO

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "lbp3d_*.npz")))
NAMES = [os.path.basename(f)[6:-4] for f in GOLDEN]


def load(name):
    z = np.load(os.path.join(HERE, "golden", f"lbp3d_{name}.npz"))
    kw = json.loads(str(z["settings"]))
    return z, kw, kw.get("lbp3DLevels", 2), kw.get("lbp3DIcosphereRadius", 1), kw.get("lbp3DIcosphereSubdivision", 1)


def assert_lbp_close(got, ref, is_f32, what, m2=None, mean=None):
    """level maps: 1e-12 relative (plus 1e-12 of the map's largest value for entries that are rounding noise around 0);
    kurtosis: 1e-10 (1e-5 for float32 samples) where m2 is not near zero; NaN positions identical."""
    L = ref.shape[0] - 1
    for n in range(L):
        scale = max(float(np.nanmax(np.abs(ref[n]))), 1.0)
        np.testing.assert_allclose(got[n], ref[n], rtol=1e-12, atol=1e-12 * scale, err_msg=f"{what} m{n + 1}")
    k_got, k_ref = got[L], ref[L]
    np.testing.assert_array_equal(np.isnan(k_got), np.isnan(k_ref), err_msg=f"{what}: kurtosis NaN positions")
    ok = ~np.isnan(k_ref)
    if m2 is not None:
        eps = np.finfo(np.float32 if is_f32 else np.float64).eps
        ok &= m2 > 1e3 * (eps * mean) ** 2
    tol = 1e-5 if is_f32 else 1e-10
    np.testing.assert_allclose(k_got[ok], k_ref[ok], rtol=tol, atol=tol, err_msg=f"{what} kurtosis")


@pytest.fixture(scope="module")
def oracle_runs():
    out = {}
    for name in NAMES:
        z, kw, L, R, S = load(name)
        out[name] = lbp3d_np.lbp3d(z["image"], z["mask"] == 1, z["vertices"], L, R)
    return out


def test_goldens_present():
    assert set(NAMES) == {"brain1", "plateau_i16", "faces_f64", "f32", "l3_r15_s2", "s0"}
    for f in GOLDEN:
        assert os.path.getsize(f) < 1 << 20


@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_golden(name, oracle_runs):
    z, kw, L, R, S = load(name)
    o = oracle_runs[name]
    assert o["maps"].shape == z["maps"].shape
    assert_lbp_close(o["maps"], z["maps"], z["image"].dtype == np.float32, name, o["m2"], o["mean"])


def test_plateau_fixture_has_nan_kurtosis():
    z, *_ = load("plateau_i16")
    assert np.isnan(z["maps"][-1]).sum() > 100


def test_oracle_prefilter_is_map_coordinates():
    """spline_filter once + prefilter=False is what map_coordinates(order=3) does on its own"""
    z, kw, L, R, S = load("faces_f64")
    img = z["image"]
    pts = np.array(np.nonzero(z["mask"]))[:, ::7].T[None] + z["vertices"][:, None, :]
    coef = ndimage.spline_filter(img, order=3, output=np.float64, mode="constant")
    a = ndimage.map_coordinates(coef, pts.T, order=3, mode="constant", prefilter=False)
    b = ndimage.map_coordinates(img, pts.T, order=3)
    np.testing.assert_array_equal(a, b)
    assert (b == 0).any()                           # the ROI touches every face: some samples fall outside


@pytest.mark.parametrize("sub,nv", [(0, 12), (1, 42), (2, 162), (3, 642)])
@pytest.mark.parametrize("radius", [1.0, 1.5])
def test_icosphere(sub, nv, radius):
    v = IO._icosphere(sub, radius)
    assert v.shape == (nv, 3)
    np.testing.assert_allclose(np.linalg.norm(v, axis=1), radius, rtol=1e-15)
    assert len(np.unique(np.round(v, 12), axis=0)) == nv


@pytest.mark.parametrize("name", NAMES)
def test_icosphere_is_the_goldens_vertex_set(name):
    z, kw, L, R, S = load(name)
    np.testing.assert_array_equal(IO._icosphere(S, R), z["vertices"])


@pytest.mark.parametrize("sub,levels,radius", [(0, 4, 1.0), (1, 2, 1.0), (1, 4, 1.0), (2, 3, 1.5), (2, 4, 2.0)])
def test_harmonics_match_scipy(sub, levels, radius):
    v = IO._icosphere(sub, radius)
    theta = np.arccos(v[:, 2] / radius)
    phi = np.arctan2(v[:, 1], v[:, 0])
    ref = np.stack([sph_harm_y(n, m, phi, theta) for n in range(levels) for m in range(-n, n + 1)], axis=1)
    got = IO._lbp3d_harmonics(v, levels, radius)
    assert not np.isnan(got).any()
    assert np.abs(got - ref).max() < 1e-13


# ---------------------------------------------------------------------------------------------- host-compiled device math
@pytest.fixture(scope="module")
def emul():
    so = os.path.join(HERE, "host_emul", "liblbp3d_emul.so")
    src = os.path.join(HERE, "host_emul", "lbp3d_emul.cpp")
    tmp = so + ".%d" % os.getpid()
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", tmp, src])
    os.replace(tmp, so)
    lib = C.CDLL(so)
    lib.lbp3d_emul.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                               C.c_longlong, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    return lib


def run_emul(lib, img, mask, levels, radius, sub, sample_dtype=None):
    img = np.ascontiguousarray(img)
    coef = np.ascontiguousarray(ndimage.spline_filter(img, order=3, output=np.float64, mode="constant"))
    coords = np.ascontiguousarray(np.array(np.nonzero(mask)), dtype=np.int64)
    verts, harm = IO._lbp3d_tables(levels, radius, sub)
    out = np.empty((levels + 1, coords.shape[1]))
    dt = _lib.DTYPE_CODE[np.dtype(sample_dtype or img.dtype)]
    rc = lib.lbp3d_emul(coef.ctypes.data, img.ctypes.data, _lib.DTYPE_CODE[img.dtype], dt, *img.shape, coords.ctypes.data,
                        coords.shape[1], verts.ctypes.data, len(verts), harm.ctypes.data, levels, out.ctypes.data)
    assert rc == 0
    return out


@pytest.mark.parametrize("name", NAMES)
def test_device_math_matches_oracle(name, emul, oracle_runs):
    z, kw, L, R, S = load(name)
    img, mask = z["image"], z["mask"] == 1
    got = run_emul(emul, img, mask, L, R, S)
    o = oracle_runs[name]
    is_f32 = img.dtype == np.float32
    if np.issubdtype(img.dtype, np.integer):
        keep = np.ones(mask.sum(), bool)
    else:                                           # a sign bit within rounding of the centre may flip
        keep = o["margin"] >= 1e-9 * np.abs(img).max()
    assert_lbp_close(got[:, keep], o["maps"][:, keep], is_f32, name, o["m2"][keep], o["mean"][keep])
    assert_lbp_close(got[:, keep], z["maps"][:, keep], is_f32, name + " (golden)", o["m2"][keep], o["mean"][keep])
    # m1 has a closed form: sqrt(Nv) * #{samples >= centre} / (4 pi)
    nv = len(z["vertices"])
    count = got[0] * 4 * np.pi / np.sqrt(nv)
    np.testing.assert_allclose(count, np.round(count), rtol=0, atol=1e-12)
    np.testing.assert_allclose(got[0], o["maps"][0], rtol=4e-16 * nv, atol=0)


def test_device_math_uint16_clamp(emul):
    """uint16 travels as int32 on the device; the samples still round and clamp to [0, 65535]"""
    rng = np.random.default_rng(3)
    img = rng.integers(0, 65536, (8, 9, 10)).astype(np.uint16)
    img[3:6, 3:6, 3:6] = 65535
    img[0:2] = 0
    mask = np.ones(img.shape, bool)
    got = run_emul(emul, img.astype(np.int32), mask, 2, 1.0, 1, sample_dtype=np.uint16)
    o = lbp3d_np.lbp3d(img, mask, IO._icosphere(1, 1.0), 2, 1.0)
    assert_lbp_close(got, o["maps"], False, "uint16", o["m2"], o["mean"])
    unclamped = run_emul(emul, img.astype(np.int32), mask, 2, 1.0, 1)
    assert not np.allclose(unclamped, got, equal_nan=True)          # without the clamp the samples differ


# ---------------------------------------------------------------------------------------------- guards
def test_2d_image_yields_nothing_with_a_warning(caplog):
    img = np.zeros((8, 9), np.int16)
    with caplog.at_level(logging.WARNING, logger="radiomics.imageoperations"):
        assert list(IO.getLBP3DImage(img, np.ones_like(img))) == []
    assert "LBP 3D only available for 3 dimensional images, found 2 dimensions" in caplog.text


@pytest.mark.parametrize("kw", [{"lbp3DIcosphereSubdivision": 3}, {"lbp3DLevels": 5}])
def test_outside_the_kernel_range_raises(kw):
    img = np.zeros((6, 6, 6), np.int16)
    with pytest.raises(ValueError, match="outside the CUDA kernel's range"):
        next(IO.getLBP3DImage(img, np.ones_like(img), **kw))
