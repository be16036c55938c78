"""Square, square root, logarithm, exponential and gradient image types on the GPU (csrc/filters.cu): the generators
against the reference's goldens for every supported input dtype, the gradient against the NumPy oracle bit for bit,
bit-reproducibility, the C entry points' argument checks and the opt-in pipeline images."""
import ctypes as C

import numpy as np
import pytest
import torch

import imagetypes_np as O
from pyradiomics_b200 import _lib, featureclasses as FC, image as I, imageoperations as IO, pipeline as PP
from test_imagetypes_cpu import CASES, assert_bits, load

pytestmark = pytest.mark.gpu

GENERATORS = {"square": IO.getSquareImage, "squareroot": IO.getSquareRootImage, "logarithm": IO.getLogarithmImage,
              "exponential": IO.getExponentialImage}
DTYPES = (np.int16, np.int32, np.int64, np.uint8, np.uint16, np.float32, np.float64)


def assert_golden(got, ref, kind, what):
    """square / squareroot: bit for bit; logarithm / exponential (CUDA log / exp, <= 1 ulp): 1e-15 relative"""
    if kind in ("square", "squareroot"):
        assert_bits(got, ref, what)
        return
    nan = np.isnan(ref)
    np.testing.assert_array_equal(np.isnan(got), nan, err_msg=f"{what}: NaN positions")
    np.testing.assert_allclose(got[~nan], ref[~nan], rtol=1e-15, atol=0, err_msg=what)


def exact_casts(img):
    """the supported dtypes that hold every value of `img` exactly"""
    x = img.astype(np.float64)
    out = []
    for dt in DTYPES:
        info = np.iinfo(dt) if np.issubdtype(dt, np.integer) else None
        if info is not None and (x.min() < info.min or x.max() > info.max):
            continue
        if np.array_equal(img.astype(dt).astype(np.float64), x):
            out.append(dt)
    return out


def test_every_dtype_is_covered():
    covered = {dt for case in CASES for dt in exact_casts(load(case)["image"])}
    assert covered == set(DTYPES)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("kind", list(GENERATORS))
def test_generators_match_golden(case, kind):
    z = load(case)
    for dt in exact_casts(z["image"]):
        img = I.ArrayImage(z["image"].astype(dt), (0.7, 0.8, 2.5)[:z["image"].ndim])
        (im, name, kw), = list(GENERATORS[kind](img, None, label=1))
        assert name == kind and kw == {"label": 1}
        got = I.as_array(im)
        assert got.dtype == np.float64 and im.GetSpacing() == img.GetSpacing()
        assert_golden(got, z[kind], kind, f"{case} as {np.dtype(dt).name}: {kind}")


def test_device_api_with_a_given_max_abs():
    z = load("ct_i16")
    x = torch.as_tensor(z["image"]).cuda()
    m = IO.image_max_abs(x)
    assert m == 1024.0
    for kind in GENERATORS:
        assert_golden(IO.pointwise_image_device(x, kind, m).cpu().numpy(), z[kind], kind, kind)


def gradient_cases():
    rng = np.random.default_rng(9)
    f = rng.normal(0, 300, (11, 12, 13))
    f[5, 6, 7], f[2, 3, 4] = np.inf, np.nan                           # spread like ITK's: 0 * f[0] is kept
    return [
        ("i16 anisotropic", rng.integers(-1024, 1500, (17, 19, 23)).astype(np.int16), (2.5, 0.7, 1.3)),
        ("u16", rng.integers(0, 65536, (9, 10, 11)).astype(np.uint16), (1.0, 1.0, 1.0)),
        ("u8", rng.integers(0, 256, (9, 10, 11)).astype(np.uint8), (0.5, 0.5, 3.0)),
        ("i32", rng.integers(-10 ** 6, 10 ** 6, (8, 9, 10)).astype(np.int32), (1.25, 0.5, 2.0)),
        ("i64", rng.integers(-10 ** 6, 10 ** 6, (8, 9, 10)).astype(np.int64), (1.0, 2.0, 3.0)),
        ("f32", rng.normal(0, 2, (10, 9, 8)).astype(np.float32), (0.3, 0.9, 1.7)),
        ("f64 inf nan", f, (1.5, 1.0, 0.75)),
        ("size-1 axes", rng.normal(0, 9, (1, 7, 1)), (2.0, 3.0, 5.0)),
        ("2-D", rng.integers(0, 4000, (33, 47)).astype(np.int16), (0.6, 0.9)),
    ]


@pytest.mark.parametrize("use_spacing", [True, False])
def test_gradient_matches_oracle_bit_for_bit(use_spacing):
    for what, img, sp_zyx in gradient_cases():
        image = I.ArrayImage(img, tuple(sp_zyx)[::-1])
        kw = {} if use_spacing else {"gradientUseSpacing": False}
        (im, name, out_kw), = list(IO.getGradientImage(image, None, **kw))
        assert name == "gradient" and out_kw == kw
        got = I.as_array(im)
        assert got.dtype == np.float64 and got.shape == img.shape
        assert_bits(got, O.gradient(img, sp_zyx if use_spacing else None), what)


def test_two_runs_are_bit_identical():
    img = gradient_cases()[0][1]
    x = torch.as_tensor(img).cuda()
    for kind in GENERATORS:
        a, b = IO.pointwise_image_device(x, kind), IO.pointwise_image_device(x, kind)
        assert torch.equal(a.view(torch.int64), b.view(torch.int64)), kind
    a, b = IO.gradient_magnitude_device(x, (2.5, 0.7, 1.3)), IO.gradient_magnitude_device(x, (2.5, 0.7, 1.3))
    assert torch.equal(a.view(torch.int64), b.view(torch.int64))


def test_entry_points_reject_bad_arguments():
    L = _lib.lib()
    x = torch.zeros((4, 5, 6), dtype=torch.int16, device="cuda")
    out = torch.empty((4, 5, 6), dtype=torch.float64, device="cuda")
    s, n = _lib.stream(), C.c_longlong(x.numel())
    c = C.c_double(1.0)
    w = (C.c_double * 3)(1.0, 1.0, 1.0)
    pw = L.rb_pointwise_image_dev
    assert pw(_lib.ptr(x), 0, n, 0, c, _lib.ptr(out), s) == _lib.RB_OK
    assert pw(None, 0, n, 0, c, _lib.ptr(out), s) == _lib.RB_ERR_ARG
    assert pw(_lib.ptr(x), 0, n, 0, c, None, s) == _lib.RB_ERR_ARG
    assert pw(_lib.ptr(x), 7, n, 0, c, _lib.ptr(out), s) == _lib.RB_ERR_ARG
    assert pw(_lib.ptr(x), -1, n, 0, c, _lib.ptr(out), s) == _lib.RB_ERR_ARG
    assert pw(_lib.ptr(x), 0, n, 4, c, _lib.ptr(out), s) == _lib.RB_ERR_ARG
    assert pw(_lib.ptr(x), 0, n, -1, c, _lib.ptr(out), s) == _lib.RB_ERR_ARG
    assert pw(_lib.ptr(x), 0, C.c_longlong(0), 0, c, _lib.ptr(out), s) == _lib.RB_ERR_ARG
    gm = L.rb_gradient_magnitude_dev
    assert gm(_lib.ptr(x), 0, 4, 5, 6, w, _lib.ptr(out), s) == _lib.RB_OK
    assert gm(None, 0, 4, 5, 6, w, _lib.ptr(out), s) == _lib.RB_ERR_ARG
    assert gm(_lib.ptr(x), 0, 4, 5, 6, None, _lib.ptr(out), s) == _lib.RB_ERR_ARG
    assert gm(_lib.ptr(x), 0, 4, 5, 6, w, None, s) == _lib.RB_ERR_ARG
    assert gm(_lib.ptr(x), 7, 4, 5, 6, w, _lib.ptr(out), s) == _lib.RB_ERR_ARG
    for Z, Y, X in ((0, 5, 6), (4, 0, 6), (4, 5, -1)):
        assert gm(_lib.ptr(x), 0, Z, Y, X, w, _lib.ptr(out), s) == _lib.RB_ERR_ARG
    torch.cuda.synchronize()


def test_pipeline_image_types_equal_per_image_plugins():
    import scipy.ndimage as ndi
    rng = np.random.default_rng(12)
    x = (ndi.gaussian_filter(rng.normal(size=(12, 13, 14)), 1.2) * 400 - 100).astype(np.int16)
    m = (rng.random(x.shape) < 0.8).astype(np.uint8)
    spacing_zyx = (2.0, 0.8, 0.6)
    types = ("square", "squareroot", "logarithm", "exponential", "gradient")
    got = {}
    xt, mt = torch.as_tensor(x).cuda(), torch.as_tensor(m).cuda()
    info = PP.voxel_suite_with_filters(xt, mt, classes=("gldm",), spacing_zyx=spacing_zyx, wavelet=None, sigmas=(),
                                       image_types=types, binCount=16,
                                       consume=lambda n, c, t: got.__setitem__((n, c), t.cpu().numpy().copy()))
    names = [n for n, _, _ in info]
    assert names == ["original", *types]
    default = PP.voxel_suite_with_filters(xt, mt, classes=("gldm",), spacing_zyx=spacing_zyx, wavelet=None, sigmas=(),
                                          binCount=16)
    assert [n for n, _, _ in default] == ["original"]
    image = I.ArrayImage(x, spacing_zyx[::-1])
    imgs = {n: im for t in types
            for im, n, _ in (IO.getGradientImage if t == "gradient" else GENERATORS[t])(image, None)}
    dev = dict(PP.derived_images(xt, spacing_zyx, wavelet=None, sigmas=(), original=False, image_types=types))
    for n in types:
        np.testing.assert_array_equal(dev[n].cpu().numpy(), I.as_array(imgs[n]), err_msg=n)
        ref = FC.FEATURE_CLASSES["gldm"](imgs[n], I.ArrayImage(m, spacing_zyx[::-1]), voxelBased=True, binCount=16).execute()
        for k, f in enumerate(_lib.feature_names("gldm")):
            assert np.allclose(got[(n, "gldm")][k], I.as_array(ref[f]), rtol=1e-9, atol=1e-11, equal_nan=True), (n, f)
