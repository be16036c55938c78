"""Square, square root, logarithm, exponential and gradient image types without a GPU: the NumPy oracle
(oracle/imagetypes_np.py) against the reference's goldens, the host scalars of rb_pointwise_image_dev against the oracle's,
the gradient oracle's properties, and the generators' and the pipeline's host logic with the device stubbed out."""
import glob
import logging
import os

import numpy as np
import pytest
import torch

import imagetypes_np as O
from pyradiomics_b200 import image as I, imageoperations as IO, pipeline as PP

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "imagetypes_*.npz")))
CASES = [os.path.basename(f)[len("imagetypes_"):-4] for f in GOLDEN]


def load(case):
    return np.load(os.path.join(HERE, "golden", f"imagetypes_{case}.npz"))


def assert_bits(got, ref, what, max_ulp=0):
    """same NaN positions; elsewhere the same value and sign of zero (max_ulp=0), or at most max_ulp units apart"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, what
    nan = np.isnan(ref)
    np.testing.assert_array_equal(np.isnan(got), nan, err_msg=f"{what}: NaN positions")
    if max_ulp == 0:
        np.testing.assert_array_equal(got[~nan], ref[~nan], err_msg=what)
        np.testing.assert_array_equal(np.signbit(got[~nan]), np.signbit(ref[~nan]), err_msg=f"{what}: sign of zero")
    else:
        np.testing.assert_array_max_ulp(got[~nan], ref[~nan], maxulp=max_ulp)


def test_goldens_present():
    assert set(CASES) == {"brain1", "ct_i16", "f32_small", "f64_signs", "u8_2d", "unit_i32", "zeros_u16"}
    for f in GOLDEN:
        assert os.path.getsize(f) < 1 << 20
    z = load("ct_i16")["image"].astype(np.float64)
    assert -z.min() > z.max()                                  # M comes from the minimum
    assert 0 < np.abs(load("f32_small")["image"]).max() < 1
    assert load("u8_2d")["image"].ndim == 2


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("kind", O.POINTWISE)
def test_oracle_reproduces_golden(case, kind):
    """square and square root are correctly rounded products and roots: bit for bit.  Logarithm and exponential go
    through NumPy's log / exp, which is the CPU's SIMD or libm routine; goldens written on one x86 CPU may be read on
    another, so those two may differ by 1 ulp (they are bit-identical where the goldens were written)."""
    z = load(case)
    assert_bits(O.pointwise(z["image"], kind), z[kind], f"{case} {kind}",
                max_ulp=0 if kind in ("square", "squareroot") else 1)


def test_degenerate_goldens_follow_the_reference():
    z = load("zeros_u16")
    for kind in ("square", "logarithm", "exponential"):
        assert np.isnan(z[kind]).all(), kind
    assert (z["squareroot"] == 0).all()
    assert (load("unit_i32")["exponential"] == 1).all()


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("kind", O.POINTWISE)
def test_host_scalar_is_the_references(case, kind):
    """pointwise_scalar(kind, max(-min, max)) == the oracle's whole-image scalar, to the bit; for logarithm that is
    log(M + 1) standing in for the second reduction max|transformed image|"""
    img = load(case)["image"]
    x = img.astype(np.float64)
    m = abs(max(-float(x.min()), float(x.max())))              # what image_max_abs reduces on the device
    got, ref = IO.pointwise_scalar(kind, m), O.scalar(img, kind)
    assert np.array_equal(got, ref, equal_nan=True), (case, kind, got, ref)


def test_logarithm_shortcut_on_random_images():
    rng = np.random.default_rng(2)
    for trial in range(300):
        scale = 10.0 ** rng.uniform(-3, 5)
        x = rng.normal(0, scale, rng.integers(1, 200))
        if trial % 3 == 0:
            x = np.round(x)
        if trial % 5 == 0:
            x[rng.integers(x.size)] = -np.abs(x).max() * 1.5          # M from the minimum
        m = abs(max(-float(x.min()), float(x.max())))
        got, ref = IO.pointwise_scalar("logarithm", m), O.scalar(x, "logarithm")
        assert np.array_equal(got, ref, equal_nan=True), (trial, m, got, ref)


def test_unknown_pointwise_kind_raises():
    with pytest.raises(ValueError, match="unknown image type"):
        IO.pointwise_scalar("cube", 3.0)


# ---------------------------------------------------------------------------------------------- gradient oracle
def test_gradient_of_a_linear_ramp():
    a = np.array([3, -2, 5])                                   # per z, y, x
    sp = np.array([0.5, 1.25, 2.0])
    zz, yy, xx = np.meshgrid(np.arange(6), np.arange(7), np.arange(8), indexing="ij")
    f = (a[0] * zz + a[1] * yy + a[2] * xx).astype(np.int32)
    g = O.gradient(f, sp)
    full = a / sp
    np.testing.assert_allclose(g[1:-1, 1:-1, 1:-1], np.sqrt((full ** 2).sum()), rtol=1e-13)
    half = full.copy()
    half[2] /= 2                                                # the x faces: half the one-sided difference
    np.testing.assert_allclose(g[1:-1, 1:-1, 0], np.sqrt((half ** 2).sum()), rtol=1e-13)
    np.testing.assert_allclose(g[1:-1, 1:-1, -1], np.sqrt((half ** 2).sum()), rtol=1e-13)
    corner = full / 2
    np.testing.assert_allclose(g[0, 0, 0], np.sqrt((corner ** 2).sum()), rtol=1e-13)


def test_gradient_without_spacing_is_unit_spacing():
    f = np.random.default_rng(4).normal(size=(5, 6, 7))
    assert_bits(O.gradient(f, None), O.gradient(f, (1.0, 1.0, 1.0)), "unit spacing")


def test_gradient_size_one_axis_contributes_nothing():
    f = np.random.default_rng(5).normal(size=(6, 7))
    assert_bits(O.gradient(f[:, None, :], (0.7, 3.0, 1.1)), O.gradient(f, (0.7, 1.1))[:, None, :], "y of size 1")


def test_gradient_2d_is_one_plane():
    f = np.random.default_rng(6).integers(-500, 500, (9, 11)).astype(np.int16)
    assert_bits(O.gradient(f, (0.8, 1.3)), O.gradient(f[None], (2.5, 0.8, 1.3))[0], "2-D")


def test_gradient_zero_spacing_raises():
    with pytest.raises(ValueError, match="cannot be zero"):
        O.gradient(np.zeros((3, 4, 5)), (1.0, 0.0, 1.0))
    with pytest.raises(ValueError, match="cannot be zero"):
        IO.gradient_magnitude_device(torch.zeros((3, 4, 5)), (1.0, 0.0, 1.0))
    with pytest.raises(ValueError, match="2-D or 3-D"):
        IO.gradient_magnitude_device(torch.zeros((2, 3, 4, 5)))
    with pytest.raises(ValueError, match="spacings"):
        IO.gradient_magnitude_device(torch.zeros((3, 4, 5)), (1.0, 1.0))


# ---------------------------------------------------------------------------------------------- generators, stubbed device
@pytest.fixture
def stubbed(monkeypatch):
    """the real _to_device onto the CPU; the device filters replaced by recorders that return x as float64"""
    calls = []
    monkeypatch.setattr(IO, "_dev", lambda: torch.device("cpu"))
    monkeypatch.setattr(IO, "pointwise_image_device",
                        lambda x, kind, max_abs=None: calls.append((kind, x.dtype, tuple(x.shape))) or x.to(torch.float64))
    monkeypatch.setattr(IO, "gradient_magnitude_device",
                        lambda x, spacing_zyx=None: calls.append(("gradient", x.dtype, spacing_zyx)) or x.to(torch.float64))
    return calls


GENERATORS = {"square": IO.getSquareImage, "squareroot": IO.getSquareRootImage, "logarithm": IO.getLogarithmImage,
              "exponential": IO.getExponentialImage, "gradient": IO.getGradientImage}


@pytest.mark.parametrize("name", list(GENERATORS))
@pytest.mark.parametrize("shape", [(4, 5, 6), (5, 6)])
def test_generator_names_dtypes_and_kwargs(stubbed, caplog, name, shape):
    nd = len(shape)
    img = I.ArrayImage(np.arange(np.prod(shape), dtype=np.uint16).reshape(shape), (0.5, 1.0, 2.0)[:nd], (1, 2, 3)[:nd])
    kw = {"binWidth": 5, "label": 2}
    with caplog.at_level(logging.DEBUG, logger="radiomics.imageoperations"):
        out = list(GENERATORS[name](img, None, **kw))
    assert len(out) == 1
    im, yielded, kwargs = out[0]
    assert yielded == name and kwargs == kw
    arr = I.as_array(im)
    assert arr.dtype == np.float64 and arr.shape == shape
    assert im.GetSpacing() == img.GetSpacing() and im.GetOrigin() == img.GetOrigin()
    assert stubbed[0][:2] == (name, torch.int32)                # uint16 travels as int32
    if name == "gradient":
        assert stubbed[0][2] == (2.0, 1.0, 0.5)[3 - nd:]         # z, y, x spacing
    else:
        assert f"Yielding {name} image" in caplog.text


def test_gradient_generator_spacing_switch_and_guards(stubbed):
    img = I.ArrayImage(np.zeros((4, 5, 6), np.int16), (0.5, 1.0, 2.0))
    list(IO.getGradientImage(img, None, gradientUseSpacing=False))
    assert stubbed[-1] == ("gradient", torch.int16, None)
    with pytest.raises(ValueError, match="2-D or 3-D"):
        next(IO.getGradientImage(I.ArrayImage(np.zeros((2, 3, 4, 5))), None))


def test_pipeline_image_types_order_and_one_reduction(monkeypatch):
    reductions, calls = [], []
    monkeypatch.setattr(IO, "image_max_abs", lambda x: reductions.append(1) or 7.0)
    monkeypatch.setattr(IO, "pointwise_image_device", lambda x, kind, max_abs=None: calls.append((kind, max_abs)) or x)
    monkeypatch.setattr(IO, "gradient_magnitude_device", lambda x, sp=None: calls.append(("gradient", sp)) or x)
    x = torch.zeros((3, 4, 5))
    types = ("exponential", "gradient", "square", "logarithm", "squareroot")
    names = [n for n, _ in PP.derived_images(x, (2.0, 1.0, 0.5), wavelet=None, sigmas=(), image_types=types)]
    assert names == ["original", *types]
    assert len(reductions) == 1
    assert calls == [("exponential", 7.0), ("gradient", (2.0, 1.0, 0.5)), ("square", 7.0), ("logarithm", 7.0),
                     ("squareroot", 7.0)]
    calls.clear()
    list(PP.derived_images(x, (2.0, 1.0, 0.5), wavelet=None, sigmas=(), original=False, image_types=("gradient",),
                           gradient_use_spacing=False))
    assert calls == [("gradient", None)]
    assert [n for n, _ in PP.derived_images(x, wavelet=None, sigmas=())] == ["original"]


def test_pipeline_unknown_image_type_raises():
    with pytest.raises(ValueError, match="unknown image types"):
        next(PP.derived_images(torch.zeros((2, 2, 2)), wavelet=None, sigmas=(), image_types=("square", "cube")))
