"""The oracle additions the GPU pre-filter tests rest on (tests/test_prefilters_gpu.py), checked without a GPU: ITK's
B-spline decomposition and the resampler's evaluation (oracle/resample_np.py) against SciPy and against a long-double
evaluation, and the LoG restatement (oracle/filters_np.py) against the float64 chain and an analytic Laplacian."""
import numpy as np
import pytest
import scipy.ndimage as ndi

import filters_np as FN
import resample_np as RS
from helpers import (RESAMPLE_DTYPES, RESAMPLE_NEAR_TIE_SHARE, RESAMPLE_NEW_SPACING_XYZ, RESAMPLE_SPACING_XYZ, near_integer,
                     resample_case)


def _lines(n, axis, seed=0):
    shape = [3, 4, 5]
    shape[axis] = n
    return np.random.default_rng(seed).normal(size=shape) * 100


# ---------------------------------------------------------------------------------------------------------------- B-spline
@pytest.mark.parametrize("n", [1, 2, 3, 5, 18, 19, 64, 200])
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_bspline_coefficients_exact_equal_scipy_and_itk_start_stays_close(n, axis):
    x = _lines(n, axis)
    exact = RS.bspline_coefficients(x, exact=True)
    ref = ndi.spline_filter(x, order=3, mode="mirror")
    scale = np.abs(ref).max()
    assert np.abs(exact - ref).max() <= 1e-13 * scale
    itk = RS.bspline_coefficients(x, exact=False)
    if n <= RS.HORIZON:                      # the same closed-form start: identical arithmetic
        assert np.array_equal(itk, exact)
    else:                                    # the causal start truncated after 18 samples: |pole|^18 ~ 5e-11
        assert np.abs(itk - exact).max() <= 1e-9 * scale


@pytest.mark.parametrize("shape", [(6, 7, 8), (1, 9, 10), (5, 1, 2), (19, 3, 20)])
def test_bspline_interpolation_reproduces_the_samples(shape):
    x = np.random.default_rng(1).normal(size=shape) * 50
    c = RS.bspline_coefficients(x, exact=True)
    back = RS.evaluate(c, shape, (0.0, 0.0, 0.0), (1.0, 1.0, 1.0), 3)
    assert np.abs(back - x).max() <= 1e-12 * np.abs(x).max()
    # linear and nearest on the input grid are the samples themselves
    assert np.array_equal(RS.evaluate(x, shape, (0.0, 0.0, 0.0), (1.0, 1.0, 1.0), 1), x)
    assert np.array_equal(RS.evaluate(x, shape, (0.0, 0.0, 0.0), (1.0, 1.0, 1.0), 0), x)


def test_evaluation_rules_at_half_samples_and_outside():
    x = np.arange(4.0)[None, None, :]
    # nearest rounds half up (ITK's RoundHalfIntegerUp); map_coordinates(order=0) would round 0.5 -> 0 and 2.5 -> 2
    got = RS.evaluate(x, (1, 1, 4), (0.0, 0.0, -0.5), (1.0, 1.0, 1.0), 0, default_value=-7.0)
    assert got.ravel().tolist() == [0.0, 1.0, 2.0, 3.0]
    # inside = [-0.5, n - 0.5) on every axis; outside gives the default value
    got = RS.evaluate(x, (1, 1, 3), (0.0, 0.0, -0.75), (1.0, 1.0, 4.25), 1, default_value=-7.0)      # -0.75, 3.5, 7.75
    assert got.ravel().tolist() == [-7.0, -7.0, -7.0]
    got = RS.evaluate(x, (1, 1, 2), (0.0, 0.0, -0.25), (1.0, 1.0, 3.5), 1, default_value=-7.0)
    assert got.ravel().tolist() == [0.0, 3.0]           # linear: clamped neighbours at both ends


def test_cast_clamps_and_truncates():
    v = np.array([-1e30, -129.7, -0.9, 0.9, 127.9, 300.2, 1e30])
    assert RS.cast(v, np.int8).tolist() == [-128, -128, 0, 0, 127, 127, 127]
    assert RS.cast(v, np.uint16).tolist() == [0, 0, 0, 0, 127, 300, 65535]
    assert RS.cast(v, np.uint64).tolist() == [0, 0, 0, 0, 127, 300, 2 ** 64 - 2048]
    assert RS.cast(v, np.int64)[0] == -(2 ** 63) and RS.cast(v, np.int64)[-1] == 2 ** 63 - 1024
    assert RS.cast(np.array([0.1]), np.float32)[0] == np.float32(0.1)


# ---------------------------------------------------------------------------------------------------------------- near ties
def _case_values(dtype):
    img, msk = resample_case(dtype)
    newSize, start, step, _ = RS.grid(msk, RESAMPLE_SPACING_XYZ, RESAMPLE_NEW_SPACING_XYZ, 20)
    geo = (tuple(newSize[::-1]), tuple(start[::-1]), tuple(step[::-1]))
    coef = RS.bspline_coefficients(img)
    return img, msk, coef, geo


@pytest.mark.parametrize("dtype", RESAMPLE_DTYPES)
def test_near_tie_margin_bounds_float64_evaluation(dtype):
    """tau = 1e-12 * max|coefficients| bounds the rounding of the float64 evaluation (against long double), and the
    share of inside-the-buffer values within tau of an integer stays below the bound the GPU test allows"""
    img, msk, coef, geo = _case_values(dtype)
    tau = 1e-12 * np.abs(coef).max()
    val = RS.evaluate(coef, *geo, 3, default_value=np.nan)
    ld = RS.evaluate(coef, *geo, 3, default_value=np.nan, dtype=np.longdouble)
    inside = ~np.isnan(val)
    assert inside.mean() > 0.9 and (~inside).any()
    assert np.abs(ld[inside] - val[inside]).max() <= tau
    share = near_integer(val[inside], tau).mean()
    print(f"{dtype}: tau {tau:.3g}, near-tie share {share:.4f}")
    assert share <= RESAMPLE_NEAR_TIE_SHARE
    if np.issubdtype(img.dtype, np.integer) and img.dtype.itemsize < 8:
        info = np.iinfo(img.dtype)
        assert (val[inside] < info.min).any() and (val[inside] > info.max).any()      # both clamps are exercised
    # the oracle's whole resampling agrees with its pieces
    v2, out, m, _ = RS.resample_itk(img, msk, RESAMPLE_SPACING_XYZ, RESAMPLE_NEW_SPACING_XYZ, padDistance=20)
    assert out.dtype == img.dtype and np.array_equal(np.where(inside, val, 0.0), v2)
    assert np.array_equal(m, RS.resample(img, msk, RESAMPLE_SPACING_XYZ, RESAMPLE_NEW_SPACING_XYZ, 20)[1])


# ---------------------------------------------------------------------------------------------------------------- LoG
def _float64_chain(x, sigma_mm, spacing_zyx):
    """the restatement the earlier GPU tests carried (isotropic only there): per direction d the two smoothing passes in
    axis order, float64 sum of the three terms"""
    import pyradiomics_b200.imageoperations as IO
    s = [sigma_mm / v for v in spacing_zyx]
    ref = np.zeros(x.shape)
    xf = x.astype(np.float32).astype(np.float64)
    for d in range(3):
        cur = xf
        for e in range(3):
            if e != d:
                cur = FN.recursive_gaussian_axis(cur, IO.recursive_gaussian_coefficients(s[e], 0), e).astype(np.float32).astype(np.float64)
        ref += (FN.recursive_gaussian_axis(cur, IO.recursive_gaussian_coefficients(s[d], 2), d) * s[d] ** 2).astype(np.float32)
    return ref


def _smooth(shape, seed=3):
    return ndi.gaussian_filter(np.random.default_rng(seed).normal(size=shape), 2.0) * 100


@pytest.mark.parametrize("spacing_zyx", [(1.0, 1.0, 1.0), (2.0, 0.8, 0.6)])
def test_log_restatement_matches_float64_chain(spacing_zyx):
    x = _smooth((24, 30, 36)).astype(np.float32)
    for sigma in (2.0, 3.0):
        got, terms = FN.log_restatement(x, sigma, spacing_zyx, return_terms=True)
        ref = _float64_chain(x, sigma, spacing_zyx)
        assert got.dtype == np.float32 and len(terms) == 3
        assert np.allclose(got, ref, rtol=2e-4, atol=2e-4 * np.abs(ref).max())


@pytest.mark.parametrize("sigma", [2.0, 3.0])
def test_log_restatement_matches_analytic_anisotropic_laplacian(sigma):
    """sum_d sigma_d^2 d2/dd2 of a Gaussian with sigma_d = sigma / spacing_d voxels (SciPy FIR): no shared coefficient
    code, so a swapped axis or scale fails here"""
    spacing_zyx = (2.0, 0.8, 0.6)
    x = _smooth((30, 56, 72))
    got = FN.log_restatement(x, sigma, spacing_zyx, in_dtype=np.float64)
    s = [sigma / v for v in spacing_zyx]
    ana = sum(s[d] ** 2 * ndi.gaussian_filter(x, s, order=[2 if e == d else 0 for e in range(3)], mode="nearest", truncate=6.0)
              for d in range(3))
    c = tuple(slice(int(np.ceil(4 * v)) + 2, -int(np.ceil(4 * v)) - 2) for v in s)
    err = np.abs(got[c] - ana[c]).max() / np.abs(ana[c]).max()
    assert err < 0.03, err
    # the same with the spacing reversed is a different image: the check does see the axes
    wrong = FN.log_restatement(x, sigma, spacing_zyx[::-1], in_dtype=np.float64)
    assert np.abs(wrong[c] - ana[c]).max() / np.abs(ana[c]).max() > 0.1
