"""GPU resampling (rb_bspline_prefilter_dev + rb_resample_dev behind imageoperations.resampleImage) against the oracle
restatement and, through the plugin classes, against the reference's `breast1_resampling` baseline column."""
import os

import numpy as np
import pytest

import resample_np as RS
from helpers import near_integer
from pyradiomics_b200 import featureclasses as FC, image as I, imageoperations as IO

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_resample_image_matches_oracle_and_reference_baseline():
    z = np.load(os.path.join(G, "resample_breast1.npz"))
    exp = dict(zip(z["names"], z["values"]))
    sp = tuple(z["spacing"])
    ri, rm = IO.resampleImage(I.ArrayImage(z["image"], sp), I.ArrayImage(z["mask"], sp), resampledPixelSpacing=[2, 2, 2],
                              interpolator="sitkBSpline", padDistance=5)
    oi, om, new = RS.resample(z["image"], z["mask"], sp, (2, 2, 2))
    assert ri.array.dtype == z["image"].dtype and ri.GetSpacing() == (2.0, 2.0, 2.0)
    assert np.array_equal(rm.array, om)
    assert np.array_equal(ri.array, oi)                 # (ITK-style truncated filter start vs SciPy's exact one: same integers)
    # segment-based features of the resampled case through the plugin classes == the reference's baseline column
    idx = np.array(np.where(rm.array == 1))
    sl = tuple(slice(a, b + 1) for a, b in zip(idx.min(1), idx.max(1)))
    ci, cm = I.ArrayImage(ri.array[sl], ri.GetSpacing()), I.ArrayImage(rm.array[sl], ri.GetSpacing())
    n = 0
    for cname, cls in {**FC.FEATURE_CLASSES, **FC.NEXT_CLASSES}.items():
        if cname == "shape2D":
            continue
        for k, v in cls(ci, cm, binWidth=25).execute().items():
            key = f"original_{cname}_{k}"
            if key in exp:
                assert float(v) == pytest.approx(exp[key], rel=1e-7, abs=1e-10), key
                n += 1
    assert n >= 100


@pytest.mark.parametrize("case", ["upsample", "inplane", "linear", "float", "2d"])
def test_resample_variants_against_oracle(case):
    rng = np.random.default_rng(3)
    import scipy.ndimage as ndi
    img = (ndi.gaussian_filter(rng.normal(size=(14, 40, 37)), 1.2) * 300 + 100)
    msk = np.zeros(img.shape, np.uint8)
    msk[3:11, 8:30, 6:29] = 1
    sp = (0.8, 0.9, 2.5)
    kw = dict(resampledPixelSpacing=[1.7, 1.7, 1.7], interpolator="sitkBSpline", padDistance=3)
    order = 3
    arr = img.astype(np.int16)
    if case == "upsample":
        kw["resampledPixelSpacing"] = [0.5, 0.6, 1.0]
    elif case == "inplane":
        kw["resampledPixelSpacing"] = [1.3, 1.3, 0]
    elif case == "linear":
        kw["interpolator"] = "sitkLinear"
        order = 1
    elif case == "float":
        arr = img.astype(np.float32)
    elif case == "2d":
        arr, msk, sp = arr[5], msk[5], sp[:2]
        kw["resampledPixelSpacing"] = [1.7, 1.7]
    ri, rm = IO.resampleImage(I.ArrayImage(arr, sp), I.ArrayImage(msk, sp), **kw)
    if case == "2d":
        oi, om, _ = RS.resample(arr[None], msk[None], sp + (1.0,), tuple(kw["resampledPixelSpacing"]) + (0,), 3, 1, order)
        val, itk, _, _ = RS.resample_itk(arr[None], msk[None], sp + (1.0,), tuple(kw["resampledPixelSpacing"]) + (0,), 3, 1, order)
        oi, om, val, itk = oi[0], om[0], val[0], itk[0]
    else:
        oi, om, _ = RS.resample(arr, msk, sp, kw["resampledPixelSpacing"], 3, 1, order)
        val, itk, _, _ = RS.resample_itk(arr, msk, sp, kw["resampledPixelSpacing"], 3, 1, order)
    assert ri.array.shape == oi.shape and np.array_equal(rm.array, om)
    # against ITK's truncated filter start and the kernel's own evaluation: float32 within 1 ulp; integers equal except
    # where the float64 value lies within tau of an integer (there the last bits decide the truncation: linear
    # interpolation of integers lands on integers wherever the grids coincide)
    src = RS.bspline_coefficients(arr.reshape((1,) * (3 - arr.ndim) + arr.shape)) if order == 3 else arr
    tau = 1e-12 * np.abs(src).max()
    if arr.dtype == np.float32:
        assert (np.abs(ri.array.astype(np.float64) - itk) <= np.spacing(np.abs(itk))).all()
        assert np.allclose(ri.array, oi, rtol=1e-5, atol=1e-3)
    else:
        ties = near_integer(val, tau) & (val != 0)
        d = np.abs(ri.array.astype(np.int64) - itk.astype(np.int64))
        assert not ((d > 0) & ~ties).any() and d.max() <= 1
        assert ties.mean() < (0.03 if case == "linear" else 1e-3)
