"""Segment-based first order on the device (voxel.firstorder_segment, rb_firstorder_segment_dev) against a float64 NumPy
oracle on the same ROI vector: the order statistics bit for bit, every sum within 1e-12 of the same expression on absolute
values, and the reference's baseline columns within 1e-9."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN
from pyradiomics_b200 import featureclasses as FC, image as I, voxel

pytestmark = pytest.mark.gpu

EPS = np.spacing(1)
EXACT = ("Minimum", "Maximum", "Range", "10Percentile", "90Percentile", "InterquartileRange", "Median")


def oracle(x, lev, shift=0.0, vv=1.0):
    """(features, summation scale S_f) of the ROI vector x (float64) and its levels, as the reference's firstorder.py"""
    x = np.sort(np.asarray(x, np.float64))
    n = x.size
    sh = x + shift
    en = np.sum(sh ** 2)
    mean = x.mean()
    d = x - mean
    m2, m3, m4 = np.mean(d ** 2), np.mean(d ** 3), np.mean(d ** 4)
    m2s = 1.0 if m2 == 0 else m2
    p10, p90 = np.percentile(x, 10), np.percentile(x, 90)
    kept = x[(x >= p10) & (x <= p90)]
    _, cnt = np.unique(lev, return_counts=True)
    p = cnt / cnt.sum()
    with np.errstate(invalid="ignore", divide="ignore"):
        rmad = np.mean(np.abs(kept - kept.mean())) if kept.size else np.nan
        f = {"10Percentile": p10, "90Percentile": p90, "Energy": en, "Entropy": -np.sum(p * np.log2(p + EPS)),
             "InterquartileRange": np.percentile(x, 75) - np.percentile(x, 25), "Kurtosis": m4 / m2s ** 2,
             "Maximum": x[-1], "MeanAbsoluteDeviation": np.mean(np.abs(d)), "Mean": mean, "Median": np.median(x),
             "Minimum": x[0], "Range": x[-1] - x[0], "RobustMeanAbsoluteDeviation": rmad,
             "RootMeanSquared": np.sqrt(en / n), "Skewness": m3 / m2s ** 1.5, "TotalEnergy": en * vv,
             "Uniformity": np.sum(p ** 2), "Variance": m2}
        ax = np.abs(x)
        s = {"Mean": ax.mean(), "Energy": en, "TotalEnergy": en * vv, "RootMeanSquared": f["RootMeanSquared"],
             "Variance": m2, "MeanAbsoluteDeviation": ax.mean(),
             "RobustMeanAbsoluteDeviation": np.abs(kept).mean() if kept.size else 0.0,
             "Skewness": np.mean(np.abs(d) ** 3) / m2s ** 1.5, "Kurtosis": m4 / m2s ** 2, "Entropy": 1.0, "Uniformity": 1.0}
    return f, s


def check(got, x, lev, shift=0.0, vv=1.0, what=""):
    exp, scale = oracle(x, lev, shift, vv)
    assert list(got) == FC.RadiomicsFirstOrder.NAMES
    for k, v in exp.items():
        g = float(got[k])
        if k in EXACT:
            assert g == v, (what, k, g, v)                     # == : bit for bit except the sign of a zero
        elif np.isnan(v):
            assert np.isnan(g), (what, k, g)
        else:
            assert abs(g - v) <= 1e-12 * scale[k], (what, k, g, v, scale[k])


def run(img, roi, Ng_levels=None, binWidth=25, shift=0.0, spacing_zyx=(1.0, 1.0, 1.0), **bin_kw):
    """binned on the device like the pipeline, then the reduction; returns (features, ROI vector, ROI levels)"""
    img_t = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    roi_t = torch.from_numpy(np.ascontiguousarray(roi).astype(np.uint8)).cuda()
    _, _, lev, _, _ = voxel.discretize(img_t, roi_t, binWidth=binWidth, **bin_kw)
    got = voxel.firstorder_segment(img_t, lev, roi_t, voxelArrayShift=shift, spacing_zyx=spacing_zyx)
    lev_h = lev.cpu().numpy().astype(np.int64)
    m = np.asarray(roi) != 0
    return got, np.asarray(img)[m].astype(np.float64), lev_h[m]


def ellipsoid(shape, frac=0.8, seed=0):
    g = np.meshgrid(*[np.linspace(-1, 1, s) for s in shape], indexing="ij")
    r = sum(a ** 2 for a in g)
    rng = np.random.default_rng(seed)
    return (r < frac) & (rng.random(shape) < 0.97)


DTYPES = (np.int16, np.int32, np.float32, np.float64, np.uint8, np.int64)


@pytest.mark.parametrize("n", [1, 2, 3, 10, 11])
@pytest.mark.parametrize("dt", DTYPES)
def test_small_rois_every_pixel_type(n, dt):
    rng = np.random.default_rng(n)
    img = rng.integers(0 if dt == np.uint8 else -50, 120, (4, 5, 6)).astype(dt)
    if np.dtype(dt).kind == "f":
        img = (img * 0.37).astype(dt)
    roi = np.zeros(img.shape, bool)
    roi.reshape(-1)[rng.choice(img.size, n, replace=False)] = True
    got, x, lev = run(img, roi, binWidth=5)
    check(got, x, lev, what=(n, dt))


@pytest.mark.parametrize("case", ["all_equal", "two_values", "dups_at_ranks", "signed_zeros", "negative"])
def test_ties_and_signs(case):
    rng = np.random.default_rng(1)
    shape = (9, 10, 11)
    if case == "all_equal":
        img = np.full(shape, -7.25)
    elif case == "two_values":
        img = np.where(rng.random(shape) < 0.3, -3.0, 4.5)
    elif case == "dups_at_ranks":
        img = np.round(rng.normal(0, 2, shape)) * 0.5
    elif case == "signed_zeros":
        img = np.where(rng.random(shape) < 0.5, -0.0, 0.0) + np.where(rng.random(shape) < 0.2, 1.0, 0.0)
    else:
        img = -np.abs(rng.normal(100, 30, shape))
    roi = ellipsoid(shape, 0.9, 2)
    got, x, lev = run(img, roi, binCount=16)
    check(got, x, lev, what=case)


def test_shift_spacing_and_16bit_levels():
    rng = np.random.default_rng(3)
    img = rng.integers(-2000, 3000, (20, 30, 40)).astype(np.int16)
    roi = ellipsoid(img.shape, 0.95, 3)
    sp = (2.5, 0.75, 0.6)
    got, x, lev = run(img, roi, binWidth=1, shift=2000, spacing_zyx=sp)
    assert lev.max() > 255
    check(got, x, lev, shift=2000.0, vv=float(np.multiply.reduce(np.array(sp)[::-1])))


def test_two_dimensional_image():
    rng = np.random.default_rng(4)
    img = rng.normal(10, 5, (37, 41))
    roi = ellipsoid(img.shape, 0.7, 4)
    got, x, lev = run(img, roi, binWidth=2, shift=3, spacing_zyx=(0.5, 0.8))
    check(got, x, lev, shift=3.0, vv=0.8 * 0.5)


def test_ragged_ellipsoid_and_full_256_cube():
    rng = np.random.default_rng(5)
    img = rng.integers(-1000, 2000, (257, 263, 271)).astype(np.int16)
    roi = ellipsoid(img.shape, 0.6, 5)
    got, x, lev = run(img, roi, binWidth=25)
    check(got, x, lev, what="ellipsoid")
    img = (rng.normal(0, 1, (256, 256, 256)) * 300).astype(np.float32)
    roi = np.ones(img.shape, bool)
    got, x, lev = run(img, roi, binCount=64)
    check(got, x, lev, what="full")


def test_reference_baselines():
    cases = np.load(os.path.join(GOLDEN, "segment_cases.npz"))
    extra = json.load(open(os.path.join(GOLDEN, "segment_expect_extra.json")))
    masks = np.load(os.path.join(GOLDEN, "segment_extra.npz"))
    cols = dict(json.load(open(os.path.join(GOLDEN, "segment_expect_firstorder.json"))))
    cols.update(extra["firstorder"])
    assert len(cols) == 15
    for test, e in cols.items():
        c = e["case"]
        img = cases[c + "_image"]
        m = masks[test + "_mask"] if test + "_mask" in masks.files else cases[c + "_mask"]
        if "normalize" in e:
            n = e["normalize"]
            img = (img.astype(np.float64) - n["mean"]) / n["std"] * n["scale"]
        s = e["settings"]
        roi = m == s.get("label", 1)
        sp_zyx = tuple(cases[c + "_spacing"])[::-1]
        img_t = torch.from_numpy(np.ascontiguousarray(img)).cuda()
        dev = FC.DeviceImage(img_t, torch.from_numpy(roi.astype(np.uint8)).cuda(), 1, True, s)
        got = voxel.firstorder_segment(img_t, dev.levels, dev.mask_dev, voxelArrayShift=s.get("voxelArrayShift", 0),
                                       spacing_zyx=sp_zyx)
        for f, v in e["features"].items():
            assert abs(float(got[f]) - v) <= 1e-9 * max(abs(v), 1e-12), (test, f, float(got[f]), v)


def test_empty_roi_raises():
    img = torch.zeros((3, 4, 5), dtype=torch.int16, device="cuda")
    lev = torch.zeros((3, 4, 5), dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError):
        voxel.firstorder_segment(img, lev, torch.zeros_like(lev))


def test_side_stream_and_repeat_are_bit_identical():
    rng = np.random.default_rng(6)
    img_h = rng.normal(50, 20, (64, 70, 80))
    roi_h = ellipsoid(img_h.shape, 0.8, 6)
    ref, x, lev_h = run(img_h, roi_h, binWidth=3, shift=7)
    check(ref, x, lev_h, shift=7.0)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        img = torch.empty(img_h.shape, dtype=torch.float64, device="cuda")
        img.copy_(torch.from_numpy(img_h), non_blocking=True)
        roi = torch.from_numpy(roi_h.astype(np.uint8)).cuda(non_blocking=True)
        _, _, lev, _, _ = voxel.discretize(img, roi, binWidth=3)
        got = voxel.firstorder_segment(img, lev, roi, voxelArrayShift=7)
        again = voxel.firstorder_segment(img, lev, roi, voxelArrayShift=7)
    for k in ref:
        assert np.float64(got[k]).tobytes() == np.float64(ref[k]).tobytes(), k
        assert np.float64(again[k]).tobytes() == np.float64(ref[k]).tobytes(), k
