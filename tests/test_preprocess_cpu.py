"""Normalisation and resegmentation without a GPU: the NumPy oracle (oracle/preprocess_np.py) against the reference's
own resegmentMask / normalizeImage runs (tests/golden/preprocess_*) and the resegmented baseline masks, and the
product's host threshold logic (dtype rules, sorting, the relative-mode NaN rule, error texts) against the oracle."""
import json
import os

import numpy as np
import pytest
import torch

import preprocess_np as O
from helpers import GOLDEN
from pyradiomics_b200 import imageoperations as IO


def load_resegment():
    return np.load(os.path.join(GOLDEN, "preprocess_resegment.npz")), \
        json.load(open(os.path.join(GOLDEN, "preprocess_resegment.json")))


def load_normalize():
    """{case: (image, reference output, kwargs, (ITK stub mean, sigma))}"""
    z = np.load(os.path.join(GOLDEN, "preprocess_normalize.npz"))
    meta = json.load(open(os.path.join(GOLDEN, "preprocess_normalize.json")))
    whole = np.load(os.path.join(GOLDEN, "preprocess_breast1.npz"))
    return {c: (whole["image"] if c == "breast1" else z[c + "_image"], z[c + "_out"], e["kwargs"],
                (e["itk_mean"], e["itk_sigma"])) for c, e in meta.items()}


def baseline_resegmentations():
    """[(test, case, resegmentRange, resegmentMode)] of the ten `_flatRegion` / `_resegmentation` baseline columns"""
    base = json.load(open(os.path.join(GOLDEN, "preprocess_baseline.json")))
    return [(t, e["case"], e["resegmentRange"], e["resegmentMode"] or "absolute") for t, e in sorted(base.items())
            if e["resegmentRange"] is not None]


def assert_ulps(got, ref, max_ulp, what):
    nan = np.isnan(ref)
    np.testing.assert_array_equal(np.isnan(got), nan, err_msg=f"{what}: NaN positions")
    if max_ulp == 0:
        np.testing.assert_array_equal(got[~nan], ref[~nan], err_msg=what)
    else:
        np.testing.assert_array_max_ulp(got[~nan], ref[~nan], maxulp=max_ulp)


def test_goldens_cover_the_issue_cases():
    z, meta = load_resegment()
    assert {e["dtype"] for e in meta.values()} >= {"int16", "float32", "float64", "uint8"}
    modes = {(e["kwargs"].get("resegmentMode", "absolute"), e["dtype"]) for e in meta.values()}
    assert {("relative", "int16"), ("relative", "float32"), ("sigma", "int16"), ("sigma", "float32"),
            ("sigma", "float64")} <= modes
    assert meta["label2"]["kwargs"]["label"] == 2 and set(np.unique(z["label2_mask"])) == {0, 1, 2, 3}
    assert "error" in meta["too_few"] and "error" in meta["rel_nan_f32"]
    b = np.load(os.path.join(GOLDEN, "preprocess_breast1.npz"))
    assert b["image"].shape == (21, 120, 45) and b["image"].dtype == np.int16
    assert len(baseline_resegmentations()) == 10


@pytest.mark.parametrize("case", sorted(load_resegment()[1]))
def test_oracle_reproduces_the_reference_resegmentations(case):
    z, meta = load_resegment()
    e = meta[case]
    kw = dict(e["kwargs"])
    if "error" in e:
        with pytest.raises(ValueError) as exc:
            O.resegment(z[case + "_image"], z[case + "_mask"], **kw)
        assert str(exc.value) == e["error"]
        return
    got, ts = O.resegment(z[case + "_image"], z[case + "_mask"], **kw)
    ref = z[case + "_out"]
    np.testing.assert_array_equal(got, ref != 0)
    assert set(np.unique(ref[ref != 0])) == {kw.get("label", 1)}
    assert [float(t) for t in ts] == e["thresholds"]


def test_float32_threshold_rounding_case_depends_on_the_comparison_dtype():
    z, meta = load_resegment()
    img, t = z["f32_rounding_image"], meta["f32_rounding"]["kwargs"]["resegmentRange"][0]
    at = img == np.float32(0.1)
    assert at.any() and (z["f32_rounding_out"][at] == 1).all()                  # NumPy compares in float32: kept
    assert not (img[at].astype(np.float64) >= t).any()                           # a float64 comparison drops them


@pytest.mark.parametrize("case", sorted(load_normalize()))
def test_oracle_reproduces_the_reference_normalisations(case):
    """with the ITK stub's statistics the oracle's arithmetic is the reference's to the bit; its own two-pass statistics
    (NumPy's) differ from the stub's one-pass ones by at most 1e-12 relative"""
    img, ref, kw, (mean, sigma) = load_normalize()[case]
    scale, outliers = kw.get("normalizeScale", 1), kw.get("removeOutliers")
    assert_ulps(O.normalize(img, scale, outliers, stats=(mean, sigma)), ref, 0, case)
    m2, s2 = O.whole_image_stats(img)
    if np.isfinite(sigma) and sigma > 0:
        assert abs(m2 - mean) <= 1e-12 * max(abs(mean), 1.0) and abs(s2 - sigma) <= 1e-12 * sigma, (case, m2, mean, s2, sigma)
        np.testing.assert_allclose(O.normalize(img, scale, outliers), ref, rtol=1e-12, atol=1e-12 * abs(scale))
    else:
        assert_ulps(O.normalize(img, scale, outliers), ref, 0, case)            # NaN / constant images: all NaN


def test_breast1_whole_image_statistics_are_the_baselines():
    img = np.load(os.path.join(GOLDEN, "preprocess_breast1.npz"))["image"]
    n = json.load(open(os.path.join(GOLDEN, "segment_expect_extra.json")))["glcm"]["breast1_normalization"]["normalize"]
    mean, std = O.whole_image_stats(img)
    assert mean == n["mean"] and std == n["std"]


@pytest.mark.parametrize("test,case,rng,mode", baseline_resegmentations())
def test_oracle_reproduces_the_baseline_resegmented_masks(test, case, rng, mode):
    cases = np.load(os.path.join(GOLDEN, "segment_cases.npz"))
    masks = np.load(os.path.join(GOLDEN, "segment_extra.npz"))
    got, _ = O.resegment(cases[case + "_image"], cases[case + "_mask"], rng, mode)
    np.testing.assert_array_equal(got, masks[test + "_mask"])


# ---------------------------------------------------------------------------------------------------- host logic
def host_resegment(img, mask, rng, mode, label=1):
    """the product's thresholds (imageoperations.resegment_thresholds) from NumPy's ROI statistics, compared in float64
    the way rb_resegment_dev compares; raises like resegment_mask_device"""
    roi = mask == label
    vals = img[roi]
    stats = {}
    if mode == "relative":
        stats["max_gl"] = np.max(vals)
    elif mode == "sigma":
        stats["mean_gl"], stats["sd_gl"] = np.mean(vals), np.std(vals)
    _, cmp = IO.resegment_thresholds(img.dtype.type, rng, mode, **stats)
    x = img.astype(np.float64)
    keep = roi & (x >= cmp[0])
    if len(cmp) == 2:
        keep &= x <= cmp[1]
    if keep.sum() <= 1:
        raise ValueError(f"Resegmentation excluded too many voxels with label {label} "
                         f"(retained {keep.sum()} voxel(s))! Cannot extract features")
    return keep


def sweep_images():
    rng = np.random.default_rng(44)
    shp = (6, 7, 8)
    base = rng.normal(100, 60, shp)
    tenths = np.round(rng.random(shp), 1)                # many voxels on a float32-rounded decimal
    out = []
    for dt in (np.int16, np.int32, np.int64, np.uint8, np.float32, np.float64):
        if np.issubdtype(dt, np.integer):
            info = np.iinfo(dt)
            out.append((np.dtype(dt).name, np.clip(np.round(base), max(info.min, -1000), min(info.max, 1000)).astype(dt)))
        else:
            out.append((np.dtype(dt).name, base.astype(dt)))
            out.append((np.dtype(dt).name + " tenths", tenths.astype(dt)))
    return out


RANGES = {
    "absolute": ([60], [150, 40], [0.3], [0.1, 0.7], [100.5, 20], [-5]),
    "relative": ([0.5], [0.8, 0.2], [1], [0, 1], [0.3, 0.65]),
    "sigma": ([-1, 1], [0], [1.5, -0.5], [-3, 3]),
}


@pytest.mark.parametrize("mode", sorted(RANGES))
def test_host_threshold_logic_equals_the_oracle(mode):
    rng = np.random.default_rng(3)
    n = 0
    for what, img in sweep_images():
        for label in (1, 3):
            mask = rng.integers(0, 4, img.shape).astype(np.uint8)
            for r in RANGES[mode]:
                try:
                    ref, _ = O.resegment(img, mask, r, mode, label)
                except ValueError as e:
                    with pytest.raises(ValueError) as exc:
                        host_resegment(img, mask, r, mode, label)
                    assert str(exc.value) == str(e)
                    continue
                np.testing.assert_array_equal(host_resegment(img, mask, r, mode, label), ref,
                                              err_msg=f"{what} {mode} {r} label {label}")
                n += 1
    assert n > 30


def test_relative_mode_nan_keeps_nothing():
    img = np.linspace(1, 2, 60).astype(np.float32).reshape(3, 4, 5)
    img[1, 1, 1] = np.nan
    mask = np.ones(img.shape, np.uint8)
    with pytest.raises(ValueError, match=r"retained 0 voxel"):
        O.resegment(img, mask, [0.5], "relative")
    with pytest.raises(ValueError, match=r"retained 0 voxel"):
        host_resegment(img, mask, [0.5], "relative")


def test_threshold_dtypes_follow_numpy():
    f32, i16 = np.float32, np.int16
    assert IO._comparison_value(f32, 0.1 + 1e-12) == float(np.float32(0.1))
    assert IO._comparison_value(np.float64, 0.1 + 1e-12) == 0.1 + 1e-12
    assert IO._comparison_value(i16, 0.5) == 0.5
    assert IO._comparison_value(np.uint8, -5) == -5.0 and IO._comparison_value(i16, 10 ** 6) == 1e6
    ts, _ = IO.resegment_thresholds(f32, [0.8, 0.2], "relative", max_gl=np.float32(3.0))
    assert [type(t) for t in ts] == [np.float32, np.float32]
    ts, _ = IO.resegment_thresholds(i16, [2, 1], "relative", max_gl=np.int16(30))
    assert ts == [30, 60] and type(ts[0]) is np.int16
    ts, _ = IO.resegment_thresholds(i16, [-1, 1], "sigma", mean_gl=np.float64(10), sd_gl=np.float64(2))
    assert ts == [8.0, 12.0]
    assert IO._stat_type(np.float32) is np.float32 and IO._stat_type(np.int16) is np.float64


@pytest.mark.parametrize("rng,mode,text", [
    (None, "absolute", "resegmentRange is None."),
    ([], "absolute", "Length 0 is not allowed for resegmentRange"),
    ([1, 2, 3], "absolute", "Length 3 is not allowed for resegmentRange"),
    ([1], "percentile", "Resegment mode percentile not recognized."),
])
def test_argument_errors_raise_the_reference_texts_before_any_device_work(rng, mode, text):
    img = torch.zeros((2, 3, 4), dtype=torch.int16)
    mask = torch.ones((2, 3, 4), dtype=torch.uint8)
    with pytest.raises(ValueError) as exc:
        IO.resegment_mask_device(img, mask, rng, mode)
    assert str(exc.value) == text
    with pytest.raises(ValueError) as exc:
        O.resegment(img.numpy(), mask.numpy(), rng, mode)
    assert str(exc.value) == text
