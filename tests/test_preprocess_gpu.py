"""Normalisation and resegmentation on the GPU (csrc/filters.cu roi_moments / normalize / resegment kernels): the ROI
moments against NumPy, the normalisation against the oracle bit for bit and against the reference's runs, the
resegmentation against every reference mask, the baseline `_normalization` / `_resegmentation` / `_flatRegion` columns
end to end, the opt-in pipeline steps, bit-reproducibility and the C entry points' argument checks."""
import ctypes as C
import json
import logging
import os

import numpy as np
import pytest
import torch

import preprocess_np as O
from helpers import GOLDEN, RTOL
from pyradiomics_b200 import _lib, featureclasses as FC, image as I, imageoperations as IO, pipeline as PP
from test_preprocess_cpu import assert_ulps, baseline_resegmentations, load_normalize, load_resegment

pytestmark = pytest.mark.gpu

DTYPES = (np.int16, np.int32, np.int64, np.uint8, np.float32, np.float64)
SIZES = (1, 255, 257, 1024 * 256 + 1)          # one voxel, a block - 1, a block + 1, past the fixed grid's 1024 blocks


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def moment_case(dt, n, seed):
    rng = np.random.default_rng(seed)
    if np.issubdtype(dt, np.integer):
        info = np.iinfo(dt)
        return rng.integers(max(info.min, -30000), min(info.max, 30000), n, endpoint=True).astype(dt)
    return (rng.normal(50, 400, n) * rng.choice([1, 1e-3], n)).astype(dt)


def np_moments(x, roi, ddof=0):
    v = x[roi].astype(np.float64)
    return v.size, int(np.isnan(v).sum()), v.mean(), v.std(ddof=ddof), v.max()


def assert_rel(got, ref, what, tol=1e-13):
    if np.isnan(ref):
        assert np.isnan(got), what
    else:
        assert abs(got - ref) <= tol * max(abs(ref), 1e-300), (what, got, ref)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("n", SIZES)
def test_roi_moments_match_numpy_and_repeat_bit_for_bit(dt, n):
    x = moment_case(dt, n, n)
    labels = np.random.default_rng(n + 1).integers(0, 3, n).astype(np.uint8)
    labels[0] = 2                                                   # the ROI of label 2 is never empty
    xt, mt = dev(x), dev(labels)
    for mask, label, roi in ((None, 1, np.ones(n, bool)), (mt, 2, labels == 2)):
        got = IO.roi_moments_device(xt, mask, label=label)
        ref = np_moments(x, roi)
        assert got[:2] == ref[:2]
        for k, what in ((2, "mean"), (3, "std"), (4, "max")):
            assert_rel(got[k], ref[k], f"{np.dtype(dt).name} n={n} label={label} {what}")
        again = IO.roi_moments_device(xt, mask, label=label)
        assert np.array(got, np.float64).tobytes() == np.array(again, np.float64).tobytes()


@pytest.mark.parametrize("dt", (np.float32, np.float64))
def test_roi_moments_with_nan(dt):
    x = moment_case(dt, 3000, 5)
    x[17] = np.nan
    mask = np.zeros(3000, np.uint8)
    mask[::2] = 1
    n, n_nan, mean, std, mx = IO.roi_moments_device(dev(x), dev(mask))
    assert (n, n_nan) == (1500, 0) and np.isfinite([mean, std, mx]).all()     # the NaN is outside the ROI
    n, n_nan, mean, std, mx = IO.roi_moments_device(dev(x))
    assert (n, n_nan) == (3000, 1) and np.isnan([mean, std, mx]).all()
    assert IO.roi_moments_device(dev(x), dev(np.zeros(3000, np.uint8)))[0] == 0


def test_breast1_whole_image_statistics():
    img = np.load(os.path.join(GOLDEN, "preprocess_breast1.npz"))["image"]
    ref = json.load(open(os.path.join(GOLDEN, "segment_expect_extra.json")))["glcm"]["breast1_normalization"]["normalize"]
    n, _, mean, std, _ = IO.roi_moments_device(dev(img), ddof=1)
    assert n == img.size
    assert_rel(mean, ref["mean"], "mean")
    assert_rel(std, ref["std"], "std")


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("scale,outliers", [(1, None), (100, None), (1, 2), (37.5, 1.5)])
def test_normalize_equals_oracle_bit_for_bit(dt, scale, outliers):
    x = moment_case(dt, 20000, 11).reshape(20, 25, 40)
    if np.issubdtype(dt, np.floating):
        x[3, 4, 5] = np.nan
    xt = dev(x)
    _, _, mean, std, _ = IO.roi_moments_device(xt, ddof=1)
    got = IO.normalize_image_device(xt, scale, outliers).cpu().numpy()
    assert got.dtype == np.float64 and got.shape == x.shape
    assert_ulps(got, O.normalize(x, scale, outliers, stats=(mean, std)), 0, f"{np.dtype(dt).name} {scale} {outliers}")
    if np.issubdtype(dt, np.floating):
        assert np.isnan(got).all()                                  # a NaN makes the mean NaN: ITK's sums
    else:
        np.testing.assert_allclose(got, O.normalize(x, scale, outliers), rtol=1e-13, atol=1e-13 * scale)
    if outliers is not None and not np.isnan(got).all():
        assert np.abs(got).max() <= outliers * scale


@pytest.mark.parametrize("case", sorted(load_normalize()))
def test_normalize_matches_the_reference_runs(case):
    img, ref, kw, (mean, sigma) = load_normalize()[case]
    scale, outliers = kw.get("normalizeScale", 1), kw.get("removeOutliers")
    xt = dev(img)
    assert_ulps(IO.normalize_image_device(xt, scale, outliers, stats=(mean, sigma)).cpu().numpy(), ref, 0, case)
    im = IO.normalizeImage(I.ArrayImage(img, (0.5, 0.7, 1.1)[:img.ndim]), **kw)
    got = I.as_array(im)
    assert got.dtype == np.float64 and im.GetSpacing() == (0.5, 0.7, 1.1)[:img.ndim]
    if np.isnan(ref).all():
        assert np.isnan(got).all()
    else:
        np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-12 * scale)


def test_normalize_constant_image_is_nan():
    got = IO.normalize_image_device(dev(np.full((3, 4, 5), 9, np.int16)), 10, 3).cpu().numpy()
    assert np.isnan(got).all()


@pytest.mark.parametrize("case", sorted(load_resegment()[1]))
def test_resegment_matches_the_reference_runs(case):
    z, meta = load_resegment()
    e = meta[case]
    img, mask, kw = z[case + "_image"], z[case + "_mask"], dict(e["kwargs"])
    mode = kw.get("resegmentMode", "absolute")
    if mode == "sigma" and "error" not in e:
        # sums taken in another order: no ROI voxel may sit this close to a threshold (float: float32 vs float64 sums)
        assert e["nearest_relative_gap"] > (1e-5 if img.dtype.kind == "f" else 1e-9), e["nearest_relative_gap"]
    image = I.ArrayImage(img, (0.8, 0.9, 2.0))
    maskimg = I.ArrayImage(mask, (0.8, 0.9, 2.0))
    if "error" in e:
        with pytest.raises(ValueError) as exc:
            IO.resegmentMask(image, maskimg, **kw)
        assert str(exc.value) == e["error"]
        return
    out = IO.resegmentMask(image, maskimg, **kw)
    got = I.as_array(out)
    assert got.dtype == np.int64 and out.GetSpacing() == maskimg.GetSpacing()
    np.testing.assert_array_equal(got, z[case + "_out"])
    m, kept, ts = IO.resegment_mask_device(dev(img), dev(mask), kw["resegmentRange"], mode, kw.get("label", 1))
    assert kept == e["kept"] == int(m.sum().item())
    if mode == "sigma":                                  # device statistics: other summation order
        np.testing.assert_allclose([float(t) for t in ts], e["thresholds"], rtol=1e-5 if img.dtype == np.float32 else 1e-12)
    else:
        assert [float(t) for t in ts] == e["thresholds"]


@pytest.mark.parametrize("test,case,rng,mode", baseline_resegmentations())
def test_resegment_reproduces_the_baseline_masks(test, case, rng, mode):
    cases = np.load(os.path.join(GOLDEN, "segment_cases.npz"))
    masks = np.load(os.path.join(GOLDEN, "segment_extra.npz"))
    m, kept, _ = IO.resegment_mask_device(dev(cases[case + "_image"]), dev(cases[case + "_mask"]), rng, mode)
    np.testing.assert_array_equal(m.cpu().numpy().astype(bool), masks[test + "_mask"])
    assert kept == int(masks[test + "_mask"].sum())


def test_resegment_logs_like_the_reference(caplog):
    z, _ = load_resegment()
    with caplog.at_level(logging.DEBUG, logger="radiomics.imageoperations"):
        IO.resegmentMask(I.ArrayImage(z["sigma_i16_image"]), I.ArrayImage(z["sigma_i16_mask"]), resegmentRange=[-1.5, 1.5],
                         resegmentMode="sigma")
        IO.normalizeImage(I.ArrayImage(z["sigma_i16_image"]), normalizeScale=3, removeOutliers=2)
    msgs = [r.getMessage() for r in caplog.records if r.name == "radiomics.imageoperations"]
    assert msgs[0] == "Resegmenting mask (range [-1.5, 1.5], mode sigma)"
    assert msgs[1].startswith("Resegmenting in sigma mode, mean ") and ", std " in msgs[1]
    assert msgs[2].startswith("Applying lower threshold (") and msgs[3].startswith("Applying upper threshold (")
    assert msgs[4].startswith("Resegmentation complete, new size: ")
    assert msgs[5:] == ["Normalizing image with scale 3", "Removing outliers > 2 standard deviations"]


# ------------------------------------------------------------------------------ baseline columns end to end
def _crop_of_whole_breast1():
    b = np.load(os.path.join(GOLDEN, "preprocess_breast1.npz"))
    idx = np.where(b["label"] == 1)
    return b["image"], tuple(slice(int(i.min()), int(i.max()) + 1) for i in idx)


def preprocessed_columns():
    """(test, class, preprocessed crop, mask, spacing, settings, expected features) of the 50 texture and 10 first-order
    `_normalization` / `_resegmentation` columns and the 25 `_flatRegion` columns, the preprocessing run on the device"""
    cases = np.load(os.path.join(GOLDEN, "segment_cases.npz"))
    expect = json.load(open(os.path.join(GOLDEN, "segment_expect_extra.json")))
    base = json.load(open(os.path.join(GOLDEN, "preprocess_baseline.json")))
    out = []
    for cname, cols in sorted(expect.items()):
        for test, e in sorted(cols.items()):
            c, b = e["case"], base[test]
            img, mask = cases[c + "_image"], cases[c + "_mask"]
            if b["normalize"]:
                if c == "breast1":                          # the whole image is committed: its statistics come from the GPU
                    whole, crop = _crop_of_whole_breast1()
                    assert np.array_equal(whole[crop], img)
                    img = IO.normalize_image_device(dev(whole), b["normalizeScale"], b["removeOutliers"]).cpu().numpy()[crop]
                else:
                    n = e["normalize"]
                    img = IO.normalize_image_device(dev(img), b["normalizeScale"], b["removeOutliers"],
                                                    stats=(n["mean"], n["std"])).cpu().numpy()
            if b["resegmentRange"] is not None:
                m, _, _ = IO.resegment_mask_device(dev(img), dev(mask), b["resegmentRange"], b["resegmentMode"] or "absolute")
                mask = m.cpu().numpy()
            out.append((test, cname, img, mask.astype(np.uint8), cases[c + "_spacing"], e["settings"], e["features"]))
    return out


def test_baseline_columns_through_device_preprocessing():
    cols = preprocessed_columns()
    kinds = {}
    for test, cname, img, mask, sp, settings, feats in cols:
        kinds[test.split("_", 1)[1]] = kinds.get(test.split("_", 1)[1], 0) + 1
        cls = FC.RadiomicsFirstOrder if cname == "firstorder" else FC.FEATURE_CLASSES[cname]
        got = cls(I.ArrayImage(img, sp), I.ArrayImage(mask, sp), **settings).execute()
        for f, v in feats.items():
            assert abs(float(got[f]) - v) <= RTOL * max(abs(v), 1e-12), (cname, test, f, float(got[f]), v)
    assert kinds == {"normalization": 30, "resegmentation": 30, "flatRegion": 25}


# ------------------------------------------------------------------------------ pipeline, C ABI
def test_pipeline_preprocessing_equals_the_manual_chain():
    import scipy.ndimage as ndi
    rng = np.random.default_rng(21)
    x = (ndi.gaussian_filter(rng.normal(size=(12, 13, 14)), 1.2) * 400 + 100).astype(np.int16)
    m = (rng.random(x.shape) < 0.8).astype(np.uint8)
    xt, mt = dev(x), dev(m)
    norm, reseg = {"normalizeScale": 100, "removeOutliers": 3}, {"resegmentRange": [-2, 2], "resegmentMode": "sigma"}
    kw = dict(classes=("glcm", "gldm"), wavelet="coif1", sigmas=(1.0,), image_types=("square",), binWidth=5)

    def run(image, mask, **extra):
        got = {}
        info = PP.voxel_suite_with_filters(image, mask, consume=lambda n, c, t: got.__setitem__((n, c), t.cpu().numpy().copy()),
                                           **kw, **extra)
        return info, got

    info, got = run(xt, mt, normalize=norm, resegment=reseg)
    xn = IO.normalize_image_device(xt, 100, 3)
    mr, kept, _ = IO.resegment_mask_device(xn, (mt != 0).to(torch.uint8), [-2, 2], "sigma")
    assert 0 < kept < int(m.sum())
    info2, ref = run(xn, mr)
    assert info == info2 and got.keys() == ref.keys()
    for k in ref:
        assert got[k].tobytes() == ref[k].tobytes(), k
    info3, plain = run(xt, mt)
    info4, plain2 = run(xt, mt, normalize=None, resegment=None)
    assert info3 == info4 and all(plain[k].tobytes() == plain2[k].tobytes() for k in plain)
    assert [n for n, _, _ in info3] == [n for n, _, _ in info]


def test_preprocessing_is_bit_reproducible():
    x = dev(moment_case(np.float32, 300000, 4).reshape(60, 50, 100))
    m = dev((np.random.default_rng(2).random((60, 50, 100)) < 0.5).astype(np.uint8))
    a, b = IO.normalize_image_device(x, 100, 3), IO.normalize_image_device(x, 100, 3)
    assert torch.equal(a.view(torch.int64), b.view(torch.int64))
    r1, r2 = (IO.resegment_mask_device(x, m, [-1, 1], "sigma") for _ in range(2))
    assert torch.equal(r1[0], r2[0]) and r1[1] == r2[1] and r1[2] == r2[2]


def test_entry_points_reject_bad_arguments():
    L = _lib.lib()
    x = torch.zeros((4, 5, 6), dtype=torch.int16, device="cuda")
    m = torch.ones((4, 5, 6), dtype=torch.uint8, device="cuda")
    out8 = torch.empty((4, 5, 6), dtype=torch.uint8, device="cuda")
    outd = torch.empty((4, 5, 6), dtype=torch.float64, device="cuda")
    res = torch.empty(5, dtype=torch.float64, device="cuda")
    counts = torch.empty(2, dtype=torch.int64, device="cuda")
    scratch = torch.empty(IO._MOMENTS_SCRATCH_BYTES, dtype=torch.uint8, device="cuda")
    s, n, z = _lib.stream(), C.c_longlong(x.numel()), C.c_longlong(0)
    p, d = _lib.ptr, C.c_double
    mo = L.rb_roi_moments_dev
    assert mo(p(x), 0, p(m), n, 2, p(scratch), p(res), s) == _lib.RB_OK
    assert mo(p(x), 0, None, n, 1, p(scratch), p(res), s) == _lib.RB_OK
    for args in ((None, 0, p(m), n, 2, p(scratch), p(res)), (p(x), 0, p(m), n, 2, None, p(res)),
                 (p(x), 0, p(m), n, 2, p(scratch), None), (p(x), 7, p(m), n, 2, p(scratch), p(res)),
                 (p(x), -1, p(m), n, 2, p(scratch), p(res)), (p(x), 0, p(m), z, 2, p(scratch), p(res)),
                 (p(x), 0, p(m), n, 3, p(scratch), p(res)), (p(x), 0, p(m), n, 0, p(scratch), p(res))):
        assert mo(*args, s) == _lib.RB_ERR_ARG, args
    nz = L.rb_normalize_dev
    assert nz(p(x), 0, n, d(1.0), d(2.0), 1, d(3.0), d(1.0), p(outd), s) == _lib.RB_OK
    for args in ((None, 0, n), (p(x), 7, n), (p(x), 0, z)):
        assert nz(*args, d(1.0), d(2.0), 0, d(0.0), d(1.0), p(outd), s) == _lib.RB_ERR_ARG, args
    assert nz(p(x), 0, n, d(1.0), d(2.0), 0, d(0.0), d(1.0), None, s) == _lib.RB_ERR_ARG
    rs = L.rb_resegment_dev
    assert rs(p(x), 0, p(m), n, d(0.0), d(1.0), 2, p(out8), p(counts), s) == _lib.RB_OK
    for args in ((None, 0, p(m), n, d(0.0), d(1.0), 2, p(out8), p(counts)),
                 (p(x), 0, None, n, d(0.0), d(1.0), 2, p(out8), p(counts)),
                 (p(x), 0, p(m), n, d(0.0), d(1.0), 2, None, p(counts)),
                 (p(x), 0, p(m), n, d(0.0), d(1.0), 2, p(out8), None),
                 (p(x), 7, p(m), n, d(0.0), d(1.0), 2, p(out8), p(counts)),
                 (p(x), 0, p(m), z, d(0.0), d(1.0), 2, p(out8), p(counts)),
                 (p(x), 0, p(m), n, d(0.0), d(1.0), 0, p(out8), p(counts)),
                 (p(x), 0, p(m), n, d(0.0), d(1.0), 3, p(out8), p(counts))):
        assert rs(*args, s) == _lib.RB_ERR_ARG, args
    torch.cuda.synchronize()
    assert counts.tolist() == [120, 120]
