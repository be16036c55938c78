"""Generates tests/golden/preprocess_* FROM THE REFERENCE ITSELF: its own resegmentMask and normalizeImage
(radiomics/imageoperations.py:615-742).

Run in the build container only (needs /root/reference):  python tests/golden/make_golden_preprocess.py

* preprocess_resegment.npz / .json: resegmentMask on thirteen image / mask / setting cases (absolute mode with one, two
  and unsorted thresholds; relative mode on int16 and float32; sigma mode on int16, float32 and float64; label 2 of a
  multi-label mask; a uint8 image; a float32 voxel equal to a threshold only in float32; a range that keeps no voxel
  and a NaN in a relative-mode ROI, which both raise).  Stored: image, mask, the returned int mask or the error text,
  the thresholds and how close the nearest ROI voxel comes to one.
* preprocess_normalize.npz / .json: normalizeImage on six images.  SimpleITK is absent, so sitk.Normalize is a stub
  here that restates ITK's NormalizeImageFilter (StatisticsImageFilter: compensated sums, mean = S / N, sigma =
  sqrt((SS - S^2 / N) / (N - 1)); ShiftScaleImageFilter: (x + (-mean)) * (1 / sigma), float64); the reference's own
  removeOutliers and `image *= scale` code runs on its result.  The stub and the `*=` it needs exist only here.
* preprocess_breast1.npz: the whole breast1 image and label (the only bundled case small enough to commit whole).
* preprocess_baseline.json: resegmentRange / resegmentMode / normalize settings of the `_flatRegion`,
  `_resegmentation` and `_normalization` columns of the baseline CSVs, read from their diagnostics.
"""
from __future__ import annotations

import ast
import csv
import json
import logging
import math
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle"))
import ref_harness as rh  # noqa: E402

BASELINE_CSVS = ("firstorder", "glcm", "glrlm", "glszm", "gldm", "ngtdm")


class _ScalableImage(rh._Image):
    """the harness image plus the `image *= scale` normalizeImage applies (SimpleITK multiplies by a constant)"""

    def __imul__(self, s):
        return _ScalableImage(self._arr * s, self._spacing)


_ITK_STATS = {}


def _itk_normalize(image):
    x = np.asarray(image._arr, dtype=np.float64)
    n = x.size
    s, ss = math.fsum(x.ravel()), math.fsum((x * x).ravel())
    mean = np.float64(s) / n
    with np.errstate(divide="ignore", invalid="ignore"):
        sigma = np.sqrt((np.float64(ss) - np.float64(s) * np.float64(s) / n) / (n - 1))
        _ITK_STATS.update(mean=float(mean), sigma=float(sigma))
        return _ScalableImage((x + (-mean)) * (np.float64(1.0) / sigma), image._spacing)


def resegment_cases():
    rng = np.random.default_rng(20261015)
    b1, m1, _ = rh.load_case("brain1")
    b2, m2, _ = rh.load_case("brain2")
    shp = (9, 14, 16)
    box = np.zeros(shp, bool)
    box[1:8, 2:12, 3:14] = True
    f32 = (rng.gamma(3.0, 40.0, shp) - 30).astype(np.float32)
    f64 = rng.normal(-200, 35, shp)
    labels = rng.integers(0, 4, shp).astype(np.uint8)
    lab_img = rng.integers(-500, 1500, shp).astype(np.int16)
    u8 = rng.integers(0, 256, shp).astype(np.uint8)
    tenth = rng.random(shp).astype(np.float32) * 0.2
    tenth[::3, ::4, ::5] = np.float32(0.1)                     # equal to the float32 threshold, above the float64 one
    f32_nan = f32.copy()
    f32_nan[4, 6, 7] = np.nan
    return {
        "abs_one": (b1, m1, {"resegmentRange": [300]}),
        "abs_two": (b1, m1, {"resegmentRange": [150, 700], "resegmentMode": "absolute"}),
        "abs_unsorted": (b1, m1, {"resegmentRange": [700, 150]}),
        "rel_i16": (b2, m2, {"resegmentRange": [0.3, 0.9], "resegmentMode": "relative"}),
        "rel_f32": (f32, box, {"resegmentRange": [0.25, 0.8], "resegmentMode": "relative"}),
        "sigma_i16": (b1, m1, {"resegmentRange": [-1.5, 1.5], "resegmentMode": "sigma"}),
        "sigma_f32": (f32, box, {"resegmentRange": [-1, 2], "resegmentMode": "sigma"}),
        "sigma_f64": (f64, box, {"resegmentRange": [-2, 1.25], "resegmentMode": "sigma"}),
        "label2": (lab_img, labels, {"resegmentRange": [-1, 1], "resegmentMode": "sigma", "label": 2}),
        "u8": (u8, box, {"resegmentRange": [40, 200]}),
        "f32_rounding": (tenth, np.ones(shp, bool), {"resegmentRange": [float(np.float32(0.1)) + 1e-12]}),
        "too_few": (b1, m1, {"resegmentRange": [int(b1[m1].max()) + 1]}),
        "rel_nan_f32": (f32_nan, box, {"resegmentRange": [0.5], "resegmentMode": "relative"}),
    }


def normalize_cases(breast1):
    rng = np.random.default_rng(20261016)
    f32 = rng.normal(10, 4, (8, 9, 10)).astype(np.float32)
    f32[0, 0, :3] = (80, -70, 45)                                # outliers beyond 2.5 sigma on both sides
    nan = rng.normal(0, 1, (5, 6, 7))
    nan[2, 3, 4] = np.nan
    return {
        "breast1": (breast1, {"normalizeScale": 100, "removeOutliers": 3}),
        "i16_plain": (rng.integers(-1024, 2000, (7, 8, 9)).astype(np.int16), {}),
        "f32_outliers": (f32, {"normalizeScale": 50, "removeOutliers": 2.5}),
        "u8_2d": (rng.integers(0, 256, (20, 24)).astype(np.uint8), {"normalizeScale": 2}),
        "f64_nan": (nan, {"removeOutliers": 1}),
        "const_i32": (np.full((3, 4, 5), 7, np.int32), {"normalizeScale": 10}),
    }


def baseline_settings():
    out = {}
    for cname in BASELINE_CSVS:
        rows = list(csv.reader(open(os.path.join(rh.REF_ROOT, "data", "baseline", f"baseline_{cname}.csv"))))
        byname = {r[0]: r for r in rows}
        for col, test in enumerate(rows[0]):
            if not test.endswith(("_flatRegion", "_resegmentation", "_normalization")):
                continue
            s = ast.literal_eval(byname["diagnostics_Configuration_Settings"][col])
            entry = {k: s.get(k) for k in ("resegmentRange", "resegmentMode", "normalize", "normalizeScale",
                                           "removeOutliers", "label")}
            entry["case"] = byname["diagnostics_Configuration_TestCase"][col]
            assert out.setdefault(test, entry) == entry, (test, cname)       # the same settings in every CSV
    return out


def main():
    rh.load_reference()
    import SimpleITK as sitk  # the stub ref_harness installs
    from radiomics import imageoperations as rio
    logging.getLogger("radiomics").setLevel(logging.ERROR)

    arrays, meta = {}, {}
    for case, (img, msk, kw) in resegment_cases().items():
        arrays[f"{case}_image"], arrays[f"{case}_mask"] = img, msk.astype(np.uint8) if msk.dtype == bool else msk
        entry = {"kwargs": kw, "dtype": img.dtype.name}
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", RuntimeWarning)
                out = sitk.GetArrayFromImage(rio.resegmentMask(sitk.GetImageFromArray(img), sitk.GetImageFromArray(msk),
                                                               **kw))
            assert out.dtype == np.int64
            arrays[f"{case}_out"] = out
            entry["kept"] = int((out != 0).sum())
            roi = msk == kw.get("label", 1)
            vals = img[roi].astype(np.float64)
            mode = kw.get("resegmentMode", "absolute")
            srt = sorted(kw["resegmentRange"])
            if mode == "relative":
                ts = [np.max(img[roi]) * t for t in srt]
            elif mode == "sigma":
                ts = [np.mean(img[roi]) + np.std(img[roi]) * t for t in srt]
            else:
                ts = srt
            entry["thresholds"] = [float(t) for t in ts]
            # how close the nearest ROI voxel comes to a threshold, relative.  Sigma-mode thresholds come from sums whose
            # order differs on the device: > 1e-9 for an integer image, > 1e-5 for a float one (the device rounds a
            # float64 mean / std to float32 where NumPy sums in float32)
            gap = min(float(np.min(np.abs(vals - float(t)) / max(abs(float(t)), 1e-300))) for t in ts)
            entry["nearest_relative_gap"] = gap
            if mode == "sigma":
                assert gap > (1e-5 if img.dtype.kind == "f" else 1e-9), (case, gap)
        except ValueError as e:
            entry["error"] = str(e)
        meta[case] = entry
        print("resegment", case, img.dtype, entry.get("kept"), entry.get("error", ""))
    np.savez_compressed(os.path.join(HERE, "preprocess_resegment.npz"), **arrays)
    json.dump(meta, open(os.path.join(HERE, "preprocess_resegment.json"), "w"), indent=1, sort_keys=True)

    full, _ = rh.read_nrrd(os.path.join(rh.REF_ROOT, "data", "breast1_image.nrrd"))
    lab, _ = rh.read_nrrd(os.path.join(rh.REF_ROOT, "data", "breast1_label.nrrd"))
    np.savez_compressed(os.path.join(HERE, "preprocess_breast1.npz"), image=full, label=lab.astype(np.uint8))

    sitk.Normalize = _itk_normalize
    sitk.GetImageFromArray = _ScalableImage                  # the outlier branch rebuilds the image from its array
    arrays, meta = {}, {}
    for case, (img, kw) in normalize_cases(np.ascontiguousarray(full)).items():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            out = sitk.GetArrayFromImage(rio.normalizeImage(_ScalableImage(img), **kw))
        assert out.dtype == np.float64 and out.shape == img.shape
        if case != "breast1":
            arrays[f"{case}_image"] = img
        arrays[f"{case}_out"] = out
        meta[case] = {"kwargs": kw, "dtype": img.dtype.name, "itk_mean": _ITK_STATS["mean"],
                      "itk_sigma": _ITK_STATS["sigma"]}
        print("normalize", case, img.dtype, img.shape)
    np.savez_compressed(os.path.join(HERE, "preprocess_normalize.npz"), **arrays)
    json.dump(meta, open(os.path.join(HERE, "preprocess_normalize.json"), "w"), indent=1, sort_keys=True)

    base = baseline_settings()
    json.dump(base, open(os.path.join(HERE, "preprocess_baseline.json"), "w"), indent=1, sort_keys=True)
    for test, e in sorted(base.items()):
        print("baseline", test, e)
    for f in ("preprocess_resegment.npz", "preprocess_normalize.npz", "preprocess_breast1.npz"):
        size = os.path.getsize(os.path.join(HERE, f))
        assert size < 1 << 20, f
        print(f, size, "bytes")


if __name__ == "__main__":
    main()
