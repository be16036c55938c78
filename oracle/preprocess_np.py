"""NumPy restatement of the reference's two preprocessing steps (radiomics/imageoperations.py:615-742), the oracle of
csrc/filters.cu's roi_moments / normalize / resegment kernels.

* normalize: sitk.Normalize as ITK's NormalizeImageFilter computes it (StatisticsImageFilter's mean and sigma with
  N - 1 over the WHOLE image, then ShiftScale: shift -mean, scale 1 / sigma, float64), the clamp to +-removeOutliers
  and the multiplication by normalizeScale.  ITK is not available here, so the ShiftScale order and the float64 output
  type are as recalled; mean / std are NumPy's two-pass ones unless the caller supplies them.
* resegment: the thresholds of resegmentMask, computed from NumPy's np.max / np.mean / np.std of the ROI in the ROI's
  own dtype, and NumPy's comparisons of the ROI voxels with them."""
from __future__ import annotations

import numpy as np


def whole_image_stats(img):
    """(mean, std with N - 1) of every voxel, in float64"""
    x = np.asarray(img, dtype=np.float64)
    return float(x.mean()), float(x.std(ddof=1))


def normalize(img, scale=1, outliers=None, stats=None):
    """((x - mean) * (1 / std)), clamped to +-outliers (NaN stays NaN), times scale -> float64.  `stats` = (mean, std);
    None = whole_image_stats(img)."""
    mean, std = whole_image_stats(img) if stats is None else stats
    x = np.asarray(img, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        z = (x - mean) * (np.float64(1.0) / np.float64(std))
    if outliers is not None:
        z = np.where(z > outliers, np.float64(outliers), z)
        z = np.where(z < -outliers, -np.float64(outliers), z)
    return z * scale


def resegment(img, mask, resegmentRange, resegmentMode="absolute", label=1):
    """-> (boolean mask, thresholds): the ROI (mask == label) voxels within the thresholds, as resegmentMask keeps them.
    Raises resegmentMask's ValueErrors."""
    if resegmentRange is None:
        raise ValueError("resegmentRange is None.")
    k = len(resegmentRange)
    if k == 0 or k > 2:
        raise ValueError(f"Length {k} is not allowed for resegmentRange")
    roi = np.asarray(mask) == label
    vals = np.asarray(img)[roi]
    factors = sorted(resegmentRange)
    if resegmentMode == "absolute":
        ts = factors
    elif resegmentMode == "relative":
        top = np.max(vals)                                  # NaN in the ROI -> NaN thresholds -> nothing kept
        ts = [top * f for f in factors]
    elif resegmentMode == "sigma":
        mu, sd = np.mean(vals), np.std(vals)
        ts = [mu + sd * f for f in factors]
    else:
        raise ValueError(f"Resegment mode {resegmentMode} not recognized.")
    keep = vals >= ts[0]
    if k == 2:
        keep &= vals <= ts[1]
    out = np.zeros(roi.shape, dtype=bool)
    out[roi] = keep
    kept = int(keep.sum())
    if kept <= 1:
        raise ValueError(f"Resegmentation excluded too many voxels with label {label} "
                         f"(retained {kept} voxel(s))! Cannot extract features")
    return out, ts
