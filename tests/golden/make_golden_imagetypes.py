"""Generates tests/golden/imagetypes_*.npz FROM THE REFERENCE ITSELF: its own getSquareImage, getSquareRootImage,
getLogarithmImage and getExponentialImage (radiomics/imageoperations.py:973-1073) on seven small images.

Run in the build container only (needs /root/reference):  python tests/golden/make_golden_imagetypes.py

The generators run through oracle/ref_harness.py's SimpleITK stub (GetArrayFromImage, GetImageFromArray and
CopyInformation are all they use).  Stored per case: the image and the four float64 outputs under their yielded names.
getGradientImage has no golden: it is SimpleITK's GradientMagnitudeImageFilter, which cannot run here.
"""
from __future__ import annotations

import logging
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle"))
import ref_harness as rh  # noqa: E402

NAMES = ("square", "squareroot", "logarithm", "exponential")


def cases():
    rng = np.random.default_rng(20261016)
    img_b, _, _ = rh.load_case("brain1")
    ct = rng.integers(-40, 900, (14, 20, 22)).astype(np.int16)
    ct[:3] = -1024                                              # air: M = 1024 comes from the minimum
    f64 = np.round(rng.normal(0, 50, (10, 12, 14)), 1)
    f64[rng.random(f64.shape) < 0.2] = 0.0
    return {
        "brain1": np.ascontiguousarray(img_b[:, :40, :40]).astype(np.int16),
        "ct_i16": ct,
        "f32_small": (rng.random((9, 11, 13)) * 0.8 - 0.3).astype(np.float32),     # M < 1: exponential's c < 0
        "f64_signs": f64,
        "u8_2d": rng.integers(0, 256, (40, 50)).astype(np.uint8),
        "unit_i32": rng.integers(-1, 2, (8, 9, 10)).astype(np.int32),               # M == 1: exponential is all ones
        "zeros_u16": np.zeros((6, 7, 8), np.uint16),                                 # M == 0: NaN images
    }


def main():
    rh.load_reference()
    import SimpleITK as sitk  # the stub ref_harness installs
    from radiomics import imageoperations as rio
    logging.getLogger("radiomics").setLevel(logging.ERROR)
    gens = {"square": rio.getSquareImage, "squareroot": rio.getSquareRootImage, "logarithm": rio.getLogarithmImage,
            "exponential": rio.getExponentialImage}
    for case, img in cases().items():
        out = {}
        for name in NAMES:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", RuntimeWarning)      # the all-zero image divides by zero
                (im, yielded, kw), = list(gens[name](sitk.GetImageFromArray(img), None, marker=case))
            assert yielded == name and kw == {"marker": case}, (yielded, kw)
            out[name] = sitk.GetArrayFromImage(im)
            assert out[name].dtype == np.float64 and out[name].shape == img.shape
        path = os.path.join(HERE, f"imagetypes_{case}.npz")
        np.savez_compressed(path, image=img, **out)
        assert os.path.getsize(path) < 1 << 20, path
        print("imagetypes", case, img.shape, img.dtype, "M =", float(np.abs(img.astype(np.float64)).max()),
              os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
