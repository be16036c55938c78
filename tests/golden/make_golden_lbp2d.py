"""Generates tests/golden/lbp2d_*.npz FROM THE REFERENCE ITSELF: its own getLBP2DImage
(radiomics/imageoperations.py:1094-1166) on small images.

Run in the build container only (needs /root/reference):  python tests/golden/make_golden_lbp2d.py

scikit-image is unavailable and stubbed: skimage.feature.local_binary_pattern is the NumPy restatement
oracle/lbp2d_np.py, the way make_golden_lbp3d.py stubs trimesh.  What these goldens pin is therefore the reference's
wrapper -- settings and defaults, the slicing axis, the cast of each slice to the image's dtype, the float64 result of a
2-D image, the name and the warnings -- on top of the restated per-pixel arithmetic.  Stored: image, settings, the
yielded array (its dtype included) and the warnings the generator logged.
"""
from __future__ import annotations

import json
import logging
import os
import sys
import types
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle"))
import lbp2d_np  # noqa: E402
import ref_harness as rh  # noqa: E402


class _Collect(logging.Handler):
    def __init__(self):
        super().__init__(logging.WARNING)
        self.messages = []

    def emit(self, record):
        self.messages.append(record.getMessage())


def main():
    sk, skf = types.ModuleType("skimage"), types.ModuleType("skimage.feature")
    skf.local_binary_pattern = lbp2d_np.local_binary_pattern
    sk.feature = skf
    sys.modules.setdefault("skimage", sk)
    sys.modules.setdefault("skimage.feature", skf)
    rh.load_reference()
    import SimpleITK as sitk  # the stub ref_harness installs
    from radiomics import imageoperations as rio
    log = logging.getLogger("radiomics.imageoperations")
    collect = _Collect()
    log.addHandler(collect)

    rng = np.random.default_rng(20261016)

    def smooth(shape, scale, offset=0.0):
        f = rng.normal(size=shape)
        for ax in range(f.ndim):
            f = (np.roll(f, 1, ax) + 2 * f + np.roll(f, -1, ax)) / 4
        return f * scale + offset

    img_b, _, _ = rh.load_case("brain1")
    brain = np.ascontiguousarray(img_b[:9, :33, :37])
    f32 = smooth((7, 15, 16), 3.0, 1.0).astype(np.float32)
    f32[1, 3, 4], f32[2, 7, 7], f32[4, 10, 2], f32[5, 0, 9] = np.nan, np.inf, -np.inf, np.inf
    f32[3, 5:7, 5:7] = np.inf                                   # inf - inf = NaN: no sign bit next to a centre of inf
    f64 = smooth((6, 14, 13), 50.0)
    f64[0, 0, 0], f64[2, 6, 6], f64[3, 9, 2], f64[5, 13, 12] = np.nan, -np.inf, np.inf, np.nan
    cases = {
        "brain1_a0": (brain, {}),
        "brain1_a1": (brain, {"force2Ddimension": 1, "force2D": True}),
        "brain1_a2": (brain, {"force2Ddimension": 2, "lbp2DMethod": "nri_uniform"}),
        "u8_2d": (np.round(smooth((23, 29), 40.0, 120.0)).clip(0, 255).astype(np.uint8), {}),
        "f32_naninf": (f32, {"lbp2DMethod": "default"}),
        "f64_naninf": (f64, {"lbp2DMethod": "ror", "force2Ddimension": 2}),
        "f64_naninf_var": (f64, {"lbp2DMethod": "var", "force2Ddimension": 1}),
        "const_var_i16": (np.full((3, 8, 9), 7, np.int16), {"lbp2DMethod": "var"}),
        "var_i16": (np.round(smooth((5, 17, 19), 300.0)).astype(np.int16), {"lbp2DMethod": "var", "lbp2DRadius": 1.5}),
        "u8_default_p9": (rng.integers(0, 256, (4, 12, 14)).astype(np.uint8), {"lbp2DMethod": "default", "lbp2DSamples": 9}),
        "p24_r3": (np.round(smooth((5, 21, 22), 500.0)).astype(np.int16),
                   {"lbp2DSamples": 24, "lbp2DRadius": 3, "lbp2DMethod": "nri_uniform", "force2Ddimension": 1}),
        "p24_r3_default_f64": (smooth((20, 18), 10.0), {"lbp2DSamples": 24, "lbp2DRadius": 3, "lbp2DMethod": "default"}),
        "r05_ror": (np.round(smooth((4, 13, 15), 200.0)).astype(np.int32),
                    {"lbp2DRadius": 0.5, "lbp2DMethod": "ror", "force2D": True}),
    }
    for name, (img, kw) in cases.items():
        img = np.ascontiguousarray(img)
        collect.messages.clear()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)                   # NumPy's cast of NaN / inf
            got = [(nm, np.array(im._arr)) for im, nm, _ in rio.getLBP2DImage(sitk.GetImageFromArray(img), None, **kw)]
        assert [nm for nm, _ in got] == ["lbp-2D"], got
        out = got[0][1]
        assert out.dtype == (img.dtype if img.ndim == 3 else np.float64), (name, out.dtype)
        np.savez_compressed(os.path.join(HERE, f"lbp2d_{name}.npz"), image=img, out=out, settings=json.dumps(kw),
                            warnings=json.dumps(list(collect.messages)))
        print("lbp2d", name, img.shape, img.dtype, "->", out.dtype, collect.messages)


if __name__ == "__main__":
    main()
