"""Generates tests/golden/lbp3d_*.npz FROM THE REFERENCE ITSELF: its own getLBP3DImage
(radiomics/imageoperations.py:1169-1314) on six small volumes.

Run in the build container only (needs /root/reference):  python tests/golden/make_golden_lbp3d.py

Two imports of the reference are unavailable and stubbed: trimesh.creation.icosphere (the product's restatement,
pyradiomics_b200.imageoperations._icosphere) and scipy.special.sph_harm (removed from SciPy; the old argument order maps
to sph_harm_y(n, m, phi, theta)).  Each yielded image is copied before the generator advances: the reference reuses one
result buffer and the SimpleITK stub does not copy.  Stored: image, mask, vertices, settings and the (levels + 1, Np) maps
at the ROI voxels (np.nonzero order); outside the ROI the reference's values are uninitialised.
"""
from __future__ import annotations

import json
import logging
import os
import sys
import types

import numpy as np
import scipy.special
from scipy.special import sph_harm_y

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle"))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
import lbp3d_np  # noqa: E402
import ref_harness as rh  # noqa: E402
from pyradiomics_b200.imageoperations import _icosphere  # noqa: E402


def main():
    tm, tmc = types.ModuleType("trimesh"), types.ModuleType("trimesh.creation")
    tmc.icosphere = lambda subdivisions, radius: types.SimpleNamespace(vertices=_icosphere(subdivisions, radius))
    tm.creation = tmc
    sys.modules.setdefault("trimesh", tm)
    sys.modules.setdefault("trimesh.creation", tmc)
    scipy.special.sph_harm = lambda m, n, theta, phi: sph_harm_y(n, m, phi, theta)
    rh.load_reference()
    import SimpleITK as sitk  # the stub ref_harness installs
    from radiomics import imageoperations as rio
    logging.getLogger("radiomics").setLevel(logging.ERROR)

    rng = np.random.default_rng(20261015)

    def smooth(shape, scale, offset=0.0):
        f = rng.normal(size=shape)
        for ax in range(3):
            f = (np.roll(f, 1, ax) + 2 * f + np.roll(f, -1, ax)) / 4
        return f * scale + offset

    img_b, m_b, _ = rh.load_case("brain1")
    # constant 11^3 blocks with small steps (the spline's ringing at a block's core rounds away: flat integer samples,
    # NaN kurtosis), a noisy slab on top
    plateau = np.kron(rng.integers(-2, 3, (2, 2, 2)) * 10, np.ones((11, 11, 11), np.int64))
    plateau[16:] += rng.integers(-60, 60, plateau[16:].shape)
    cases = {
        "brain1": (img_b, m_b, {}),
        "plateau_i16": (plateau.astype(np.int16), rng.random(plateau.shape) < 0.7, {}),
        "faces_f64": (smooth((11, 12, 13), 300.0, 40.0), np.ones((11, 12, 13), bool), {}),
        "f32": (smooth((12, 13, 14), 2.5, 1.0).astype(np.float32), rng.random((12, 13, 14)) < 0.6, {}),
        "l3_r15_s2": (np.round(smooth((13, 14, 15), 500.0)).astype(np.int16), rng.random((13, 14, 15)) < 0.5,
                      {"lbp3DLevels": 3, "lbp3DIcosphereRadius": 1.5, "lbp3DIcosphereSubdivision": 2}),
        "s0": (np.round(smooth((10, 11, 12), 800.0, 100.0)).astype(np.int16), rng.random((10, 11, 12)) < 0.6,
               {"lbp3DIcosphereSubdivision": 0}),
    }
    for name, (img, msk, kw) in cases.items():
        img = np.ascontiguousarray(img)
        mask = np.ascontiguousarray(msk).astype(np.uint8)
        levels = kw.get("lbp3DLevels", 2)
        radius = kw.get("lbp3DIcosphereRadius", 1)
        verts = _icosphere(kw.get("lbp3DIcosphereSubdivision", 1), radius)
        roi = np.nonzero(mask == 1)
        got = []
        for im, nm, _ in rio.getLBP3DImage(sitk.GetImageFromArray(img), sitk.GetImageFromArray(mask), **kw):
            got.append((nm, np.array(im._arr)[roi]))
        names = [nm for nm, _ in got]
        assert names == [f"lbp-3D-m{i + 1}" for i in range(levels)] + ["lbp-3D-k"], names
        if np.issubdtype(img.dtype, np.integer):       # no sample within 1e-9 of an integer rounding tie
            margin = lbp3d_np.lbp3d(img, mask == 1, verts, levels, radius)["margin"]
            assert margin.min() > 1e-9, (name, margin.min())
        np.savez_compressed(os.path.join(HERE, f"lbp3d_{name}.npz"), image=img, mask=mask, vertices=verts,
                            maps=np.stack([a for _, a in got]), settings=json.dumps(kw))
        print("lbp3d", name, img.shape, img.dtype, len(roi[0]), "ROI voxels")


if __name__ == "__main__":
    main()
