"""pipeline.segment_suite_with_filters: on the original image against the reference's baselines; on every derived image
against the plugin classes run on that image downloaded and cropped to the ROI's bounding box (the reference's flow):
texture bit for bit, first order within its summation bound, keys and their order as RadiomicsFeatureExtractor's."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN
from pyradiomics_b200 import featureclasses as FC, image as I, pipeline as PL
from test_firstorder_segment_gpu import check as check_firstorder, ellipsoid

pytestmark = pytest.mark.gpu

TEXTURE = ("glcm", "glrlm", "glszm", "gldm", "ngtdm")


def _bbox(m):
    sl = []
    for d in range(m.ndim):
        on = np.flatnonzero(m.any(axis=tuple(k for k in range(m.ndim) if k != d)))
        sl.append(slice(on[0], on[-1] + 1))
    return tuple(sl)


@pytest.mark.parametrize("cname", ("firstorder",) + TEXTURE)
def test_original_image_matches_the_reference_baselines(cname):
    cases = np.load(os.path.join(GOLDEN, "segment_cases.npz"))
    if cname == "firstorder":
        cols = json.load(open(os.path.join(GOLDEN, "segment_expect_firstorder.json")))
        tol = 1e-9
    else:
        cols = json.load(open(os.path.join(GOLDEN, "segment_expect.json")))[cname]
        tol = 1e-7
    for test, e in cols.items():
        c = e["case"]
        s = dict(e["settings"])
        sp_zyx = tuple(cases[c + "_spacing"])[::-1]
        got = PL.segment_suite_with_filters(torch.from_numpy(cases[c + "_image"]).cuda(),
                                            torch.from_numpy(cases[c + "_mask"].astype(np.uint8)).cuda(), classes=(cname,),
                                            shape=False, spacing_zyx=sp_zyx, wavelet=None, sigmas=(), **s)
        for f, v in e["features"].items():
            g = float(got[f"original_{cname}_{f}"])
            assert np.isclose(g, v, rtol=tol, atol=1e-12, equal_nan=True), (test, f, g, v)


@pytest.mark.parametrize("case", ["brain1", "brain2", "breast1", "lung1", "lung2"])
def test_shape_matches_the_reference(case):
    exp = json.load(open(os.path.join(GOLDEN, "shape_expect.json")))[case]
    seg = np.load(os.path.join(GOLDEN, "segment_cases.npz"))
    got = PL.segment_suite_with_filters(torch.from_numpy(seg[case + "_image"]).cuda(),
                                        torch.from_numpy(seg[case + "_mask"].astype(np.uint8)).cuda(), classes=(),
                                        spacing_zyx=tuple(seg[case + "_spacing"])[::-1], wavelet=None, sigmas=())
    enabled = [f for f, deprecated in FC.RadiomicsShape.getFeatureNames().items() if not deprecated]
    assert list(got) == [f"original_shape_{f}" for f in enabled]
    for f, v in exp["features"].items():
        if f"original_shape_{f}" in got:
            assert float(got[f"original_shape_{f}"]) == pytest.approx(v, rel=1e-7), f


def _volume(seed=0, shape=(34, 40, 46)):
    rng = np.random.default_rng(seed)
    z, y, x = np.meshgrid(*[np.linspace(0, 3, s) for s in shape], indexing="ij")
    img = (400 * np.sin(z) * np.cos(1.3 * y) + 150 * x + rng.normal(0, 40, shape)).astype(np.int16)
    mask = np.zeros(shape, np.uint8)
    mask[ellipsoid(shape, 0.5, seed)] = 2                      # label 2: the ROI
    mask[:3] = 1
    return img, mask


def compare_with_plugins(img, mask, label=2, classes=("firstorder",) + TEXTURE, sp_zyx=(1.25, 0.75, 0.5), shape=True,
                         normalize=None, resegment=None, resegment_shape=False, **kw):
    img_t, mask_t = torch.from_numpy(img).cuda(), torch.from_numpy(mask).cuda()
    got = PL.segment_suite_with_filters(img_t, mask_t, classes=classes, shape=shape, spacing_zyx=sp_zyx, label=label,
                                        normalize=normalize, resegment=resegment, resegment_shape=resegment_shape, **kw)
    # the reference's flow: the same derived images, downloaded, cropped to the ROI's bounding box, plugin classes
    filt = {k: kw[k] for k in ("wavelet", "sigmas", "image_types", "lbp3d") if k in kw}
    settings = {k: v for k, v in kw.items() if k not in filt}
    import pyradiomics_b200.imageoperations as IO
    x = img_t if normalize is None else IO.normalize_image_device(img_t, normalize.get("normalizeScale", 1),
                                                                   normalize.get("removeOutliers"))
    roi = (mask_t == label).to(torch.uint8)
    shape_roi = roi
    if resegment is not None:
        roi, _, _ = IO.resegment_mask_device(x, roi, resegment["resegmentRange"], resegment.get("resegmentMode", "absolute"))
        shape_roi = roi if resegment_shape else shape_roi
    roi_h = roi.cpu().numpy() != 0
    bb = _bbox(roi_h)
    sp_xyz = tuple(sp_zyx)[::-1]
    keys = []
    if shape:
        sroi = shape_roi.cpu().numpy() != 0
        sb = _bbox(sroi)
        sh = FC.RadiomicsShape(I.ArrayImage(img[sb], sp_xyz), I.ArrayImage(sroi[sb].astype(np.uint8), sp_xyz)).execute()
        for f, v in sh.items():
            keys.append(f"original_shape_{f}")
            # area and volume end in per-block atomic sums: their last bits vary from run to run
            assert float(got[keys[-1]]) == pytest.approx(float(v), rel=1e-12, nan_ok=True), f
    n_images = 0
    for name, d in PL.derived_images(x, sp_zyx, mask=roi, **filt):
        n_images += 1
        dh = d.cpu().numpy()[bb]
        mh = roi_h[bb].astype(np.uint8)
        for c in classes:
            if c == "firstorder":
                obj = FC.RadiomicsFirstOrder(I.ArrayImage(dh, sp_xyz), I.ArrayImage(mh, sp_xyz), **settings)
                ref = obj.execute()
                vals = {f: got[f"{name}_{c}_{f}"] for f in FC.RadiomicsFirstOrder.NAMES}
                check_firstorder(vals, dh[mh != 0], obj.discretizedImageArray[mh != 0], settings.get("voxelArrayShift", 0),
                                 float(np.multiply.reduce(np.asarray(sp_xyz))), what=name)
            else:
                ref = FC.FEATURE_CLASSES[c](I.ArrayImage(dh, sp_xyz), I.ArrayImage(mh, sp_xyz), **settings).execute()
                for f, v in ref.items():
                    g = got[f"{name}_{c}_{f}"]
                    assert np.float64(g).tobytes() == np.float64(v).tobytes(), (name, c, f, float(g), float(v))
            keys += [f"{name}_{c}_{f}" for f in ref]
    assert list(got) == keys
    return got, n_images


def test_every_derived_image_matches_the_plugin_classes_on_the_cropped_image():
    img, mask = _volume(0)
    got, n = compare_with_plugins(img, mask, binCount=24, wavelet="coif1", sigmas=(1.0, 2.0),
                                  image_types=("square", "squareroot", "logarithm", "exponential", "gradient"), lbp3d={})
    assert n == 1 + 8 + 2 + 5 + 3


def test_normalise_and_resegment():
    img, mask = _volume(1)
    reseg = {"resegmentRange": [-200, 300]}
    roi = mask == 2
    kept = roi & (img >= -200) & (img <= 300)
    assert 0 < kept.sum() < roi.sum()
    compare_with_plugins(img, mask, binWidth=25, wavelet=None, sigmas=(1.0,), resegment=reseg)
    got_shape_label, _ = compare_with_plugins(img, mask, binWidth=25, wavelet=None, sigmas=(), resegment=reseg,
                                              classes=())
    got_shape_reseg, _ = compare_with_plugins(img, mask, binWidth=25, wavelet=None, sigmas=(), resegment=reseg,
                                              resegment_shape=True, classes=())
    assert got_shape_label["original_shape_VoxelVolume"] > got_shape_reseg["original_shape_VoxelVolume"]
    compare_with_plugins(img, mask, binWidth=0.25, wavelet=None, sigmas=(1.0,), normalize={"normalizeScale": 1},
                         resegment={"resegmentRange": [-1.0, 1.5]})


@pytest.mark.parametrize("kw", [dict(weightingNorm="euclidean", distances=[1, 2]), dict(weightingNorm="manhattan"),
                                dict(symmetricalGLCM=False, distances=[1, 3], binCount=16, gldm_a=1),
                                dict(weightingNorm="infinity", gldm_a=2, voxelArrayShift=500)])
def test_settings_pass_through(kw):
    img, mask = _volume(2)
    compare_with_plugins(img, mask, wavelet=None, sigmas=(1.0,), shape=False, **kw)


def test_errors():
    img, mask = _volume(3)
    with pytest.raises(ValueError):
        PL.segment_suite_with_filters(torch.from_numpy(img).cuda(), torch.from_numpy(mask).cuda(), classes=("nope",))
    with pytest.raises(ValueError):
        PL.segment_suite_with_filters(torch.from_numpy(img).cuda(), torch.from_numpy(mask).cuda(), label=7)
