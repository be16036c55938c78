"""The resampling step (reference radiomics/imageoperations.py:448-612) of the CPU oracle, pinned on the reference's own
baseline: the bundled breast1 case resampled to 2 mm with the B-spline interpolator must reproduce EVERY `original_*` value of
the `breast1_resampling` column of data/baseline/baseline_{firstorder,glcm,glrlm,glszm,gldm,ngtdm,shape}.csv
(tests/golden/resample_breast1.npz, written by make_golden.py --resample-only)."""
import os

import numpy as np
import pytest

import firstorder_np as FO
import pipeline as PL
import resample_np as RS
import shape_np as SH

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _features(img, msk, new):
    idx = np.array(np.where(msk == 1))
    sl = tuple(slice(a, b + 1) for a, b in zip(idx.min(1), idx.max(1)))      # segment mode: cropped to the ROI box (padDistance 0)
    ci, cm = img[sl], msk[sl] == 1
    out = {"original_firstorder_" + k: v for k, v in FO.extract(ci, cm, spacing_xyz=tuple(new), binWidth=25).items()}
    for c in PL.CLASS_NAMES:
        out.update({f"original_{c}_{k}": v for k, v in PL.extract(c, ci, cm, binWidth=25, spacing_zyx=tuple(new)[::-1]).items()})
    out.update({"original_shape_" + k: v for k, v in SH.features(cm, tuple(new)[::-1]).items()})
    return out


def test_oracle_resampling_reproduces_the_reference_baseline_column():
    z = np.load(os.path.join(G, "resample_breast1.npz"))
    exp = dict(zip(z["names"], z["values"]))
    img, msk, new = RS.resample(z["image"], z["mask"], z["spacing"], (2, 2, 2))
    assert img.shape == (16, 16, 14) and int((msk == 1).sum()) == 23 and img.dtype == z["image"].dtype
    got = _features(img, msk, new)
    hit = [k for k in exp if k in got]
    assert len(hit) >= 100
    for k in hit:
        assert np.isclose(got[k], exp[k], rtol=1e-9, atol=1e-12), (k, got[k], exp[k])
    # the cast is a truncation: rounding to nearest changes the ROI mean (126.87 instead of the baseline's 126.17)
    assert exp["original_firstorder_Mean"] == 126.17391304347827


@pytest.mark.parametrize("case", ["brain1", "brain2", "lung1", "lung2"])
def test_oracle_resampling_reproduces_the_other_four_baseline_columns(case):
    """`<case>_resampling` of the seven baseline CSVs for the other bundled cases (tests/golden/resample_case_<case>.npz: the
    ROI box + pad + a 10-16 voxel margin of each image, with the index the crop started at -- it resamples to exactly the
    whole image's arrays)"""
    z = np.load(os.path.join(G, f"resample_case_{case}.npz"))
    exp = dict(zip(z[case + "_names"], z[case + "_values"]))
    img, msk, new = RS.resample(z[case + "_image"], z[case + "_mask"], z[case + "_spacing"], (2, 2, 2),
                                offset_xyz=tuple(z[case + "_offset_xyz"]), full_size_xyz=tuple(z[case + "_full_size_xyz"]))
    got = _features(img, msk, new)
    hit = [k for k in exp if k in got]
    assert len(hit) == 107
    for k in hit:
        assert np.isclose(got[k], exp[k], rtol=1e-9, atol=1e-12), (case, k, got[k], exp[k])


def test_grid_arithmetic_special_cases():
    m = np.zeros((6, 20, 22), np.uint8)
    m[3, 4:15, 5:17] = 1                                       # single-slice ROI: no resampling across it (:509-511)
    size, start, step, new = RS.grid(m, (0.5, 0.5, 3.0), (1.0, 1.0, 1.0))
    assert new[2] == 3.0 and step[2] == 1.0 and step[0] == 2.0
    size0, _, _, new0 = RS.grid(m, (0.5, 0.5, 3.0), (1.0, 1.0, 0))          # 0 = keep the original spacing (:500-503)
    assert new0[2] == 3.0 and tuple(size0) == tuple(size)
    # the grid never leaves the image (:544-548)
    size, start, step, _ = RS.grid(np.ones((4, 5, 6), np.uint8), (1, 1, 1), (0.5, 0.5, 0.5), padDistance=50)
    assert tuple(size) == (12, 10, 8) and np.allclose(start, -0.25)
