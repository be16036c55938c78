"""Segment-mode matrices on a side stream.  The device entry points (rb_segment_texture_dev, rb_segment_glrlm_dev,
rb_segment_glszm_dev) and rb_fill_glszm run on torch's current stream, the stream the levels were written on: under
`with torch.cuda.stream(s)` on a fresh (non-blocking) stream they give the same bits as on the default stream, with no
host synchronisation between discretisation and matrices."""
import numpy as np
import pytest
import torch

from pyradiomics_b200 import cmatrices as B, featureclasses as FC
from pyradiomics_b200._lib import check, lib, ptr, stream

pytestmark = pytest.mark.gpu

SHAPE, NG = (96, 128, 160), 32


def _case_matrices():
    """one case discretised on the current stream (seeded raw image -> binWidth 25 levels 1..32 -> packed levels) and all
    its segment matrices; nothing between the raw image and the matrix calls waits on the host"""
    g = torch.Generator(device="cuda").manual_seed(7)
    raw = torch.randint(-40, 760, SHAPE, generator=g, device="cuda", dtype=torch.int32)
    lev32 = torch.div(raw - raw.min(), 25, rounding_mode="floor") + 1
    mask = torch.ones(SHAPE, dtype=torch.uint8, device="cuda")
    mask[:, :, :7] = 0
    levels = torch.empty(SHAPE, dtype=torch.uint8, device="cuda")
    check(lib().rb_pack_levels_dev(ptr(lev32), ptr(mask), lev32.numel(), NG, ptr(levels), None, None, stream()), "pack")
    tex = B.segment_texture_device(levels, [1, 2], NG, 1, False, 0)
    glrlm, _ = B.calculate_glrlm_device(levels, NG, max(SHAPE), False, 0)
    glszm = B.calculate_glszm_device(levels, NG, False, 0)           # rb_segment_glszm_dev, then rb_fill_glszm
    return {"glcm": tex["glcm"][0], "gldm": tex["gldm"], "ngtdm": tex["ngtdm"], "glrlm": glrlm, "glszm": glszm}


def test_device_entry_points_on_a_side_stream_equal_the_default_stream():
    ref = _case_matrices()
    assert ref["glszm"].shape[2] > 1 and ref["glrlm"][..., 1:, :].any()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = _case_matrices()
    for k, r in ref.items():
        assert got[k].shape == r.shape and np.array_equal(got[k], r), k


def test_plugin_segment_extraction_on_a_side_stream_equals_the_default_stream():
    rng = np.random.default_rng(11)
    raw = rng.integers(0, 800, (64, 80, 96)).astype(np.int16)
    mask = np.zeros(raw.shape, np.uint8)
    mask[4:60, 6:74, 8:90] = 1

    def extract():
        FC.clear_device_cache()           # else the second run reuses the levels the first one cached
        return {c: cls(raw, mask, binWidth=25).execute() for c, cls in FC.FEATURE_CLASSES.items()}

    ref = extract()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = extract()
    for c, feats in ref.items():
        assert got[c].keys() == feats.keys(), c
        for f, v in feats.items():
            assert np.array_equal(np.asarray(got[c][f]), np.asarray(v), equal_nan=True), (c, f)
