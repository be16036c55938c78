"""The voxel-batch mode of the cMatrices drop-in -- cmatrices.calculate_*(..., kernelRadius, voxels), one dense matrix per
listed voxel from matrix_kernels.cu (batch_matrix_kernel, batch_glszm_zones_kernel, batch_glszm_fill_kernel) --
against the compiled reference _cmatrices on the corpus of tests/helpers.py::vb_corpus: every matrix and angle set bit
for bit (NGTDM s_i within 1e-12), at every window template (27, 125, 343 positions) with 8- and 16-bit levels.  The CPU
file holds the oracle port to the same reference on the same corpus.  GLRLM runs longer than Nr are refused with
IndexError by the batch and the segment path alike."""
import numpy as np
import pytest

from helpers import VB_MODES, assert_vb_reach, vb_assert_same, vb_call, vb_check_expect, vb_corpus, vb_longest_run, \
    vb_short_nr_cases, vb_voxels
from pyradiomics_b200 import cmatrices as B
from pyradiomics_b200._lib import B200Error

pytestmark = pytest.mark.gpu
CORPUS = vb_corpus()


def _cmatrices():
    import build_ref
    try:
        return build_ref.load("_cmatrices")
    except ImportError as e:
        pytest.fail(f"the compiled reference _cmatrices is missing ({e}); build() compiles it into oracle/_ref/")


def test_corpus_reach():
    assert_vb_reach(CORPUS)


@pytest.mark.parametrize("c", CORPUS, ids=[c["name"] for c in CORPUS])
def test_batch_kernels_equal_compiled_reference(c):
    """every call of the case bit-equal to the reference, with what the case is built to reach asserted on the product's
    matrices; GLRLM at Nr = the longest run of the listed windows equals the reference, one less raises IndexError"""
    R = _cmatrices()
    L = None
    for mode in VB_MODES:
        vox = vb_voxels(c, mode)
        if vox is None:
            continue
        for alpha in (c["alphas"] if mode == "gldm" else (0,)):
            ref = vb_call(R, c, mode, vox, alpha)
            got = vb_call(B, c, mode, vox, alpha)
            vb_assert_same(got, ref, mode, (c["name"], mode, alpha))
            vb_check_expect(c, mode, got)
            if mode == "glrlm":
                L = vb_longest_run(ref[0])
    vox = vb_voxels(c, "glrlm")
    vb_assert_same(vb_call(B, c, "glrlm", vox, Nr=L), vb_call(R, c, "glrlm", vox, Nr=L), "glrlm", (c["name"], "Nr", L))
    if L > 1:
        with pytest.raises(IndexError, match="run longer than Nr"):
            vb_call(B, c, "glrlm", vox, Nr=L - 1)


@pytest.mark.parametrize("c", vb_short_nr_cases(), ids=lambda c: c["name"])
def test_runs_longer_than_nr_raise_in_batch_and_segment_mode(c):
    """the runs of 7 of a 7^3 plateau at Nr = 6, its centre the last listed voxel: at the top gray level the unguarded
    index passes the end of the batch, below it the next level's row (test_voxel_batch_matrices_cpu.py shows both).  The
    batch and the segment path raise IndexError; the next call with Nr = 7 equals the reference."""
    R = _cmatrices()
    img, msk, Ng = c["img"], c["msk"], c["Ng"]
    with pytest.raises(IndexError, match="run longer than Nr"):
        vb_call(B, c, "glrlm", c["vox"], Nr=6)
    vb_assert_same(vb_call(B, c, "glrlm", c["vox"], Nr=7), vb_call(R, c, "glrlm", c["vox"], Nr=7), "glrlm", c["name"])
    ref = R.calculate_glrlm(img, msk, Ng, max(img.shape), 0, 0)
    L = vb_longest_run(ref[0])
    assert L >= 7
    with pytest.raises(IndexError, match="run longer than Nr"):
        B.calculate_glrlm(img, msk, Ng, L - 1, 0, 0)
    vb_assert_same(B.calculate_glrlm(img, msk, Ng, L, 0, 0), R.calculate_glrlm(img, msk, Ng, L, 0, 0), "glrlm", c["name"])


def test_error_contract():
    """kernelRadius <= 0 with a voxel list: RuntimeError (the reference's); a voxel index outside the volume: ValueError;
    kernelRadius 4: refused (RB_ERR_UNSUPPORTED), for every mode"""
    c = CORPUS[0]
    vox = c["vox"][:, :5]
    for mode in VB_MODES:
        for r in (0, -1):
            with pytest.raises(RuntimeError, match="kernelRadius"):
                vb_call(B, dict(c, r=r), mode, vox)
        for d in range(3):
            for bad in (-1, c["img"].shape[d]):
                v = vox.copy()
                v[d, 2] = bad
                with pytest.raises(ValueError, match="voxel index out of range"):
                    vb_call(B, c, mode, v)
        with pytest.raises(B200Error, match="kernelRadius > 3"):
            vb_call(B, dict(c, r=4), mode, vox)
    got = vb_call(B, c, "glcm", vox)                       # the library is usable after the refusals
    vb_assert_same(got, vb_call(_cmatrices(), c, "glcm", vox), "glcm", "after errors")
    assert np.asarray(got[0]).sum() > 0
