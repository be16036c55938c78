"""The oracle port (oracle/cmatrices_port.c) against the compiled reference _cmatrices on the voxel-batch corpus
(tests/helpers.py::vb_corpus), which the GPU file runs through the CUDA batch kernels: every matrix and angle set bit
for bit (NGTDM s_i within 1e-12), so a failure there points at the kernels, not at the port.  Also the corpus's reach,
and the index arithmetic of a GLRLM run longer than Nr."""
import numpy as np
import pytest

import cmatrices_oracle as O
from helpers import VB_MODES, assert_vb_reach, vb_assert_same, vb_call, vb_check_expect, vb_corpus, vb_longest_run, \
    vb_short_nr_cases, vb_voxels

CORPUS = vb_corpus()


def _cmatrices():
    import build_ref
    try:
        return build_ref.load("_cmatrices")
    except ImportError as e:
        pytest.fail(f"the compiled reference _cmatrices is missing ({e}); build() compiles it into oracle/_ref/")


def test_corpus_reach():
    """every (window template, level width, mode), >= 8 blocks of listed voxels per template, and cases built for a
    zone of 343 voxels, zones of one voxel and GLRLM runs of 3, 5 and 7 (each asserted on the matrices by the tests)"""
    assert_vb_reach(CORPUS)


@pytest.mark.parametrize("c", CORPUS, ids=[c["name"] for c in CORPUS])
def test_port_equals_compiled_reference(c):
    R = _cmatrices()
    for mode in VB_MODES:
        vox = vb_voxels(c, mode)
        if vox is None:
            continue
        for alpha in (c["alphas"] if mode == "gldm" else (0,)):
            ref = vb_call(R, c, mode, vox, alpha)
            vb_assert_same(vb_call(O, c, mode, vox, alpha), ref, mode, (c["name"], mode, alpha))
            vb_check_expect(c, mode, ref)
    # GLRLM at Nr = the longest run of the listed windows equals the reference; one less, the port refuses the batch as
    # the product does (the reference raises only when the flat index leaves the voxel's matrix)
    vox = vb_voxels(c, "glrlm")
    L = vb_longest_run(vb_call(R, c, "glrlm", vox)[0])
    vb_assert_same(vb_call(O, c, "glrlm", vox, Nr=L), vb_call(R, c, "glrlm", vox, Nr=L), "glrlm", (c["name"], "Nr", L))
    if L > 1:
        with pytest.raises(IndexError):
            vb_call(O, c, "glrlm", vox, Nr=L - 1)


@pytest.mark.parametrize("c", vb_short_nr_cases(), ids=lambda c: c["name"])
def test_short_nr_runs_index_outside_their_row(c):
    """A batch kernel that counted a run of rl + 1 voxels at ((gl - 1) * Nr + rl) * Na + a without bounding rl writes,
    at Nr = 6, the runs of 7 of these plateaus outside their row: past the last listed voxel's matrix, i.e. past the
    end of the batch's buffer, at the top gray level (the reference raises IndexError), and into the next gray level's
    row below it (the reference counts them there without an error; the product refuses both)."""
    R = _cmatrices()
    P, _ = vb_call(R, c, "glrlm", c["vox"])
    nvox, Ng, _, Na = P.shape
    assert vb_longest_run(P) == 7
    Nr = 6
    v, g, rl, a = np.nonzero(P[:, :, Nr:, :])
    flat = ((g * Nr) + rl + Nr) * Na + a                       # g = gl - 1, offset inside the voxel's matrix
    block = Ng * Nr * Na
    if c["expect"]["short_nr"] == "raises":
        last = (v == nvox - 1) & (flat >= block)
        assert last.any()
        assert ((nvox - 1) * block + flat[last]).min() >= nvox * block   # past the end of the whole batch
        with pytest.raises(IndexError):
            vb_call(R, c, "glrlm", c["vox"], Nr=Nr)
    else:
        assert (flat < block).all() and (flat // (Nr * Na) > g).all()  # inside the matrix, in a higher level's row
        short, _ = vb_call(R, c, "glrlm", c["vox"], Nr=Nr)
        assert short.sum() == P.sum()                                  # the reference moved those runs, none dropped
        assert not np.array_equal(short, P[:, :, :Nr, :])
