"""GLCM's MCC map from the kernelRadius-1 fast path on 64^3 volumes -- i.i.d. uniform levels, a smooth volume, and both
again inside a holed, ragged ROI (zeros in the windows: the general body of phase A) -- against the numpy restatement of
phase A's classification (tests/mcc_class.py: union-find for connectivity and 2-colouring) and the window oracle.

The GPU computes every voxel; the checks run on 40 000 random centres per volume.  A centre none of whose angles needs an
eigen-solve has MCC = (number of angles classed 1) / (non-empty angles), and the map must hold exactly that double.  A
centre with eigen-tasks is checked against helpers.window_mcc (LAPACK) on a sample, to MCC_ATOL."""
import numpy as np
import pytest
import torch

from helpers import MCC_ATOL, window_mcc
from mcc_class import BIPARTITE, EMPTY, ONE, SPLIT, TASK, classify, windows_of
from pyradiomics_b200 import _lib, voxel

pytestmark = pytest.mark.gpu

N = 64
G_MCC = 19
N_CENTRES = 40000              # centres classified, per volume
N_SAMPLE = 1500                # eigen-task centres checked against the oracle, per volume


def _volume(kind):
    rng = np.random.default_rng(21)
    if kind.startswith("uniform"):
        lev = rng.integers(1, 33, (N, N, N))
    else:
        import scipy.ndimage as ndi
        f = ndi.gaussian_filter(rng.standard_normal((N, N, N)), 3.0)
        lev = np.digitize(f, np.quantile(f, np.linspace(0, 1, 33)[1:-1])) + 1
    if kind.endswith("roi"):
        # a ragged ball with 15 % holes: windows lose voxels at its surface and around every hole
        zz, yy, xx = np.mgrid[:N, :N, :N] - (N - 1) / 2
        r = np.sqrt(zz ** 2 + yy ** 2 + xx ** 2)
        roi = (r < 26 + 4 * rng.random((N, N, N))) & (rng.random((N, N, N)) > 0.15)
        lev = np.where(roi, lev, 0)
    return lev.astype(np.uint8)


@pytest.fixture(scope="module", params=["uniform", "smooth", "uniform_roi", "smooth_roi"])
def case(request):
    lev = _volume(request.param)
    cen = np.argwhere(lev > 0)
    cen = cen[np.sort(np.random.default_rng(22).choice(len(cen), min(N_CENTRES, len(cen)), replace=False))]
    W = windows_of(lev, cen)
    cls = np.stack([classify(W, s)[0] for s in range(13)], 1)          # (V, 13)
    return request.param, lev, cen, W, cls


def test_mcc_map_against_classification_and_oracle(case):
    kind, lev, cen, W, cls = case
    s = _lib.make_settings(32, int(len(np.unique(lev[lev > 0]))))
    out = voxel.voxel_features("glcm", torch.as_tensor(lev).cuda(), s)
    got = out[G_MCC].cpu().numpy()[tuple(cen.T)]
    n_ok = (cls != EMPTY).sum(1)
    ones = ((cls == SPLIT) | (cls == BIPARTITE)).sum(1)
    task = (cls == TASK).any(1)
    counts = {name: int((cls == c).sum()) for name, c in
              (("one", ONE), ("split", SPLIT), ("bipartite", BIPARTITE), ("task", TASK))}
    print(kind, "graphs per class:", counts, "voxels with tasks:", int(task.sum()), "of", len(cen))
    assert counts["split"] > 1000 and counts["task"] > 1000, counts
    # no eigen-task: the exact mean of phase A's 0 / 1 terms (NaN for a centre without any valid pair)
    with np.errstate(divide="ignore", invalid="ignore"):
        want = np.where(n_ok > 0, ones * (1.0 / n_ok), np.nan)[~task]
    assert np.array_equal(got[~task], want, equal_nan=True), (kind, np.flatnonzero(got[~task] != want)[:5])
    # eigen-tasks: the window oracle on a sample
    idx = np.flatnonzero(task)
    idx = np.random.default_rng(3).choice(idx, min(N_SAMPLE, idx.size), replace=False)
    for k in idx:
        ref, per = window_mcc(W[k])
        for slot, r in enumerate(per):
            want_cls = EMPTY if r is None else ONE if r[1] == 1 else SPLIT if not r[2] else BIPARTITE if r[3] else TASK
            assert cls[k, slot] == want_cls, (W[k], slot)
        assert abs(got[k] - ref) <= MCC_ATOL, (kind, W[k], got[k], ref)
