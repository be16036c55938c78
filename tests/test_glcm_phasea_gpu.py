"""GLCM phase A takes a full-window body for centre voxels whose 27 window levels are all non-zero and the general
body for the rest (volume faces, ROI borders and holes), both inside one launch.  These tests build volumes where
the tiles of that kernel mix the two kinds of voxels and check the maps against the generic kernel, run to run and
slab against whole volume."""
import numpy as np
import pytest
import torch

from pyradiomics_b200 import _lib, voxel

pytestmark = pytest.mark.gpu


def _levels(kind, shape, seed):
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        return rng.integers(1, 33, shape).astype(np.uint8)
    zz, yy, xx = np.meshgrid(*[np.arange(s) for s in shape], indexing="ij")
    f = np.sin(zz / 2.7) + np.cos(yy / 3.1) + np.sin(xx / 2.3 + 1) + 0.25 * rng.normal(size=shape)
    q = np.quantile(f, np.linspace(0, 1, 33)[1:-1])
    return (np.digitize(f, q) + 1).astype(np.uint8)


def _case(name):
    """(levels, centers or None): every case but all_full puts full and non-full windows into the same tiles"""
    rng = np.random.default_rng(11)
    centers = None
    if name == "all_full":                      # only interior centres: every window is full
        lev = _levels("uniform", (20, 22, 24), 1)
        centers = np.zeros(lev.shape, np.uint8)
        centers[1:-1, 1:-1, 1:-1] = 1
    elif name.startswith("holes10"):            # 10 % of the voxels outside the ROI
        lev = _levels(name.split("_")[1], (30, 33, 35), 2)
        lev[rng.random(lev.shape) < 0.1] = 0
    elif name == "thin_roi":                    # ROIs one voxel thick, in each direction
        lev = _levels("smooth", (24, 26, 28), 3)
        roi = np.zeros(lev.shape, bool)
        roi[7, 2:20, 3:25] = True
        roi[3:20, 11, 4:22] = True
        roi[2:22, 5:21, 17] = True
        roi[12:20, 2:24, 2:26] = True           # and a solid block next to them
        lev[~roi] = 0
    elif name == "faces":                       # few planes: most windows touch a face
        lev = _levels("uniform", (4, 40, 44), 4)
    elif name == "narrow":                      # 3 voxels wide: no full window at all outside the middle column
        lev = _levels("smooth", (30, 32, 3), 5)
    elif name == "centers":                     # a centre mask over a volume with holes
        lev = _levels("smooth", (26, 28, 30), 6)
        lev[rng.random(lev.shape) < 0.05] = 0
        centers = (rng.random(lev.shape) < 0.6).astype(np.uint8)
    else:
        raise ValueError(name)
    return lev, centers


CASES = ["all_full", "holes10_uniform", "holes10_smooth", "thin_roi", "faces", "narrow", "centers"]


def _glcm(lev, centers, **kw):
    s = _lib.make_settings(32, 32)
    return voxel.voxel_features("glcm", lev, s, centers=centers, **kw)


@pytest.mark.parametrize("name", CASES)
def test_phaseA_full_and_general_bodies_equal_generic_kernel(name, monkeypatch):
    lev_np, c_np = _case(name)
    lev = torch.as_tensor(lev_np).cuda()
    centers = None if c_np is None else torch.as_tensor(c_np).cuda()
    fast = _glcm(lev, centers).cpu().numpy()
    monkeypatch.setenv("B200_RADIOMICS_FORCE_GENERIC", "1")
    gen = _glcm(lev, centers).cpu().numpy()
    monkeypatch.delenv("B200_RADIOMICS_FORCE_GENERIC")
    for k, f in enumerate(_lib.feature_names("glcm")):
        # MCC: both solves are within 1e-9 of LAPACK (tests/test_fast_voxel_windows_gpu.py), an absolute bound;
        # Imc2: 1e-6 stays for the square root of rounding noise the generic kernel can return (see below)
        rtol, atol = {"MCC": (0, 1e-9), "Imc1": (2e-9, 1e-12), "Imc2": (2e-9, 1e-6)}.get(f, (1e-7, 1e-9))
        ok = np.isclose(fast[k], gen[k], rtol=rtol, atol=atol, equal_nan=True)
        if f == "Imc2":
            # An angle with exactly independent margins has HXY2 == HXY.  The fast path counts its Imc2 as 0 when the two
            # agree to 1e-12; the generic kernel follows the reference's exact comparison of the rounded entropies and
            # drops the angle (NaN) when rounding puts HXY2 below HXY.  The means then differ by the factor m / (m - 1)
            # for m angles, a property of the two conventions, not of the body that ran.
            for m in range(2, 14):
                ok |= np.isclose(fast[k] * m / (m - 1), gen[k], rtol=1e-7, atol=atol)
        assert ok.all(), (f, np.argwhere(~ok)[:3])


def test_phaseA_two_runs_bit_identical():
    lev_np, _ = _case("holes10_smooth")
    lev = torch.as_tensor(lev_np).cuda()
    a = _glcm(lev, None)
    b = _glcm(lev, None)
    assert torch.equal(a.nan_to_num(nan=-7.0), b.nan_to_num(nan=-7.0))


def test_phaseA_slabs_through_hole_rich_planes_equal_whole_volume():
    """slab cuts at planes where most windows are not full: each voxel still takes the body its window selects"""
    rng = np.random.default_rng(12)
    lev_np = _levels("uniform", (40, 41, 43), 7)
    for z in (9, 10, 23, 31):
        lev_np[z][rng.random(lev_np.shape[1:]) < 0.4] = 0
    lev = torch.as_tensor(lev_np).cuda()
    whole = _glcm(lev, None)
    parts = [_glcm(lev, None, z0=a, z1=b) for a, b in ((0, 10), (10, 23), (23, 24), (24, 40))]
    assert torch.equal(torch.cat(parts, 1).nan_to_num(nan=-7.0), whole.nan_to_num(nan=-7.0))
