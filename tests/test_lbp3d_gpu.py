"""3-D LBP on the GPU (csrc/lbp3d.cu): getLBP3DImage against the reference's goldens and the NumPy/SciPy oracle, zeros
outside the ROI, bit-reproducibility, the uint16 clamp, the kernel's range and the opt-in pipeline images."""
import numpy as np
import pytest
import torch

import lbp3d_np
from pyradiomics_b200 import _lib, featureclasses as FC, image as I, imageoperations as IO
from test_lbp3d_cpu import NAMES, assert_lbp_close, load

pytestmark = pytest.mark.gpu


def run(img, mask, **kw):
    out = list(IO.getLBP3DImage(I.ArrayImage(img), I.ArrayImage(mask), **kw))
    return [n for _, n, _ in out], np.stack([I.as_array(im) for im, _, _ in out])


@pytest.mark.parametrize("name", NAMES)
def test_matches_golden_and_oracle(name):
    z, kw, L, R, S = load(name)
    img, mask = z["image"], z["mask"]
    roi = mask == 1
    names, maps = run(img, mask, **kw)
    assert names == [f"lbp-3D-m{i + 1}" for i in range(L)] + ["lbp-3D-k"]
    assert maps.dtype == np.float64 and maps.shape == (L + 1,) + img.shape
    got = maps[:, roi]
    o = lbp3d_np.lbp3d(img, roi, z["vertices"], L, R)
    if np.issubdtype(img.dtype, np.integer):
        keep = np.ones(roi.sum(), bool)             # no voxel within 1e-9 of a rounding tie (make_golden_lbp3d.py asserts it)
    else:
        keep = o["margin"] >= 1e-9 * np.abs(img).max()
        print(f"{name}: {int((~keep).sum())} of {keep.size} voxels within 1e-9 * max|img| of a sign flip, excluded")
        assert keep.mean() > 0.99
    is_f32 = img.dtype == np.float32
    assert_lbp_close(got[:, keep], o["maps"][:, keep], is_f32, name, o["m2"][keep], o["mean"][keep])
    assert_lbp_close(got[:, keep], z["maps"][:, keep], is_f32, name + " (golden)", o["m2"][keep], o["mean"][keep])
    assert (maps[:, ~roi] == 0).all()


def test_label_selects_the_roi():
    z, kw, L, R, S = load("s0")
    mask = z["mask"].astype(np.uint8) * 2                 # label 2 instead of 1
    _, a = run(z["image"], z["mask"], **kw)
    _, b = run(z["image"], mask, label=2, **kw)
    np.testing.assert_array_equal(a, b)


def test_two_runs_are_bit_identical():
    z, kw, L, R, S = load("brain1")
    _, a = run(z["image"], z["mask"], **kw)
    _, b = run(z["image"], z["mask"], **kw)
    assert a.tobytes() == b.tobytes()


def test_uint16_clamp():
    rng = np.random.default_rng(5)
    img = rng.integers(0, 65536, (10, 11, 12)).astype(np.uint16)
    img[3:7, 3:7, 3:7] = 65535                             # overshoot above 65535 and below 0 next to the steps
    img[:2] = 0
    mask = np.ones(img.shape, np.uint8)
    _, got = run(img, mask)
    o = lbp3d_np.lbp3d(img, mask == 1, IO._icosphere(1, 1.0), 2, 1.0)
    assert_lbp_close(got[:, mask == 1], o["maps"], False, "uint16", o["m2"], o["mean"])


def test_kernel_range_is_enforced_by_the_library():
    verts = np.ascontiguousarray(IO._icosphere(3, 1.0))
    harm = np.zeros((len(verts), 3, 2))
    t = torch.zeros((4, 4, 4), dtype=torch.int16, device="cuda")
    roi = torch.ones((4, 4, 4), dtype=torch.uint8, device="cuda")
    scratch = torch.empty((4, 4, 4), dtype=torch.float64, device="cuda")
    out = torch.empty((3, 4, 4, 4), dtype=torch.float64, device="cuda")
    import ctypes as C
    rc = _lib.lib().rb_lbp3d_dev(_lib.ptr(t), 0, 0, _lib.ptr(roi), 4, 4, 4, verts.ctypes.data_as(C.c_void_p), len(verts),
                                 harm.ctypes.data_as(C.c_void_p), 2, _lib.ptr(scratch), _lib.ptr(out), _lib.stream())
    assert rc == _lib.RB_ERR_UNSUPPORTED


def test_pipeline_lbp3d_images_equal_per_image_plugins():
    from pyradiomics_b200 import pipeline as PP
    import scipy.ndimage as ndi
    rng = np.random.default_rng(11)
    x = (ndi.gaussian_filter(rng.normal(size=(12, 13, 14)), 1.2) * 400 + 300).astype(np.int16)
    m = (rng.random(x.shape) < 0.8).astype(np.uint8)
    got = {}
    xt, mt = torch.as_tensor(x).cuda(), torch.as_tensor(m).cuda()
    info = PP.voxel_suite_with_filters(xt, mt, classes=("gldm",), wavelet=None, sigmas=(), lbp3d={}, binWidth=2,
                                       consume=lambda n, c, t: got.__setitem__((n, c), t.cpu().numpy().copy()))
    names = [n for n, _, _ in info]
    assert names == ["original", "lbp-3D-m1", "lbp-3D-m2", "lbp-3D-k"]
    default = PP.voxel_suite_with_filters(xt, mt, classes=("gldm",), wavelet=None, sigmas=(), binWidth=2)
    assert [n for n, _, _ in default] == ["original"]
    imgs = {n: im for im, n, _ in IO.getLBP3DImage(I.ArrayImage(x), I.ArrayImage(m))}
    dev = dict(PP.derived_images(xt, wavelet=None, sigmas=(), original=False, lbp3d={}, mask=mt))
    for n in names[1:]:
        np.testing.assert_array_equal(dev[n].cpu().numpy(), I.as_array(imgs[n]))
        ref = FC.FEATURE_CLASSES["gldm"](imgs[n], I.ArrayImage(m), voxelBased=True, binWidth=2).execute()
        for k, f in enumerate(_lib.feature_names("gldm")):
            assert np.allclose(got[(n, "gldm")][k], I.as_array(ref[f]), rtol=1e-9, atol=1e-11, equal_nan=True), (n, f)
