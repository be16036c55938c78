"""2-D LBP on the GPU (csrc/lbp2d.cu): lbp2d_device against the NumPy oracle bit for bit for every method, slicing axis
and upload dtype, getLBP2DImage against the reference's goldens, bit-reproducibility, the envelope and degenerate slices."""
import ctypes as C

import numpy as np
import pytest
import torch

import lbp2d_np
from pyradiomics_b200 import _lib, image as I, imageoperations as IO
from test_lbp2d_cpu import NAMES, assert_bits_equal, load

pytestmark = pytest.mark.gpu

METHODS = list(IO.LBP2D_METHODS)


def smooth_int(shape, seed, scale=200.0):
    f = np.random.default_rng(seed).normal(size=shape)
    for ax in range(f.ndim):
        f = (np.roll(f, 1, ax) + 2 * f + np.roll(f, -1, ax)) / 4
    return np.round(f * scale)


def device(img, P, R, method, axis):
    return IO.lbp2d_device(IO._to_device(img), axis, P, R, method).cpu().numpy()


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("axis", [0, 1, 2, "2d"])
def test_every_method_and_axis_matches_oracle(method, axis):
    if axis == "2d":
        img, axis = smooth_int((37, 41), 1).astype(np.int16), 0
    else:
        img = smooth_int((9, 21, 23), 2).astype(np.int16)
    for P, R in [(8, 1), (24, 3), (6, 1.5), (4, 0.5)]:
        assert_bits_equal(device(img, P, R, method, axis), lbp2d_np.lbp2d_volume(img, P, R, method, axis),
                          f"{method} axis {axis} P {P} R {R}")


@pytest.mark.parametrize("dtype", [np.uint8, np.int16, np.uint16, np.int32, np.int64, np.float32, np.float64])
@pytest.mark.parametrize("method", METHODS)
def test_every_upload_dtype_matches_oracle(dtype, method):
    raw = smooth_int((6, 17, 19), 3, 60.0)
    if np.issubdtype(dtype, np.unsignedinteger):
        raw = raw - raw.min()
    img = raw.astype(dtype)
    if dtype == np.uint16:
        img = img + np.uint16(60000)                          # values only uint16 holds: travel as int32
    if np.issubdtype(dtype, np.floating):
        img = img + np.asarray(0.37, dtype) * np.arange(img.size, dtype=dtype).reshape(img.shape) % 3
        img[1, 4, 4], img[2, 8, 9], img[3, 1, 1], img[4, 10, 10] = np.nan, np.inf, -np.inf, np.inf
    for axis in (0, 2):
        assert_bits_equal(device(img, 8, 1, method, axis), lbp2d_np.lbp2d_volume(img, 8, 1, method, axis),
                          f"{np.dtype(dtype)} {method} axis {axis}")


@pytest.mark.parametrize("name", NAMES)
def test_generator_matches_golden(name):
    z, kw, _ = load(name)
    out = list(IO.getLBP2DImage(I.ArrayImage(z["image"]), None, **kw))
    assert [n for _, n, _ in out] == ["lbp-2D"]
    assert out[0][2] is not None
    assert_bits_equal(np.ascontiguousarray(I.as_array(out[0][0])), z["out"], name)


def test_two_runs_are_bit_identical():
    img = torch.as_tensor(smooth_int((12, 40, 44), 4).astype(np.int16)).cuda()
    for method in METHODS:
        a = IO.lbp2d_device(img, 2, 24, 3, method)
        b = IO.lbp2d_device(img, 2, 24, 3, method)
        assert torch.equal(a.view(torch.int64), b.view(torch.int64)), method


@pytest.mark.parametrize("kw,exc", [({"samples": 0}, ValueError), ({"samples": 32}, ValueError),
                                    ({"radius": 0}, ValueError), ({"radius": -2}, ValueError),
                                    ({"method": "sobel"}, KeyError)])
def test_envelope_rejections_raise_before_a_launch(kw, exc):
    img = torch.zeros((3, 4, 5), dtype=torch.int16, device="cuda")
    torch.cuda.synchronize()
    with pytest.raises(exc):
        IO.lbp2d_device(img, **kw)


def test_library_rejects_32_samples():
    P = 32
    rp = np.zeros(P)
    cp = np.ones(P)
    t = torch.zeros((2, 4, 4), dtype=torch.int16, device="cuda")
    out = torch.empty((2, 4, 4), dtype=torch.float64, device="cuda")
    rc = _lib.lib().rb_lbp2d_dev(_lib.ptr(t), 0, 2, 4, 4, 0, P, rp.ctypes.data_as(C.c_void_p), cp.ctypes.data_as(C.c_void_p),
                                 IO.LBP2D_METHODS["default"], _lib.ptr(out), _lib.stream())
    assert rc == _lib.RB_ERR_UNSUPPORTED


@pytest.mark.parametrize("shape,axis", [((1, 9), 0), ((9, 1), 0), ((1, 1), 0), ((1, 1, 1), 0), ((4, 1, 7), 0),
                                        ((4, 7, 1), 0), ((1, 5, 6), 1), ((5, 1, 6), 1), ((5, 6, 1), 2), ((1, 6, 5), 2)])
@pytest.mark.parametrize("method", METHODS)
def test_degenerate_slices(shape, axis, method):
    img = smooth_int(shape, 6, 50.0).astype(np.int32) + np.arange(int(np.prod(shape)), dtype=np.int32).reshape(shape) % 4
    for P, R in [(8, 1), (4, 2)]:
        assert_bits_equal(device(img, P, R, method, axis), lbp2d_np.lbp2d_volume(img, P, R, method, axis),
                          f"{shape} axis {axis} {method}")


def test_2d_generator_is_float64_and_3d_keeps_dtype():
    img = smooth_int((2, 9, 10), 7).astype(np.int16)
    (im3, n3, _), = IO.getLBP2DImage(I.ArrayImage(img), None, force2D=True)
    (im2, n2, _), = IO.getLBP2DImage(I.ArrayImage(img[0]), None)
    assert I.as_array(im3).dtype == np.int16 and I.as_array(im2).dtype == np.float64
    np.testing.assert_array_equal(I.as_array(im3)[0], I.as_array(im2).astype(np.int16))


def test_negative_axis_is_swapaxes():
    img = smooth_int((5, 8, 9), 8).astype(np.int16)
    (a, _, _), = IO.getLBP2DImage(I.ArrayImage(img), None, force2Ddimension=-1)
    (b, _, _), = IO.getLBP2DImage(I.ArrayImage(img), None, force2Ddimension=2)
    np.testing.assert_array_equal(I.as_array(a), I.as_array(b))
