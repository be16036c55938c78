"""The 2-D LBP image of the device-resident suites on the GPU: pipeline.derived_images' 'lbp-2D' image (rb_lbp2d_cast_dev,
the codes stored in the image's own dtype) against getLBP2DImage's host cast bit for bit, and the voxel and segment suites
on it against the same suites run on the host-made image as 'original'."""
import numpy as np
import pytest
import torch

from pyradiomics_b200 import image as I, imageoperations as IO, pipeline
from test_lbp2d_cpu import NAMES, assert_bits_equal, load
from test_lbp2d_gpu import smooth_int

pytestmark = pytest.mark.gpu

METHODS = list(IO.LBP2D_METHODS)
DTYPES = [np.int16, np.int32, np.float32, np.float64, np.uint8, np.uint16, np.int64]


def upload(img):
    """a NumPy image on the device in its own dtype (a uint16 one as torch.uint16, which the LBP kernels read as such)"""
    return torch.from_numpy(np.ascontiguousarray(img)).cuda() if img.dtype == np.uint16 else IO._to_device(img)


def device_lbp(img, settings):
    out = dict(pipeline.derived_images(upload(img), wavelet=None, sigmas=(), original=False, lbp2d=settings))
    assert list(out) == ["lbp-2D"]
    return out["lbp-2D"].cpu().numpy()


def host_lbp(img, settings):
    (im, name, _), = IO.getLBP2DImage(I.ArrayImage(img), None, **settings)
    assert name == "lbp-2D"
    return np.ascontiguousarray(I.as_array(im))


def image_of(dtype, seed=3):
    raw = smooth_int((6, 15, 17), seed, 60.0)
    if np.issubdtype(dtype, np.unsignedinteger):
        raw = raw - raw.min()
    img = raw.astype(dtype)
    if dtype == np.uint16:
        img += np.uint16(60000)
    if dtype == np.int32:
        img *= 50000                                            # VAR beyond the int32 range
    if dtype == np.int64:
        img *= 1 << 40                                          # and beyond the int64 range
    if np.issubdtype(dtype, np.floating):
        img = img + np.asarray(0.37, dtype) * np.arange(img.size, dtype=dtype).reshape(img.shape) % 3
        img[1, 4, 4], img[2, 8, 9], img[3, 1, 1], img[4, 10, 10] = np.nan, np.inf, -np.inf, 1e30
    return img


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("method", METHODS)
def test_derived_image_matches_host_cast(dtype, method):
    img = image_of(dtype)
    for axis, P, R in [(0, 8, 1), (1, 9, 1), (2, 24, 3)]:     # P 9 'default' wraps uint8 and int16 codes
        kw = {"lbp2DMethod": method, "lbp2DSamples": P, "lbp2DRadius": R, "force2D": True, "force2Ddimension": axis}
        got, ref = device_lbp(img, kw), host_lbp(img, kw)
        assert ref.dtype == img.dtype
        assert_bits_equal(got, ref, f"{np.dtype(dtype)} {method} axis {axis}")


@pytest.mark.parametrize("name", [n for n in NAMES if load(n)[0]["image"].ndim == 3])
def test_derived_image_matches_golden(name):
    z, kw, _ = load(name)
    assert_bits_equal(device_lbp(z["image"], kw), z["out"], name)


def value(v):
    """a segment feature value as a 1-element float64 array (assert_bits_equal compares arrays)"""
    return np.atleast_1d(np.asarray(v, np.float64))


def case(dtype=np.int16, seed=11, shape=(9, 13, 15)):
    img = smooth_int(shape, seed, 80.0).astype(dtype)
    mask = (np.random.default_rng(seed).random(shape) < 0.85).astype(np.uint8)
    mask[0] = 0
    return img, mask


def voxel_maps(image, mask, **kw):
    maps = {}
    pipeline.voxel_suite_with_filters(image, mask, classes=("firstorder",) + pipeline.CLASSES, wavelet=None, sigmas=(),
                                      consume=lambda n, c, m: maps.__setitem__((n, c), m.cpu().numpy().copy()), **kw)
    return maps


@pytest.mark.parametrize("map_dtype,axis", [(torch.float64, None), (torch.float32, None), (torch.float64, 0),
                                            (torch.float64, 1), (torch.float64, 2)])
def test_voxel_suite_matches_host_made_image(map_dtype, axis):
    img, mask = case()
    kw = {"binCount": 16, "map_dtype": map_dtype}
    if axis is not None:
        kw.update(force2D=True, force2Ddimension=axis)
    lbp = {"lbp2DMethod": "uniform", "lbp2DSamples": 8}
    got = voxel_maps(upload(img), upload(mask), lbp2d=lbp, **kw)
    ref = voxel_maps(upload(host_lbp(img, {**lbp, "force2D": axis is not None, "force2Ddimension": axis or 0})),
                     upload(mask), **kw)
    classes = ("firstorder",) + pipeline.CLASSES
    assert sorted(got) == sorted([("original", c) for c in classes] + [("lbp-2D", c) for c in classes])
    for c in classes:
        assert_bits_equal(got[("lbp-2D", c)], ref[("original", c)], f"{c} axis {axis} {map_dtype}")


@pytest.mark.parametrize("dtype,lbp", [(np.int16, {}), (np.float32, {"lbp2DMethod": "var", "lbp2DRadius": 1.5}),
                                       (np.uint8, {"lbp2DMethod": "default", "lbp2DSamples": 9, "force2Ddimension": 2})])
def test_segment_suite_matches_host_made_image(dtype, lbp):
    img, mask = case(dtype, 12)
    kw = {"binCount": 16, "shape": False, "wavelet": None, "sigmas": ()}
    got = pipeline.segment_suite_with_filters(upload(img), upload(mask), lbp2d=lbp, **kw)
    ref = pipeline.segment_suite_with_filters(upload(host_lbp(img, lbp)), upload(mask), **kw)
    lbp_keys = [k for k in got if k.startswith("lbp-2D_")]
    assert lbp_keys == ["lbp-2D_" + k[len("original_"):] for k in ref]
    for k in lbp_keys:
        assert_bits_equal(value(got[k]), value(ref["original_" + k[len("lbp-2D_"):]]), k)


def test_segment_suite_resegmented_roi():
    img, mask = case(np.int16, 13)
    roi = torch.as_tensor(mask).cuda()
    reseg, _, _ = IO.resegment_mask_device(upload(img), roi, [-40, 60], "absolute")
    kw = {"binCount": 16, "shape": False, "wavelet": None, "sigmas": ()}
    got = pipeline.segment_suite_with_filters(upload(img), roi, lbp2d={}, resegment={"resegmentRange": [-40, 60]}, **kw)
    ref = pipeline.segment_suite_with_filters(upload(host_lbp(img, {})), reseg, **kw)
    for k, v in ref.items():
        assert_bits_equal(value(got["lbp-2D_" + k[len("original_"):]]), value(v), k)


def test_caller_stream_and_repeat_runs_are_bit_identical():
    for dtype in (np.int16, np.float32):
        x = upload(image_of(dtype, 5))
        for method in METHODS:
            kw = {"lbp2DMethod": method, "lbp2DSamples": 24, "lbp2DRadius": 3, "force2Ddimension": 2}
            a = dict(pipeline.derived_images(x, wavelet=None, sigmas=(), original=False, lbp2d=kw))["lbp-2D"]
            b = dict(pipeline.derived_images(x, wavelet=None, sigmas=(), original=False, lbp2d=kw))["lbp-2D"]
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                c = dict(pipeline.derived_images(x, wavelet=None, sigmas=(), original=False, lbp2d=kw))["lbp-2D"]
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            assert_bits_equal(b.cpu().numpy(), a.cpu().numpy(), f"{method} repeat")
            assert_bits_equal(c.cpu().numpy(), a.cpu().numpy(), f"{method} stream")


def test_without_lbp2d_nothing_changes():
    img, mask = case(np.int16, 14)
    kw = {"binWidth": 10, "wavelet": None, "sigmas": (1.0,), "image_types": ("square",)}
    base = pipeline.segment_suite_with_filters(upload(img), upload(mask), **kw)
    with_lbp = pipeline.segment_suite_with_filters(upload(img), upload(mask), lbp2d={}, **kw)
    assert not [k for k in base if k.startswith("lbp-2D")]
    assert [k for k in with_lbp if not k.startswith("lbp-2D")] == list(base)
    for k, v in base.items():
        assert_bits_equal(value(with_lbp[k]), value(v), k)
    names = [n for n, _, _ in pipeline.voxel_suite_with_filters(upload(img), upload(mask), classes=("glcm",), **kw)]
    assert names == ["original", "log-sigma-1-0-mm-3D", "square"]
