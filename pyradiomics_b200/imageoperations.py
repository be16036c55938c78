"""GPU versions of the pyradiomics image operations that sit on the texture hot path
(reference radiomics/imageoperations.py): gray-level discretisation (getBinEdges / binImage,
:67-174), the level-1 stationary wavelet decomposition (getWaveletImage / _swt3, :839-970), the
Laplacian-of-Gaussian filter (getLoGImage, :756-836), the per-voxel square / square root /
logarithm / exponential images (getSquareImage ... getExponentialImage, :973-1073), the gradient
magnitude (getGradientImage, :1076-1091), the 3-D local binary pattern (getLBP3DImage,
:1169-1314), and the two preprocessing steps in front of them: image normalisation (normalizeImage,
:615-654) and mask resegmentation (resegmentMask, :657-742).  Same function names, arguments and
yielded tuples as the reference so they can be dropped into ``radiomics.imageoperations``.

Parity status (DESIGN.md): resegmentation masks equal the reference's (float32 sigma mode up to the
few-ulp difference of a float64 ROI reduction); normalisation restates ITK's Normalize (unpinned
details in DESIGN.md section 5); binning, square and square root are bit-identical to NumPy, logarithm and
exponential within CUDA's 1-ulp log / exp; wavelet, LoG and gradient restate PyWavelets' and ITK's
published algorithms -- neither library is available offline and the reference's own tests do not
pin them (SURVEY.md section 8c) -> "parity unpinned" for those three.
"""
from __future__ import annotations

import ctypes as C
import logging
import math

import numpy as np
import torch

from . import image as I
from ._lib import check, lib

logger = logging.getLogger("radiomics.imageoperations")

_DT = {np.dtype("int16"): 0, np.dtype("int32"): 1, np.dtype("float32"): 2, np.dtype("float64"): 3,
       np.dtype("uint8"): 4, np.dtype("uint16"): 5, np.dtype("int64"): 6}
_TORCH_DT = {torch.int16: 0, torch.int32: 1, torch.float32: 2, torch.float64: 3, torch.uint8: 4, torch.int64: 6}


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev():
    return torch.device("cuda", torch.cuda.current_device())


_TORCH_OF_NP = {np.int16: torch.int16, np.int32: torch.int32, np.float32: torch.float32, np.float64: torch.float64,
                np.uint8: torch.uint8, np.int64: torch.int64}
_STAGE = {"bufs": None, "pool": None}
_STAGE_CHUNK = 32 << 20
_STAGE_MIN = 64 << 20


def _upload_staged(a):
    """pageable NumPy array -> CUDA tensor through two page-locked 32 MB staging blocks: a few threads copy chunk k+1 into
    one block (NumPy releases the GIL) while the DMA engine drains chunk k from the other.  A plain ``tensor.to(device)`` of
    pageable memory lets the driver stage it single-threaded, at a fraction of the link's rate."""
    import concurrent.futures as cf
    flat = a.reshape(-1).view(np.uint8)
    n = flat.size
    dev = _dev()
    out = torch.empty(n, dtype=torch.uint8, device=dev)
    if _STAGE["bufs"] is None:
        _STAGE["bufs"] = [torch.empty(_STAGE_CHUNK, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
        _STAGE["pool"] = cf.ThreadPoolExecutor(max_workers=4)
    bufs, pool = _STAGE["bufs"], _STAGE["pool"]
    views = [b.numpy() for b in bufs]
    done = [None, None]
    stream = torch.cuda.current_stream()
    for k, off in enumerate(range(0, n, _STAGE_CHUNK)):
        m = min(_STAGE_CHUNK, n - off)
        j = k & 1
        if done[j] is not None:
            done[j].synchronize()                   # the DMA out of this block has finished
        q = (m + 3) // 4
        list(pool.map(lambda s: np.copyto(views[j][s:min(s + q, m)], flat[off + s:off + min(s + q, m)]), range(0, m, q)))
        out[off:off + m].copy_(bufs[j][:m], non_blocking=True)
        done[j] = torch.cuda.Event()
        done[j].record(stream)
    for e in done:
        if e is not None:
            e.synchronize()                         # the staging blocks are reused by the next upload
    return out.view(_TORCH_OF_NP[a.dtype.type]).reshape(a.shape)


def _to_device(arr):
    """NumPy / torch -> contiguous CUDA tensor of a supported dtype (uint16 travels as int32)."""
    if isinstance(arr, torch.Tensor):
        t = arr
        if t.dtype == torch.bool:
            t = t.to(torch.uint8)
        if t.dtype not in _TORCH_DT:
            t = t.to(torch.float64)
        return t.to(_dev()).contiguous()
    a = np.asarray(arr)
    if a.dtype == np.bool_:
        a = a.view(np.uint8)
    elif a.dtype == np.uint16:
        a = a.astype(np.int32)
    elif a.dtype not in _DT:
        a = a.astype(np.float64)
    a = np.ascontiguousarray(a)
    if a.nbytes >= _STAGE_MIN and a.dtype.type in _TORCH_OF_NP:
        return _upload_staged(a)
    return torch.from_numpy(a).to(_dev())


def _decode_key(k: int) -> float:
    bits = k if k >= 0 else k ^ 0x7FFFFFFFFFFFFFFF
    return float(np.array([bits], dtype=np.int64).view(np.float64)[0])


def roi_minmax(img_t: torch.Tensor, mask_t: torch.Tensor | None):
    """(min, max, count) of the ROI, one streaming kernel (replaces builtin min()/max())."""
    keys = torch.tensor([2 ** 63 - 1, -(2 ** 63), 0], dtype=torch.int64, device=img_t.device)
    check(lib().rb_minmax_dev(_ptr(img_t), _TORCH_DT[img_t.dtype], _ptr(mask_t), C.c_longlong(img_t.numel()), _ptr(keys),
                              _stream()), "minmax")
    k = keys.cpu().tolist()
    if k[2] == 0:
        raise ValueError("empty ROI")
    return _decode_key(k[0]), _decode_key(k[1]), k[2]


_NP_OF_TORCH = {torch.int16: np.int16, torch.int32: np.int32, torch.float32: np.float32, torch.float64: np.float64,
                torch.uint8: np.uint8, torch.int64: np.int64}


def _edges_from_minmax(minimum, maximum, np_type, **kwargs):
    """reference getBinEdges arithmetic (imageoperations.py:119-149) on the scalars min / max, carried
    out in the image's own NumPy scalar type so that float32 / integer inputs round exactly as
    `min(values) - (min(values) % binWidth)`, np.arange and np.histogram do in the reference."""
    binWidth = kwargs.get("binWidth", 25)
    binCount = kwargs.get("binCount")
    minimum, maximum = np_type(minimum), np_type(maximum)
    if binCount is not None:
        # np.histogram(values, binCount)[1]: linspace(min, max, binCount + 1) in the result type of
        # the data (float64 for integers), degenerate range widened by +-0.5; then last edge + 1
        et = np.dtype(np.float64) if np.issubdtype(np_type, np.integer) else np.dtype(np_type)
        lo, hi = et.type(minimum), et.type(maximum)
        if lo == hi:
            lo, hi = lo - et.type(0.5), hi + et.type(0.5)
        e = np.linspace(lo, hi, int(binCount) + 1, endpoint=True, dtype=et)
        e[-1] += 1
        return e
    lowBound = minimum - (minimum % binWidth)
    highBound = maximum + 2 * binWidth
    e = np.arange(lowBound, highBound, binWidth)
    if len(e) == 1:
        e = np.array([e[0] - 0.5, e[0] + 0.5])
    return e


def getBinEdges(parameterValues, **kwargs):
    """reference signature: 1-D array of the segmented voxel values -> bin edges."""
    t = _to_device(parameterValues).reshape(-1)
    mn, mx, _ = roi_minmax(t, None)
    return _edges_from_minmax(mn, mx, _NP_OF_TORCH[t.dtype], **kwargs)


def bin_image_device(img_t: torch.Tensor, mask_t: torch.Tensor | None, minmax_reduce=None, **kwargs):
    """device tensors in -> (int32 levels tensor (0 outside the mask), edges ndarray).  `minmax_reduce(mn, mx)` turns a
    slab's ROI minimum / maximum into the whole ROI's (multi-GPU: all-reduce MIN / MAX), so every rank bins with the
    same edges."""
    mn, mx, _ = roi_minmax(img_t, mask_t)
    if minmax_reduce is not None:
        mn, mx = minmax_reduce(mn, mx)
    edges_native = _edges_from_minmax(mn, mx, _NP_OF_TORCH[img_t.dtype], **kwargs)
    edges = np.ascontiguousarray(edges_native, dtype=np.float64)
    e_t = torch.from_numpy(edges).to(img_t.device)
    out = torch.empty(img_t.shape, dtype=torch.int32, device=img_t.device)
    check(lib().rb_digitize_dev(_ptr(img_t), _TORCH_DT[img_t.dtype], _ptr(mask_t), C.c_longlong(img_t.numel()), _ptr(e_t),
                                int(edges.size), _ptr(out), _stream()), "digitize")
    return out, edges_native


def binImage(parameterMatrix, parameterMatrixCoordinates=None, **kwargs):
    """reference signature (imageoperations.py:156): returns (discretised int array, binEdges).
    `parameterMatrixCoordinates` is the boolean ROI mask the feature classes pass."""
    img_t = _to_device(parameterMatrix)
    mask_t = None
    if parameterMatrixCoordinates is not None:
        m = np.asarray(parameterMatrixCoordinates)
        if m.dtype != np.bool_ or m.shape != tuple(img_t.shape):
            mm = np.zeros(tuple(img_t.shape), dtype=bool)
            mm[parameterMatrixCoordinates] = True
            m = mm
        mask_t = _to_device(m)
    out, edges = bin_image_device(img_t, mask_t, **kwargs)
    return out.cpu().numpy().astype(np.int64), edges


# ------------------------------------------------------------------------------------ cropping
def cropToTumorMask(imageNode, maskNode, boundingBox, **kwargs):
    """reference signature (imageoperations.py:407-445): crop image and mask to the ROI's bounding box
    `boundingBox` = (x_lo, x_hi, y_lo, y_hi, z_lo, z_hi) (inclusive, SimpleITK x,y,z order, as checkMask returns it),
    grown by kwargs['padDistance'] voxels on every side and clipped to the image (the orchestrator passes
    padDistance = kernelRadius in voxel-based mode, 0 otherwise: featureextractor.py:304-307,385-387).  Host-side
    slicing (views, no copy): the crop decides which voxels ever reach the GPU."""
    padDistance = int(kwargs.get("padDistance", 0))
    bb = np.asarray(boundingBox, dtype=np.int64)
    size = np.array(I.size_xyz(maskNode), dtype=np.int64)
    nd = size.size
    lo = np.maximum(bb[0::2][:nd] - padDistance, 0)
    hi = np.minimum(bb[1::2][:nd] + padDistance, size - 1)
    logger.debug("Cropping to size %s", (bb[1::2][:nd] - bb[0::2][:nd]) + 1)
    sl = tuple(slice(int(lo[d]), int(hi[d]) + 1) for d in range(nd))[::-1]          # arrays are (z,y,x)
    return I.like(imageNode, I.as_array(imageNode)[sl]), I.like(maskNode, I.as_array(maskNode)[sl])


# ------------------------------------------------------------------------------------ resampling
_INTERPOLATORS = {"sitkNearestNeighbor": 0, "sitkLinear": 1, "sitkBSpline": 3, 1: 0, 2: 1, 3: 3}      # (sitk enum values 1, 2, 3)
_NP_DT = {np.dtype("int16"): 0, np.dtype("int32"): 1, np.dtype("float32"): 2, np.dtype("float64"): 3, np.dtype("uint8"): 4,
          np.dtype("int64"): 6}


def resample_device(arr_t: torch.Tensor, out_size_zyx, start_zyx, step_zyx, interpolator=3, default_value=0.0, out_dtype=None):
    """CUDA tensor (Z,Y,X) -> CUDA tensor of `out_size_zyx` sampled at input continuous indices start + k * step
    (rb_bspline_prefilter_dev + rb_resample_dev); cubic B-spline (3), linear (1) or nearest neighbour (0); the result is
    clamped and truncated to `out_dtype` (default: the input's) like ITK's ResampleImageFilter"""
    src = arr_t.contiguous()
    out_dtype = out_dtype or src.dtype
    if out_dtype not in _TORCH_DT:
        raise ValueError(f"unsupported pixel type {out_dtype}")
    Z, Y, X = src.shape
    dst = torch.empty(tuple(int(v) for v in out_size_zyx), dtype=out_dtype, device=src.device)
    if interpolator == 3:
        src = src.to(torch.float64).clone()
        check(lib().rb_bspline_prefilter_dev(_ptr(src), Z, Y, X, _stream()), "bspline prefilter")
    elif src.dtype not in _TORCH_DT:
        src = src.to(torch.float64)
    isz = (C.c_int * 3)(Z, Y, X)
    osz = (C.c_int * 3)(*[int(v) for v in out_size_zyx])
    st = (C.c_double * 3)(*[float(v) for v in start_zyx])
    sp = (C.c_double * 3)(*[float(v) for v in step_zyx])
    check(lib().rb_resample_dev(_ptr(src), _TORCH_DT[src.dtype], isz, _ptr(dst), _TORCH_DT[out_dtype], osz, st, sp, int(interpolator),
                                C.c_double(float(default_value)), _stream()), "resample")
    return dst


def resampleImage(imageNode, maskNode, **kwargs):
    """reference signature (radiomics/imageoperations.py:448-612): resample image (B-spline by default) and mask (nearest
    neighbour) to `resampledPixelSpacing`, cropped to the ROI's bounding box grown by `padDistance` new-grid voxels; the
    grid is aligned to the input origin.  The geometry arithmetic is the reference's (:509-566); image and mask are taken
    to share one axis-aligned grid (the array stand-in of SimpleITK images carries spacing and origin, no direction
    cosines).  Interpolation and cast happen on the GPU (resample_device)."""
    resampledPixelSpacing = kwargs["resampledPixelSpacing"]
    interpolator = kwargs.get("interpolator", "sitkBSpline")
    padDistance = kwargs.get("padDistance", 5)
    label = int(kwargs.get("label", 1))
    if imageNode is None or maskNode is None:
        raise ValueError("Requires both image and mask to resample")
    img, msk = I.as_array(imageNode), I.as_array(maskNode)
    if img.shape != msk.shape:
        raise ValueError("image and mask must share one grid")
    nd = msk.ndim
    maskSpacing = np.array(I.spacing_xyz(maskNode), dtype=np.float64)
    assert len(resampledPixelSpacing) == nd, f"Wrong dimensionality ({len(resampledPixelSpacing)}-D) of resampledPixelSpacing!, {nd}-D required"
    newSp = np.array(resampledPixelSpacing, dtype=np.float64)
    newSp = np.where(newSp == 0, maskSpacing, newSp)
    # bounding box (lower bounds then sizes, x,y,z) of the label: what LabelShapeStatisticsImageFilter gives _checkROI (:346-404)
    idx = np.array(np.where(msk == label))
    if idx.shape[1] == 0:
        raise ValueError(f"Label ({label}) not present in mask")
    lo, hi = idx.min(1)[::-1], idx.max(1)[::-1]
    bb = np.concatenate([lo, hi - lo + 1]).astype(np.float64)
    maskSize = np.array(msk.shape[::-1], dtype=np.float64)
    newSp = np.where(bb[nd:] != 1, newSp, maskSpacing)                  # no resampling across a single-slice ROI (:509-511)
    if np.allclose(maskSpacing, newSp):                                  # nothing to interpolate: crop only (:517-537)
        low_up = np.empty(nd * 2, dtype=int)
        low_up[::2], low_up[1::2] = lo, hi
        return cropToTumorMask(imageNode, maskNode, low_up, **kwargs)
    ratio = maskSpacing / newSp
    L = np.floor((bb[:nd] - 0.5) * ratio - padDistance)
    U = np.ceil((bb[:nd] + bb[nd:] - 0.5) * ratio + padDistance)
    maxU = np.ceil(maskSize * ratio) - 1
    L = np.where(L < 0, 0, L)
    U = np.where(U > maxU, maxU, U)
    newSize = np.array(U - L + 1, dtype=int)
    start = 0.5 * (newSp - maskSpacing) / maskSpacing + L / ratio       # continuous index of output voxel 0 (:549-556)
    step = newSp / maskSpacing
    if isinstance(interpolator, str) and interpolator not in _INTERPOLATORS:
        logger.warning('interpolator "%s" not recognized, using sitkBSpline', interpolator)
        interpolator = "sitkBSpline"
    if interpolator not in _INTERPOLATORS:
        raise ValueError(f"interpolator {interpolator!r} is not implemented (sitkBSpline, sitkLinear, sitkNearestNeighbor)")
    logger.info("Applying resampling from spacing %s and size %s to spacing %s and size %s", maskSpacing, maskSize, newSp, newSize)
    pad3 = (1,) * (3 - nd)
    img_t = _to_device(img).reshape(pad3 + img.shape)
    msk_t = _to_device(msk).reshape(pad3 + msk.shape)
    osz = pad3 + tuple(int(v) for v in newSize[::-1])
    st3 = (0.0,) * (3 - nd) + tuple(start[::-1])
    sp3 = (1.0,) * (3 - nd) + tuple(step[::-1])
    out_img = resample_device(img_t, osz, st3, sp3, _INTERPOLATORS[interpolator])
    out_msk = resample_device(msk_t, osz, st3, sp3, 0)
    origin = np.array(I.origin_xyz(maskNode), dtype=np.float64) + start * maskSpacing      # TransformContinuousIndexToPhysicalPoint (:557)
    a_img = out_img.cpu().numpy().reshape(osz[3 - nd:]).astype(img.dtype, copy=False)
    a_msk = out_msk.cpu().numpy().reshape(osz[3 - nd:]).astype(msk.dtype if msk.dtype != np.bool_ else np.uint8, copy=False)
    return I.ArrayImage(a_img, tuple(newSp), tuple(origin)), I.ArrayImage(a_msk, tuple(newSp), tuple(origin))


# ------------------------------------------------------------------------------------ wavelet
# decomposition low-pass filters (PyWavelets conventions); dec_hi[k] = (-1)^(k+1) dec_lo[F-1-k]
_DEC_LO = {
    "haar": [0.7071067811865476, 0.7071067811865476],
    "db1": [0.7071067811865476, 0.7071067811865476],
    "db2": [-0.12940952255126037, 0.2241438680420134, 0.8365163037378079, 0.48296291314453416],
    "sym2": [-0.12940952255126037, 0.2241438680420134, 0.8365163037378079, 0.48296291314453416],
    "coif1": [-0.01565572813546454, -0.0727326195128539, 0.38486484686420286, 0.8525720202122554,
              0.3378976624578092, -0.0727326195128539],
}


def wavelet_filters(name):
    if not isinstance(name, str):          # a pywt.Wavelet-like object
        return np.asarray(name.dec_lo, float), np.asarray(name.dec_hi, float)
    if name not in _DEC_LO:
        raise ValueError(f"wavelet '{name}' is not in the built-in table {sorted(_DEC_LO)}; pass an object with dec_lo/dec_hi")
    lo = np.asarray(_DEC_LO[name], float)
    F = lo.size
    hi = np.array([(-1) ** (k + 1) * lo[F - 1 - k] for k in range(F)])
    return lo, hi


def swt_level1_device(x: torch.Tensor, axes, lo, hi, z_range=None):
    """one undecimated level over `axes` (in that order) of a float64 CUDA volume (Z,Y,X), periodic extension:
    {'aad': tensor, ...} with one letter per axis in `axes` order, like pywt.swtn.  Three axes with a 2/4/6/8-tap
    filter take the fused single-pass kernel (rb_swt3d_dev); anything else runs one axis per pass."""
    Z, Y, X = x.shape
    lo = np.ascontiguousarray(lo, dtype=np.float64)
    hi = np.ascontiguousarray(hi, dtype=np.float64)
    axes = [int(a) for a in axes]
    if sorted(axes) == [0, 1, 2] and lo.size in (2, 4, 6, 8):
        x = x.contiguous()
        zb, ze = (0, Z) if z_range is None else (int(z_range[0]), int(z_range[1]))      # slab + halo in, interior planes out
        out = torch.empty((8, ze - zb, Y, X), dtype=torch.float64, device=x.device)
        check(lib().rb_swt3d_dev(_ptr(x), Z, Y, X, lo.ctypes.data_as(C.c_void_p), hi.ctypes.data_as(C.c_void_p), int(lo.size),
                                 _ptr(out), C.c_longlong(out.stride(0)), zb, ze, _stream()), "swt3d")
        res = {}
        for b in range(8):
            band = {2: b & 1, 1: b >> 1 & 1, 0: b >> 2 & 1}          # axis (0 = z, 1 = y, 2 = x) -> high-pass?
            res["".join("d" if band[a] else "a" for a in axes)] = out[b]
        return res
    if z_range is not None:
        raise ValueError("z_range needs the fused 3-D kernel (three axes, 2/4/6/8 taps)")
    cur = {"": x}
    for ax in axes:
        nxt = {}
        for key, t in cur.items():
            a = torch.empty_like(t)
            d = torch.empty_like(t)
            check(lib().rb_swt_axis_dev(_ptr(t), Z, Y, X, int(ax), lo.ctypes.data_as(C.c_void_p), hi.ctypes.data_as(C.c_void_p),
                                        int(lo.size), _ptr(a), _ptr(d), _stream()), "swt")
            nxt[key + "a"], nxt[key + "d"] = a, d
        cur = nxt
    return cur


def _wrap_pad_even(data: torch.Tensor, axes3):
    """reference imageoperations.py:914-919: every transformed axis of odd length gets ONE wrap-around sample appended;
    returns the padded tensor and the crop slices that undo it (:947-951, :961-963)"""
    crop = [slice(None)] * 3
    for ax in axes3:
        if data.shape[ax] % 2:
            crop[ax] = slice(0, data.shape[ax])
            data = torch.cat([data, data.narrow(ax, 0, 1)], dim=ax)
    return data.contiguous(), tuple(crop)


def _swt3(inputImage, axes, **kwargs):
    """reference _swt3 (imageoperations.py:899-970): pad ONCE, keep the padded approximation between the levels (each
    level is a level-1 transform of the previous approximation), crop only what is handed out"""
    wavelet = kwargs.get("wavelet", "coif1")
    level = kwargs.get("level", 1)
    start_level = kwargs.get("start_level", 0)
    lo, hi = wavelet_filters(wavelet)
    arr = I.as_array(inputImage)
    nd = arr.ndim
    data = _to_device(arr).to(torch.float64)
    if nd == 2:
        data = data[None]
    ax3 = [a + (3 - nd) for a in axes]
    data, crop = _wrap_pad_even(data, ax3)
    key_a = "a" * len(axes)
    for _ in range(start_level):
        data = swt_level1_device(data, ax3, lo, hi)[key_a]
    ret = []
    for _ in range(start_level, start_level + level):
        dec = swt_level1_device(data, ax3, lo, hi)
        data = dec[key_a]
        dec_im = {}
        for name, t in dec.items():
            if name == key_a:
                continue
            a = t[crop].cpu().numpy()
            dec_im[name.replace("a", "L").replace("d", "H")] = I.like(inputImage, a[0] if nd == 2 else a)
        ret.append(dec_im)
    a = data[crop].cpu().numpy()
    return I.like(inputImage, a[0] if nd == 2 else a), ret


def getWaveletImage(inputImage, _inputMask, **kwargs):
    """reference generator (imageoperations.py:839-896): yields (image, name, kwargs)."""
    Nd = I.as_array(inputImage).ndim
    axes = list(range(Nd - 1, -1, -1))
    if kwargs.get("force2D", False):
        axes.remove(kwargs.get("force2Ddimension", 0))
    approx, ret = _swt3(inputImage, tuple(axes), **kwargs)
    for idx, wl in enumerate(ret, start=1):
        for decompositionName, decompositionImage in wl.items():
            name = f"wavelet-{decompositionName}" if idx == 1 else f"wavelet{idx}-{decompositionName}"
            yield decompositionImage, name, kwargs
    name = f"wavelet-{'L' * len(axes)}" if len(ret) == 1 else f"wavelet{len(ret)}-{'L' * len(axes)}"
    yield approx, name, kwargs


# ------------------------------------------------------------------------------------ LoG
def recursive_gaussian_coefficients(sigmad: float, order: int, scale_norm: float = 1.0):
    """Deriche-type 4th-order recursive Gaussian (Farneback-Westin parameterisation) as used by ITK's
    RecursiveGaussianImageFilter: returns the 20 coefficients N0..3, D1..4, M1..4, BN1..4, BM1..4 for
    smoothing (order 0) or the second derivative (order 2), sigma in voxels."""
    A1 = (1.3530, -0.6724, -1.3563); B1 = (1.8151, -3.4327, 5.2318); W1 = 0.6681; L1 = -1.3932
    A2 = (-0.3531, 0.6724, 0.3446); B2 = (0.0902, 0.6100, -2.2355); W2 = 2.0787; L2 = -1.3732
    s1, s2 = math.sin(W1 / sigmad), math.sin(W2 / sigmad)
    c1, c2 = math.cos(W1 / sigmad), math.cos(W2 / sigmad)
    e1, e2 = math.exp(L1 / sigmad), math.exp(L2 / sigmad)
    D4 = e1 * e1 * e2 * e2
    D3 = -2 * c1 * e1 * e2 * e2 - 2 * c2 * e2 * e1 * e1
    D2 = 4 * c2 * c1 * e1 * e2 + e1 * e1 + e2 * e2
    D1 = -2 * (e2 * c2 + e1 * c1)
    SD = 1 + D1 + D2 + D3 + D4
    DD = D1 + 2 * D2 + 3 * D3 + 4 * D4
    ED = D1 + 4 * D2 + 9 * D3 + 16 * D4

    def ncoef(a1, b1, a2, b2):
        N0 = a1 + a2
        N1 = e2 * (b2 * s2 - (a2 + 2 * a1) * c2) + e1 * (b1 * s1 - (a1 + 2 * a2) * c1)
        N2 = 2 * e1 * e2 * ((a1 + a2) * c2 * c1 - b1 * c2 * s1 - b2 * c1 * s2) + a2 * e1 * e1 + a1 * e2 * e2
        N3 = e2 * e1 * e1 * (b2 * s2 - a2 * c2) + e1 * e2 * e2 * (b1 * s1 - a1 * c1)
        N = np.array([N0, N1, N2, N3])
        return N, N.sum(), N1 + 2 * N2 + 3 * N3, N1 + 4 * N2 + 9 * N3

    if order == 0:
        N, SN, _, _ = ncoef(A1[0], B1[0], A2[0], B2[0])
        alpha0 = 2 * SN / SD - N[0]
        N = N * (scale_norm / alpha0)
    elif order == 2:
        N0s, SN0, DN0, EN0 = ncoef(A1[0], B1[0], A2[0], B2[0])
        N2s, SN2, DN2, EN2 = ncoef(A1[2], B1[2], A2[2], B2[2])
        beta = -(2 * SN2 - SD * N2s[0]) / (2 * SN0 - SD * N0s[0])
        N = N2s + beta * N0s
        SN, DN, EN = SN2 + beta * SN0, DN2 + beta * DN0, EN2 + beta * EN0
        alpha2 = (EN * SD * SD - ED * SN * SD - 2 * DN * DD * SD + 2 * DD * DD * SN) / (SD * SD * SD)
        N = N * (scale_norm / alpha2)
    else:
        raise ValueError("order must be 0 or 2")
    D = np.array([D1, D2, D3, D4])
    M = np.array([N[1] - D1 * N[0], N[2] - D2 * N[0], N[3] - D3 * N[0], -D4 * N[0]])   # symmetric kernel
    SNn, SM = N.sum(), M.sum()
    BN = D * SNn / SD
    BM = D * SM / SD
    return np.concatenate([N, D, M, BN, BM]).astype(np.float64)


def _rg_pass(src: torch.Tensor, axis: int, sigma_vox: float, order: int, out: torch.Tensor | None = None, scale: float = 1.0,
             accumulate: bool = False):
    """one recursive-Gaussian axis pass (order 0 = smoothing, 2 = second derivative) of a float32 / float64 CUDA volume
    into a float32 volume"""
    Z, Y, X = src.shape
    if out is None:
        out = torch.empty((Z, Y, X), dtype=torch.float32, device=src.device)
    scratch = torch.empty((Z, Y, X), dtype=torch.float64, device=src.device)
    coef = recursive_gaussian_coefficients(sigma_vox, order)
    check(lib().rb_recursive_gaussian_axis_dev(_ptr(src), int(src.dtype == torch.float32), Z, Y, X, int(axis),
                                               coef.ctypes.data_as(C.c_void_p), _ptr(out), _ptr(scratch), C.c_double(scale),
                                               int(accumulate), _stream()), "LoG")
    return out


def log_filter_device(x: torch.Tensor, sigma_mm: float, spacing_zyx, z_pass=None):
    """sigma^2-normalised Laplacian of Gaussian of a CUDA volume (Z,Y,X) -> float32 tensor: for each direction d,
    Gaussian smoothing along the other two axes (z first) then the second derivative along d, summed over d (ITK's
    LaplacianRecursiveGaussianImageFilter, reference radiomics/imageoperations.py:824-830).
    `z_pass(src, sigma_vox, order, scale)` replaces the pass along z: a multi-GPU caller holding a z-slab transposes to
    y-slabs, runs the scan over the whole lines there and transposes back (pipeline.derived_images_slab); every other
    pass is local to the slab, so the distributed result is bit-identical to the single-GPU one."""
    src = x.to(torch.float32).contiguous() if x.dtype != torch.float64 else x.contiguous()
    sz, sy, sx = (sigma_mm / spacing_zyx[0], sigma_mm / spacing_zyx[1], sigma_mm / spacing_zyx[2])
    if z_pass is None:
        z_pass = lambda t, sv, order, scale: _rg_pass(t, 0, sv, order, scale=scale)
    # d = z: smooth y, x; derivative z
    cur = _rg_pass(_rg_pass(src, 1, sy, 0), 2, sx, 0)
    out = z_pass(cur, sz, 2, sz * sz)
    # d = y and d = x both start with the smoothing along z of the input
    gz = z_pass(src, sz, 0, 1.0)
    _rg_pass(_rg_pass(gz, 2, sx, 0), 1, sy, 2, out=out, scale=sy * sy, accumulate=True)      # + sigma^2 d2/dy2
    _rg_pass(_rg_pass(gz, 1, sy, 0), 2, sx, 2, out=out, scale=sx * sx, accumulate=True)      # + sigma^2 d2/dx2
    return out


def getLoGImage(inputImage, _inputMask, **kwargs):
    """reference generator (imageoperations.py:756-836)."""
    arr = I.as_array(inputImage)
    size = np.array(arr.shape[::-1])
    spacing = np.array(I.spacing_xyz(inputImage), dtype=float)
    if arr.ndim != 3 or np.min(size) < 4:
        logger.warning("Image too small to apply LoG filter, size: %s", size)
        return
    x = _to_device(arr)
    for sigma in kwargs.get("sigma", []):
        if sigma > 0.0:
            if np.all(size >= np.ceil(sigma / spacing) + 1):
                out = log_filter_device(x, float(sigma), tuple(spacing[::-1]))
                name = f"log-sigma-{str(sigma).replace('.', '-')}-mm-3D"
                yield I.like(inputImage, out.cpu().numpy()), name, kwargs
            else:
                logger.warning("applyLoG: sigma(%s)/spacing(%s) + 1 must be greater than the size(%s) of the inputImage",
                               sigma, spacing, size)
        else:
            logger.warning("applyLoG: sigma must be greater than 0.0: %s", sigma)


# ------------------------------------------------------------------------------------ square, square root, logarithm,
# exponential, gradient
POINTWISE_KINDS = {"square": 0, "squareroot": 1, "logarithm": 2, "exponential": 3}      # rb_pointwise_image_dev codes


def pointwise_scalar(kind, max_abs):
    """the scalar rb_pointwise_image_dev applies for M = max|x| = `max_abs`, by the reference's own NumPy expressions
    (imageoperations.py:989, :1014, :1041-1044, :1066-1067), so that it is the reference's to the bit.  Logarithm: the
    reference divides M by max|transformed image|, which is log(M + 1) whichever sign M comes from (log is monotone and
    -(x - 1) == 1 + |x| exactly for x < 0), so no second reduction is needed.  That log is taken over an array, as the
    reference takes it: NumPy may evaluate a 0-d log by another routine than a contiguous array's."""
    im_max = np.float64(max_abs)
    with np.errstate(divide="ignore", invalid="ignore"):            # an all-zero image: NaN images, as in the reference
        if kind == "square":
            return float(1 / np.sqrt(im_max))
        if kind == "squareroot":
            return float(im_max)
        if kind == "logarithm":
            return float(im_max / np.log(np.array([im_max]) + 1)[0])
        if kind == "exponential":
            return float(np.log(im_max) / im_max)
    raise ValueError(f"unknown image type {kind!r} (one of {sorted(POINTWISE_KINDS)})")


def image_max_abs(x: torch.Tensor) -> float:
    """M = max|x| over the whole CUDA tensor: one rb_minmax_dev pass without a mask, |max(-min, max)| (the abs turns the
    -0.0 of an all-zero image into 0.0, as np.abs does).  NaN voxels do not take part (the reference's np.max(np.abs(im))
    would be NaN and turn the square / logarithm / exponential images into NaN everywhere)."""
    mn, mx, _ = roi_minmax(x, None)
    return abs(max(-mn, mx))


def pointwise_image_device(x: torch.Tensor, kind: str, max_abs=None):
    """square / squareroot / logarithm / exponential image (getSquareImage ... getExponentialImage) of a CUDA tensor of
    any shape -> float64 CUDA tensor of that shape (rb_pointwise_image_dev).  `max_abs`: M = max|x| over the whole
    image; None reduces it here (a caller that makes several of these types passes one image_max_abs to all)."""
    if kind not in POINTWISE_KINDS:
        raise ValueError(f"unknown image type {kind!r} (one of {sorted(POINTWISE_KINDS)})")
    src = x.contiguous()
    if src.dtype not in _TORCH_DT:
        raise ValueError(f"unsupported pixel type {src.dtype}")
    if max_abs is None:
        max_abs = image_max_abs(src)
    out = torch.empty(src.shape, dtype=torch.float64, device=src.device)
    check(lib().rb_pointwise_image_dev(_ptr(src), _TORCH_DT[src.dtype], C.c_longlong(src.numel()), POINTWISE_KINDS[kind],
                                       C.c_double(pointwise_scalar(kind, max_abs)), _ptr(out), _stream()), kind)
    return out


def gradient_magnitude_device(x: torch.Tensor, spacing_zyx=None):
    """gradient magnitude (sitk.GradientMagnitudeImageFilter, getGradientImage) of a CUDA volume (Z,Y,X) or plane (Y,X)
    -> float64 CUDA tensor of that shape (rb_gradient_magnitude_dev).  `spacing_zyx`: one spacing per axis that the
    differences are divided by (gradientUseSpacing=True); None = unit weights.  A zero spacing raises ValueError."""
    src = x.contiguous()
    if src.dim() not in (2, 3):
        raise ValueError(f"gradient: 2-D or 3-D image expected, got {src.dim()}-D")
    if src.dtype not in _TORCH_DT:
        raise ValueError(f"unsupported pixel type {src.dtype}")
    w = [1.0] * 3
    if spacing_zyx is not None:
        sp = [float(s) for s in spacing_zyx]
        if len(sp) != src.dim():
            raise ValueError(f"gradient: {len(sp)} spacings for a {src.dim()}-D image")
        if 0.0 in sp:
            raise ValueError(f"gradient: image spacing cannot be zero, got {tuple(sp)}")
        w[3 - len(sp):] = [1.0 / s for s in sp]
    Z, Y, X = (1,) * (3 - src.dim()) + tuple(src.shape)
    out = torch.empty(src.shape, dtype=torch.float64, device=src.device)
    check(lib().rb_gradient_magnitude_dev(_ptr(src), _TORCH_DT[src.dtype], Z, Y, X, (C.c_double * 3)(*w), _ptr(out),
                                          _stream()), "gradient")
    return out


def _pointwise_image(inputImage, kind, kwargs):
    out = pointwise_image_device(_to_device(I.as_array(inputImage)), kind).cpu().numpy()
    logger.debug("Yielding %s image", kind)
    yield I.like(inputImage, out), kind, kwargs


def getSquareImage(inputImage, _inputMask, **kwargs):
    """reference generator (imageoperations.py:973-994): (c x)^2 with c = 1 / sqrt(max|x|), float64.  The sign is NOT
    kept (the reference's docstring says it is; its code, followed here, squares it away)."""
    yield from _pointwise_image(inputImage, "square", kwargs)


def getSquareRootImage(inputImage, _inputMask, **kwargs):
    """reference generator (imageoperations.py:997-1021): sqrt(x M) for x > 0, -sqrt(-x M) for x < 0, M = max|x|."""
    yield from _pointwise_image(inputImage, "squareroot", kwargs)


def getLogarithmImage(inputImage, _inputMask, **kwargs):
    """reference generator (imageoperations.py:1024-1049): log(x + 1) for x > 0, -log(1 - x) for x < 0, rescaled by
    M / log(M + 1), M = max|x|."""
    yield from _pointwise_image(inputImage, "logarithm", kwargs)


def getExponentialImage(inputImage, _inputMask, **kwargs):
    """reference generator (imageoperations.py:1052-1073): exp(c x) with c = log(M) / M, M = max|x|."""
    yield from _pointwise_image(inputImage, "exponential", kwargs)


def getGradientImage(inputImage, _inputMask, **kwargs):
    """reference generator (imageoperations.py:1076-1091): gradient magnitude, divided by the image spacing unless
    gradientUseSpacing=False; float64 (ITK's real type for every scalar input).  2-D and 3-D images."""
    arr = I.as_array(inputImage)
    if arr.ndim not in (2, 3):
        raise ValueError(f"gradient: 2-D or 3-D image expected, got {arr.ndim}-D")
    spacing = tuple(I.spacing_xyz(inputImage))[::-1] if kwargs.get("gradientUseSpacing", True) else None
    out = gradient_magnitude_device(_to_device(arr), spacing).cpu().numpy()
    yield I.like(inputImage, out), "gradient", kwargs


# ------------------------------------------------------------------------------------ normalisation, resegmentation
_MOMENTS_SCRATCH_BYTES = 40960                     # RB_MOMENTS_SCRATCH_BYTES
RESEGMENT_MODES = ("absolute", "relative", "sigma")


def _checked_source(x):
    src = x.contiguous()
    if src.dtype not in _TORCH_DT:
        raise ValueError(f"unsupported pixel type {src.dtype}")
    return src


def _roi_moments(src, roi_u8, passes):
    """rb_roi_moments_dev -> [n, n_nan, sum, max, sum of (x - mean)^2] on the host (one 40-byte copy)"""
    scratch = torch.empty(_MOMENTS_SCRATCH_BYTES, dtype=torch.uint8, device=src.device)
    res = torch.empty(5, dtype=torch.float64, device=src.device)
    check(lib().rb_roi_moments_dev(_ptr(src), _TORCH_DT[src.dtype], _ptr(roi_u8), C.c_longlong(src.numel()), passes,
                                   _ptr(scratch), _ptr(res), _stream()), "roi moments")
    return res.cpu().tolist()


def _moments_of_roi(src, roi_u8, ddof):
    n, n_nan, s, mx, ssd = _roi_moments(src, roi_u8, 2)
    n, n_nan = int(n), int(n_nan)
    mean = s / n if n else math.nan
    std = math.sqrt(ssd / (n - ddof)) if n > ddof else math.nan
    return n, n_nan, mean, std, (mx if n else math.nan)


def roi_moments_device(img_t: torch.Tensor, mask_t: torch.Tensor | None = None, label=1, ddof=0):
    """(n, n_nan, mean, std, max) of the CUDA tensor's voxels with mask_t == label (mask_t None = every voxel), reduced
    in float64 in a fixed order (rb_roi_moments_dev: the same bits on every run): mean = sum / n, std =
    sqrt(sum((x - mean)^2) / (n - ddof)), max NaN when any voxel is NaN (np.max).  An empty ROI gives NaN statistics."""
    roi = None if mask_t is None else (mask_t == label).to(torch.uint8).contiguous()
    return _moments_of_roi(_checked_source(img_t), roi, ddof)


def normalize_image_device(x: torch.Tensor, scale=1, outliers=None, stats=None):
    """normalizeImage on a CUDA tensor -> float64 CUDA tensor: ((x - mean) * (1 / std)), clamped to [-outliers,
    outliers] unless `outliers` is None, times `scale` (rb_normalize_dev).  mean and std (N - 1) are those of the WHOLE
    image, as sitk.Normalize takes them; `stats` = (mean, std) supplies them, for a caller that holds only a crop."""
    src = _checked_source(x)
    if stats is None:
        _, _, mean, std, _ = roi_moments_device(src, ddof=1)
    else:
        mean, std = (float(v) for v in stats)
    out = torch.empty(src.shape, dtype=torch.float64, device=src.device)
    check(lib().rb_normalize_dev(_ptr(src), _TORCH_DT[src.dtype], C.c_longlong(src.numel()), C.c_double(mean),
                                 C.c_double(std), int(outliers is not None),
                                 C.c_double(float(outliers) if outliers is not None else 0.0), C.c_double(float(scale)),
                                 _ptr(out), _stream()), "normalize")
    return out


def _comparison_value(np_type, t):
    """the float64 that compares with an np_type voxel (exactly converted to float64) as NumPy compares the voxel with
    `t`: in np.result_type(np_type, t), where a Python scalar is weak (NEP 50).  A float32 image and a Python float
    compare in float32, so the threshold is rounded to float32 first.  A Python int against an integer image compares
    exactly, even out of the dtype's range."""
    if isinstance(t, int) and np.issubdtype(np_type, np.integer):
        return float(t)
    return float(np.result_type(np_type, t).type(t))


def resegment_thresholds(np_type, resegmentRange, resegmentMode, max_gl=None, mean_gl=None, sd_gl=None):
    """the reference's thresholds (imageoperations.py:695-711) from the ROI's np.max (`max_gl`, an np_type scalar) or
    np.mean / np.std (`mean_gl` / `sd_gl`: float32 scalars for a float32 image, float64 otherwise), with the reference's
    own expressions so that they have its dtype and value -> (thresholds, the float64 values rb_resegment_dev compares
    with)."""
    if resegmentMode == "absolute":
        thresholds = sorted(resegmentRange)
    elif resegmentMode == "relative":
        thresholds = [max_gl * th for th in sorted(resegmentRange)]
    elif resegmentMode == "sigma":
        thresholds = [mean_gl + sd_gl * th for th in sorted(resegmentRange)]
    else:
        raise ValueError(f"Resegment mode {resegmentMode} not recognized.")
    return thresholds, [_comparison_value(np_type, t) for t in thresholds]


def _stat_type(np_type):
    """the type np.mean / np.std of an np_type array return"""
    return np.float32 if np_type == np.float32 else np.float64


def resegment_mask_device(img_t: torch.Tensor, mask_t: torch.Tensor, resegmentRange, resegmentMode="absolute", label=1):
    """resegmentMask on CUDA tensors -> (uint8 CUDA mask: 1 where mask_t == label and the voxel lies within the
    thresholds, kept voxel count, thresholds as the reference computes them).  The ROI statistics come from one
    rb_roi_moments_dev (relative mode: one pass for the maximum; sigma mode: two passes) and are rounded to the type
    NumPy's reductions return; the thresholding is rb_resegment_dev.  Raises the reference's ValueErrors, including
    when at most one voxel is kept."""
    if resegmentRange is None:
        raise ValueError("resegmentRange is None.")
    if len(resegmentRange) == 0 or len(resegmentRange) > 2:
        raise ValueError(f"Length {len(resegmentRange)} is not allowed for resegmentRange")
    logger.debug(f"Resegmenting mask (range {resegmentRange}, mode {resegmentMode})")
    src = _checked_source(img_t)
    np_type = _NP_OF_TORCH[src.dtype]
    roi = (mask_t == label).to(torch.uint8).contiguous()
    if roi.shape != src.shape:
        raise ValueError(f"mask shape {tuple(roi.shape)} differs from image shape {tuple(src.shape)}")
    stats = {}
    if resegmentMode == "absolute":
        logger.debug("Resegmenting in absolute mode")
    elif resegmentMode == "relative":
        n, _, _, mx, _ = _roi_moments(src, roi, 1)
        if n == 0:                                              # np.max of an empty array
            raise ValueError("zero-size array to reduction operation maximum which has no identity")
        stats["max_gl"] = np_type(mx)
        logger.debug(f"Resegmenting in relative mode, max {stats['max_gl']}")
    elif resegmentMode == "sigma":
        _, _, mean, std, _ = _moments_of_roi(src, roi, 0)
        st = _stat_type(np_type)
        stats["mean_gl"], stats["sd_gl"] = st(mean), st(std)
        logger.debug(f"Resegmenting in sigma mode, mean {stats['mean_gl']}, std {stats['sd_gl']}")
    thresholds, cmp = resegment_thresholds(np_type, resegmentRange, resegmentMode, **stats)
    logger.debug(f"Applying lower threshold ({thresholds[0]})")
    if len(thresholds) == 2:
        logger.debug(f"Applying upper threshold ({thresholds[1]})")
    out = torch.empty(src.shape, dtype=torch.uint8, device=src.device)
    counts = torch.empty(2, dtype=torch.int64, device=src.device)
    check(lib().rb_resegment_dev(_ptr(src), _TORCH_DT[src.dtype], _ptr(roi), C.c_longlong(src.numel()),
                                 C.c_double(cmp[0]), C.c_double(cmp[-1]), len(cmp), _ptr(out), _ptr(counts), _stream()),
          "resegment")
    oldSize, roiSize = counts.cpu().tolist()
    if roiSize <= 1:
        raise ValueError(f"Resegmentation excluded too many voxels with label {label} "
                         f"(retained {roiSize} voxel(s))! Cannot extract features")
    logger.debug(f"Resegmentation complete, new size: {roiSize} voxels (excluded {oldSize - roiSize} voxels)")
    return out, roiSize, thresholds


def normalizeImage(image, **kwargs):
    """reference function (imageoperations.py:615-654): (x - mean) / std over the WHOLE image (std with N - 1), outliers
    beyond +-removeOutliers clamped, times normalizeScale; float64 image of the input's geometry."""
    scale = kwargs.get("normalizeScale", 1)
    outliers = kwargs.get("removeOutliers")
    logger.debug(f"Normalizing image with scale {scale}")
    if outliers is not None:
        logger.debug(f"Removing outliers > {outliers} standard deviations")
    out = normalize_image_device(_to_device(I.as_array(image)), scale, outliers).cpu().numpy()
    return I.like(image, out)


def resegmentMask(imageNode, maskNode, **kwargs):
    """reference function (imageoperations.py:657-742): the mask == label voxels within resegmentRange (mode absolute,
    relative to the ROI maximum, or sigma around the ROI mean) -> int64 mask holding `label`, of the mask's geometry."""
    resegmentRange = kwargs["resegmentRange"]
    resegmentMode = kwargs.get("resegmentMode", "absolute")
    label = kwargs.get("label", 1)
    out, _, _ = resegment_mask_device(_to_device(I.as_array(imageNode)), _to_device(I.as_array(maskNode)), resegmentRange,
                                      resegmentMode, label)
    newMask_arr = out.cpu().numpy().astype(np.int64) * label
    return I.like(maskNode, newMask_arr)


# ------------------------------------------------------------------------------------ LBP 3-D
_ICOSAHEDRON_T = (1.0 + 5.0 ** 0.5) / 2.0
_ICOSAHEDRON_V = [[-1, _ICOSAHEDRON_T, 0], [1, _ICOSAHEDRON_T, 0], [-1, -_ICOSAHEDRON_T, 0], [1, -_ICOSAHEDRON_T, 0],
                  [0, -1, _ICOSAHEDRON_T], [0, 1, _ICOSAHEDRON_T], [0, -1, -_ICOSAHEDRON_T], [0, 1, -_ICOSAHEDRON_T],
                  [_ICOSAHEDRON_T, 0, -1], [_ICOSAHEDRON_T, 0, 1], [-_ICOSAHEDRON_T, 0, -1], [-_ICOSAHEDRON_T, 0, 1]]
_ICOSAHEDRON_F = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6],
                  [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10],
                  [8, 6, 7], [9, 8, 1]]


def _icosphere(subdivision=1, radius=1.0):
    """vertices (Nv, 3) of the icosphere getLBP3DImage samples on (trimesh.creation.icosphere's construction, restated):
    the 12 normalised icosahedron vertices, then per subdivision the midpoints of every edge, all projected back onto the
    unit sphere; finally scaled to `radius`.  12 / 42 / 162 / 642 vertices for subdivision 0 / 1 / 2 / 3.  Only the vertex
    set matters to the filter (every reduction runs over the vertices)."""
    v = np.array(_ICOSAHEDRON_V, dtype=np.float64)
    v /= np.linalg.norm(v, axis=1)[:, None]
    faces = np.array(_ICOSAHEDRON_F, dtype=np.int64)
    for _ in range(int(subdivision)):
        edges = np.sort(np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]), axis=1)
        uniq, inv = np.unique(edges, axis=0, return_inverse=True)
        mid = (v[uniq[:, 0]] + v[uniq[:, 1]]) / 2.0
        inv = inv.reshape(3, -1) + len(v)                  # midpoint index of edge (01, 12, 20) of every face
        v = np.concatenate([v, mid])
        v /= np.linalg.norm(v, axis=1)[:, None]
        a, b, c = faces.T
        ab, bc, ca = inv
        faces = np.concatenate([np.stack([a, ab, ca], 1), np.stack([ab, b, bc], 1), np.stack([ca, bc, c], 1),
                                np.stack([ab, bc, ca], 1)])
    return v * float(radius)


def _lbp3d_harmonics(vertices, levels, radius=None):
    """complex (Nv, levels**2) table Y[v][k], k running over n = 0..levels-1, m = -n..n: the reference's
    sph_harm(m, n, theta, phi) (imageoperations.py:1238-1248) with theta = arccos(v_2 / R) and phi = arctan2(v_1, v_0) in
    SciPy's old argument order, i.e. phi is the POLAR angle and theta the azimuth.  Orthonormal harmonics with the
    Condon-Shortley phase, Y_n^-m = (-1)^m conj(Y_n^m)."""
    v = np.asarray(vertices, dtype=np.float64)
    if radius is None:
        radius = float(np.linalg.norm(v[0]))
    azimuth = np.arccos(np.true_divide(v[:, 2], radius))
    polar = np.arctan2(v[:, 1], v[:, 0])
    x, s = np.cos(polar), np.abs(np.sin(polar))
    P = {}                                            # associated Legendre P_n^m(x), m >= 0
    for m in range(levels):
        pmm = np.ones_like(x)
        for i in range(1, m + 1):
            pmm = -pmm * (2 * i - 1) * s
        P[m, m] = pmm
        if m + 1 < levels:
            P[m + 1, m] = x * (2 * m + 1) * pmm
        for n in range(m + 2, levels):
            P[n, m] = ((2 * n - 1) * x * P[n - 1, m] - (n + m - 1) * P[n - 2, m]) / (n - m)
    cols = []
    for n in range(levels):
        pos = {}
        for m in range(n + 1):
            norm = math.sqrt((2 * n + 1) / (4 * math.pi) * math.factorial(n - m) / math.factorial(n + m))
            pos[m] = norm * P[n, m] * np.exp(1j * m * azimuth)
        for m in range(-n, n + 1):
            cols.append(pos[m] if m >= 0 else (-1) ** m * np.conj(pos[-m]))
    return np.stack(cols, axis=1)


def _lbp3d_tables(levels, radius, subdivision):
    """host tables of rb_lbp3d_dev: vertices (Nv, 3) and the m >= 0 harmonics (Nv, levels (levels + 1) / 2, [re, im]).
    The kernel covers subdivision 0..2 (at most 162 vertices) and 1..4 levels; there is no other implementation."""
    if not (0 <= int(subdivision) <= 2 and 1 <= int(levels) <= 4):
        raise ValueError(f"LBP 3D: lbp3DIcosphereSubdivision {subdivision} / lbp3DLevels {levels} outside the CUDA "
                         "kernel's range (subdivision 0..2, levels 1..4)")
    levels = int(levels)
    verts = np.ascontiguousarray(_icosphere(int(subdivision), radius), dtype=np.float64)
    Y = _lbp3d_harmonics(verts, levels, float(radius))
    keep = [n * n + n + m for n in range(levels) for m in range(n + 1)]              # the m >= 0 columns
    harm = np.ascontiguousarray(np.stack([Y[:, keep].real, Y[:, keep].imag], axis=-1), dtype=np.float64)
    return verts, harm


def lbp3d_device(img_t: torch.Tensor, roi_t: torch.Tensor, levels=2, radius=1.0, subdivision=1, dtype=None):
    """3-D LBP of a CUDA volume (Z,Y,X): float64 CUDA tensor [levels + 1, Z, Y, X] holding the level maps m1..m<levels>
    and the kurtosis map, 0 outside the ROI (roi_t != 0).  `dtype` is the image's original NumPy dtype, which the sphere
    samples are rounded and clamped to (default: img_t's; a uint16 image reaches the device as int32)."""
    verts, harm = _lbp3d_tables(levels, radius, subdivision)
    levels = int(levels)
    src = img_t.contiguous()
    if src.dtype not in _TORCH_DT:
        raise ValueError(f"unsupported pixel type {src.dtype}")
    dtype = np.dtype(dtype) if dtype is not None else np.dtype(_NP_OF_TORCH[src.dtype])
    if dtype not in _DT:
        raise ValueError(f"unsupported pixel type {dtype}")
    roi = (roi_t != 0).to(torch.uint8).contiguous()
    if src.dim() != 3 or tuple(roi.shape) != tuple(src.shape):
        raise ValueError("lbp3d_device needs a 3-D image and a ROI of the same shape")
    Z, Yn, X = src.shape
    scratch = torch.empty((Z, Yn, X), dtype=torch.float64, device=src.device)
    out = torch.empty((levels + 1, Z, Yn, X), dtype=torch.float64, device=src.device)
    check(lib().rb_lbp3d_dev(_ptr(src), _TORCH_DT[src.dtype], _DT[dtype], _ptr(roi), Z, Yn, X,
                             verts.ctypes.data_as(C.c_void_p), int(len(verts)), harm.ctypes.data_as(C.c_void_p), levels,
                             _ptr(scratch), _ptr(out), _stream()), "lbp3d")
    return out


def getLBP3DImage(inputImage, inputMask, **kwargs):
    """reference generator (imageoperations.py:1169-1314): yields the level maps 'lbp-3D-m1' .. 'lbp-3D-m<lbp3DLevels>'
    then the spherical kurtosis 'lbp-3D-k', float64 images.  Settings lbp3DLevels (2), lbp3DIcosphereRadius (1, voxels),
    lbp3DIcosphereSubdivision (1) and label (1).  Deviation: voxels outside the ROI are 0 (the reference leaves them
    uninitialised)."""
    arr = I.as_array(inputImage)
    Nd = arr.ndim
    if Nd != 3:
        logger.warning(f"LBP 3D only available for 3 dimensional images, found {Nd} dimensions")
        return
    if kwargs.get("force2D", False):
        logger.warning("Calculating Local Binary Pattern in 3D, but extracting features in 2D. Use with caution!")
    label = kwargs.get("label", 1)
    levels = int(kwargs.get("lbp3DLevels", 2))
    radius = kwargs.get("lbp3DIcosphereRadius", 1)
    subdivision = int(kwargs.get("lbp3DIcosphereSubdivision", 1))
    _lbp3d_tables(levels, radius, subdivision)                  # range check before anything reaches the device
    roi = np.ascontiguousarray(I.as_array(inputMask) == label).view(np.uint8)
    out = lbp3d_device(_to_device(arr), _to_device(roi), levels, radius, subdivision, arr.dtype).cpu().numpy()
    for l_idx in range(levels):
        yield I.like(inputImage, out[l_idx]), f"lbp-3D-m{l_idx + 1}", kwargs
    yield I.like(inputImage, out[levels]), "lbp-3D-k", kwargs
