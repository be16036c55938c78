"""CUDA feature-class plugins: the same contract as the reference's ``Radiomics<Class>`` classes
(reference radiomics/base.py:60-273 and docs/developers.rst:16-64) -- constructor
``(inputImage, inputMask, **settings)``, ``enableFeatureByName`` / ``enableAllFeatures`` /
``disableAllFeatures``, ``getFeatureNames``, ``execute()`` returning ``{feature: float}``
(segment-based) or ``{feature: image}`` (voxel-based), ``_initCalculation`` exposing
``P_<class>`` -- with the hot path on the GPU:

  * gray-level discretisation: rb_minmax_dev + rb_digitize_dev (imageoperations.binImage)
  * segment-based: the matrix comes from the CUDA cMatrices drop-in (pyradiomics_b200.cmatrices);
    the O(Ng^2) scalar formulas stay on the host (_matrix_features.py), as in the reference
  * voxel-based: ONE fused CUDA kernel per class writes all feature maps (pyradiomics_b200.voxel);
    no per-voxel matrix is ever materialised and ``voxelBatch`` is not needed.

``install()`` registers them in ``radiomics.getFeatureClasses()`` when pyradiomics is importable.
"""
from __future__ import annotations

import collections
import inspect
import logging

import numpy as np
import torch

from . import _lib, _matrix_features as MF, cmatrices, image as I, imageoperations, voxel


def _weights(angles, spacing_zyx, norm, kind):
    """per-angle weights of weightingNorm (reference glcm.py:160-181 exp(-d^2), glrlm.py:130-150 d)."""
    if norm is None:
        return None
    a = np.abs(np.asarray(angles, float)) * np.asarray(spacing_zyx, float)[-angles.shape[1]:]
    if norm == "infinity":
        d = a.max(1)
    elif norm == "euclidean":
        d = np.sqrt((a ** 2).sum(1))
    elif norm == "manhattan":
        d = a.sum(1)
    else:
        if norm != "no_weighting":
            logging.getLogger("radiomics").warning('weigthing norm "%s" is unknown, W is set to 1', norm)
        return np.ones(len(angles))
    return np.exp(-d ** 2) if kind == "glcm" else d


# ---- progress reporting hook (reference radiomics/__init__.py:252-282, base.py:217,237) ------------------------
class _DummyProgressReporter:
    """accepts what the reference's voxel loop passes (iterable / total= / desc=) and does nothing"""

    def __init__(self, iterable=None, desc="", total=None):
        self.desc, self.iterable, self.total = desc, iterable, total

    def __iter__(self):
        return iter(self.iterable)

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc_value, tb):
        pass

    def update(self, n=1):
        pass


progressReporter = None


def setProgressReporter(reporter):
    """install a tqdm-like class for the voxel-based loops (the reference's ``radiomics.progressReporter``)"""
    global progressReporter
    progressReporter = reporter


def getProgressReporter(*args, **kwargs):
    """reference radiomics/__init__.py:275-282: the configured reporter when the radiomics logger is at INFO or
    below, else a dummy.  A reporter set on an already-imported ``radiomics`` module is honoured too."""
    import sys
    rep = progressReporter
    rad = sys.modules.get("radiomics")
    if rep is None and rad is not None:
        rep = getattr(rad, "progressReporter", None)
    if rep is not None and logging.getLogger("radiomics").getEffectiveLevel() <= logging.INFO:
        return rep(*args, **kwargs)
    return _DummyProgressReporter(*args, **kwargs)


# ---- per-image device state shared by the feature classes (SURVEY.md section 8f rank 1) -----------------------
_FP_POOL = None


def _fingerprint(a):
    """content key of a host array (shape, dtype, wrapped 64-bit sums over the WHOLE buffer, tail bytes): the same image
    handed to the five classes one after the other (featureextractor.py:586-602) hits the cache; an edited image does
    not.  Large arrays are summed by a few threads (NumPy releases the GIL): a 512^3 int16 image costs a few ms."""
    global _FP_POOL
    a = np.ascontiguousarray(a)
    b = a.reshape(-1).view(np.uint8)
    n8 = b.size // 8 * 8
    w = b[:n8].view(np.uint64)
    if w.size > (1 << 22):
        import concurrent.futures as cf
        if _FP_POOL is None:
            _FP_POOL = cf.ThreadPoolExecutor(max_workers=8)
        parts = np.array_split(w, 16)
        sums = list(_FP_POOL.map(lambda p: (int(p.sum(dtype=np.uint64)), int(p[::61].sum(dtype=np.uint64))), parts))
        s = sum(x[0] for x in sums) & 0xFFFFFFFFFFFFFFFF
        s2 = sum((k + 1) * x[1] for k, x in enumerate(sums)) & 0xFFFFFFFFFFFFFFFF
    else:
        s = int(w.sum(dtype=np.uint64)) if n8 else 0
        s2 = int(w[::61].sum(dtype=np.uint64)) if n8 else 0
    return (a.shape, a.dtype.str, s, s2, bytes(b[n8:]))


class DeviceImage:
    """One (image, ROI mask, binning) discretised ONCE on the GPU (voxel.discretize; reference: binImage in every class
    constructor, base.py:119-125, i.e. 5x per image)."""

    def __init__(self, imageArray, maskRaw, label, masked, settings):
        img_t = imageoperations._to_device(imageArray)
        # the ROI mask is formed on the device: label compare of the raw mask (or all ones for an unmasked kernel)
        raw_t = imageoperations._to_device(maskRaw)
        msk_t = (raw_t == label).to(torch.uint8) if masked else torch.ones(raw_t.shape, dtype=torch.uint8, device=raw_t.device)
        lev_t, self.edges, self.levels, self.grayLevels, self.Ng = voxel.discretize(img_t, msk_t, **settings)
        self.mask_dev = msk_t
        self._lev32 = lev_t                     # kept until the host copy has been asked for (or never)
        self._binned_host = None
        self._alive = {}
        self._segment = {}
        self._extent = None

    def binned_host(self):
        """the reference's ``self.imageArray`` after binning: int64 levels, 0 outside the ROI (lazy: voxel mode never needs it)"""
        if self._binned_host is None:
            self._binned_host = self._lev32.cpu().numpy().astype(np.int64)
            self._lev32 = None
        return self._binned_host

    def roi_extent(self):
        """size of the ROI's bounding box per axis (voxel.roi_extent of the device mask; computed once)"""
        if self._extent is None:
            self._extent = tuple(voxel.roi_extent(self.mask_dev))
        return self._extent

    def levels3d(self):
        return self.levels if self.levels.ndim == 3 else self.levels[None]

    def segment_texture(self, distances, alpha, force2D, force2Ddimension):
        """GLCM + GLDM + NGTDM of the ROI from ONE pass over the device-resident levels (rb_segment_texture_dev); the three
        feature classes of one image share the result"""
        key = (tuple(int(d) for d in distances), int(alpha), bool(force2D), int(force2Ddimension))
        if key not in self._segment:
            self._segment[key] = cmatrices.segment_texture_device(self.levels, list(key[0]), max(self.Ng, 1), key[1], key[2], key[3])
        return self._segment[key]

    def glcm_alive(self, settings, centers):
        key = (bytes(settings), None if centers is None else centers.data_ptr())
        if key not in self._alive:
            self._alive[key] = voxel.glcm_alive_angles(self.levels3d(), settings, centers)
        return self._alive[key]


_DEVICE_IMAGES = collections.OrderedDict()
_DEVICE_IMAGES_MAX = 2


def device_image(imageArray, maskRaw, label, masked, settings):
    """the device-resident discretised image of (image, mask, label, binning): built on first sight, shared afterwards.
    The cache key is the CONTENT of image and mask (_fingerprint: a hash over the whole buffers) unless the caller passes
    ``b200_image_key=<hashable>`` -- its promise that image and mask are the ones it used with that key before (a
    pyradiomics extraction already has such a key: the sha1 of the image in its diagnostics, generalinfo.py)."""
    ident = settings.get("b200_image_key")
    content = ("key", ident, imageArray.shape, maskRaw.shape) if ident is not None else (_fingerprint(imageArray), _fingerprint(maskRaw))
    key = (content, label, bool(masked), repr(settings.get("binWidth", 25)), repr(settings.get("binCount")), torch.cuda.current_device())
    st = _DEVICE_IMAGES.get(key)
    if st is None:
        st = DeviceImage(imageArray, maskRaw, label, masked, settings)
        _DEVICE_IMAGES[key] = st
        while len(_DEVICE_IMAGES) > _DEVICE_IMAGES_MAX:
            _DEVICE_IMAGES.popitem(last=False)
    else:
        _DEVICE_IMAGES.move_to_end(key)
    return st


def clear_device_cache(release_queues=False):
    """drop the cached device-resident discretised images (and, on request, the library's GLCM eigen-task queues)"""
    _DEVICE_IMAGES.clear()
    if release_queues:
        _lib.check(_lib.lib().rb_release_device_caches(), "release_device_caches")


class RadiomicsFeaturesBase:
    """Plugin base; named like the reference's so ``radiomics.getFeatureClasses()``'s MRO-by-name
    check (reference radiomics/__init__.py:95-99) accepts subclasses."""

    CLASS = None          # "glcm", ...
    MATRIX_ATTR = None    # "P_glcm", ...

    def __init__(self, inputImage, inputMask, **kwargs):
        self.logger = logging.getLogger("radiomics." + (self.CLASS or "base"))    # reference base.py:61: the class's module
        self.logger.debug("Initializing feature class")
        if inputImage is None or inputMask is None:
            raise ValueError("Missing input image or mask")
        self._configure(kwargs)
        self.inputImage = inputImage
        self.inputMask = inputMask
        self._rawImageArray = I.as_array(inputImage)
        self._imageArray = None
        self._device = None
        self._maskRaw = I.as_array(inputMask)
        self._labelMask = None                         # lazy: the label compare of a 512^3 mask is 0.1 s of host time per class
        self._maskArray = None
        self.masked = kwargs.get("maskedKernel", True) if self.voxelBased else True
        self._labelledVoxelCoordinates = None          # lazy: 3 x Nvox int64 (3.2 GB and seconds of np.where at 512^3)
        self._initBinning()

    def _configure(self, kwargs):
        """the state that comes from the settings alone (a class with settings of its own extends this)"""
        self.progressReporter = getProgressReporter
        self.settings = kwargs
        self.label = kwargs.get("label", 1)
        self.voxelBased = kwargs.get("voxelBased", False)
        self.coefficients = {}
        self.enabledFeatures = {}
        self.featureValues = {}
        self.featureNames = self.getFeatureNames()
        self._spacing = None
        setattr(self, self.MATRIX_ATTR, None)

    # why from_device cannot build this class (None: it can)
    FROM_DEVICE_REFUSED = None

    @classmethod
    def from_device(cls, device, spacing_zyx, **kwargs):
        """a segment-mode instance over `device`, a DeviceImage already on the GPU (built from CUDA tensors, e.g.
        ``DeviceImage(img_t, roi_t, 1, True, settings)``): no host image or mask exists, `spacing_zyx` stands for the
        image's spacing.  ``execute()`` then runs the same matrix post-processing, formulas and per-feature isolation
        as an instance built from host images of the image cropped to the ROI's bounding box (the reference's flow): the
        matrices see only ROI voxels, and GLRLM's run-length capacity is the box's largest extent.  The texture classes
        support it; the others raise NotImplementedError."""
        if cls.FROM_DEVICE_REFUSED:
            raise NotImplementedError(f"{cls.__name__}.from_device: {cls.FROM_DEVICE_REFUSED}")
        self = cls.__new__(cls)
        self.logger = logging.getLogger("radiomics." + (cls.CLASS or "base"))
        self._configure(dict(kwargs, voxelBased=False))
        self.masked = True
        self.inputImage = self.inputMask = self._rawImageArray = self._maskRaw = None
        self._imageArray = self._labelMask = self._maskArray = self._labelledVoxelCoordinates = None
        self._spacing = tuple(float(s) for s in spacing_zyx)
        self._device = device
        if device is not None:
            self.coefficients["grayLevels"] = device.grayLevels
            self.coefficients["Ng"] = device.Ng
        return self

    # ---- discretisation on the GPU, shared by the classes that see the same image (reference base.py:119-125)
    def _initBinning(self):
        self._device = device_image(self._rawImageArray, self._maskRaw, self.label, self.masked, self.settings)
        self.coefficients["grayLevels"] = self._device.grayLevels
        self.coefficients["Ng"] = self._device.Ng

    @property
    def _centerMask(self):
        """boolean ROI mask (the voxels that get a value in voxel-based mode)"""
        if self._labelMask is None:
            self._labelMask = self._maskRaw == self.label
        return self._labelMask

    @property
    def maskArray(self):
        """the reference's ``self.maskArray``: the ROI, or everything for an unmasked voxel kernel (base.py:100-104)"""
        if self._maskArray is None:
            self._maskArray = self._centerMask if self.masked else np.ones(self._rawImageArray.shape, dtype=bool)
        return self._maskArray

    @maskArray.setter
    def maskArray(self, value):
        self._maskArray = value

    @property
    def labelledVoxelCoordinates(self):
        """the reference's attribute (base.py:98): coordinates of the ROI voxels; built on first use -- the fused kernels
        take the ROI as a mask volume, nothing on the hot path needs the list"""
        if getattr(self, "_labelledVoxelCoordinates", None) is None:
            self._labelledVoxelCoordinates = np.array(np.where(self._centerMask if self.voxelBased else self.maskArray))
        return self._labelledVoxelCoordinates

    @property
    def imageArray(self):
        """the discretised image like the reference's ``self.imageArray`` (host int64; downloaded on first use)"""
        if self._imageArray is None and self._device is not None:
            self._imageArray = self._device.binned_host()
        return self._imageArray

    @imageArray.setter
    def imageArray(self, value):
        self._imageArray = value

    # ---- enabling (reference base.py:127-179)
    def enableFeatureByName(self, featureName, enable=True):
        if featureName not in self.featureNames:
            raise LookupError("Feature not found: " + featureName)
        if self.featureNames[featureName]:
            self.logger.warning("Feature %s is deprecated, use with caution!", featureName)
        self.enabledFeatures[featureName] = enable

    def enableAllFeatures(self):
        for featureName, is_deprecated in self.featureNames.items():
            if not is_deprecated:
                self.enableFeatureByName(featureName, True)

    def disableAllFeatures(self):
        self.enabledFeatures = {}
        self.featureValues = {}

    @classmethod
    def getFeatureNames(cls):
        return {a[0][3:-12]: getattr(a[1], "_is_deprecated", False) for a in inspect.getmembers(cls)
                if a[0].startswith("get") and a[0].endswith("FeatureValue")}

    # ---- execution
    def execute(self):
        if len(self.enabledFeatures) == 0:
            self.enableAllFeatures()
        if self.voxelBased:
            self._calculateVoxels()
        else:
            self._calculateSegment()
        return self.featureValues

    def _spacing_zyx(self):
        return self._spacing if self._spacing is not None else tuple(I.spacing_xyz(self.inputImage))[::-1]

    def _image_shape(self):
        """the shape of the image the matrices are built from: a from_device instance stands for the image cropped to
        the ROI's bounding box"""
        return tuple(self._rawImageArray.shape) if self._rawImageArray is not None else self._device.roi_extent()

    def _voxel_settings(self):
        kw = dict(self.settings)
        nd = self._rawImageArray.ndim
        if nd == 2 and kw.get("force2D"):
            kw["force2Ddimension"] = kw.get("force2Ddimension", 0) + 1
        sp = self._spacing_zyx()
        kw["spacing_zyx"] = (1.0,) * (3 - nd) + tuple(sp)
        return _lib.make_settings(self.coefficients["Ng"], len(self.coefficients["grayLevels"]), **kw)

    def _centers_dev(self):
        if self.masked:
            return None
        c = self._centerMask if self._centerMask.ndim == 3 else self._centerMask[None]
        return imageoperations._to_device(c)

    def _map_dtype(self):
        dt = str(self.settings.get("b200_map_dtype", "float64"))
        if dt not in ("float64", "float32"):
            raise ValueError("b200_map_dtype must be 'float64' (the reference's map type) or 'float32'")
        return torch.float64 if dt == "float64" else torch.float32

    def _zchunk(self, nz):
        """planes per chunk of the compute / copy pipeline: ``b200_zchunk``, else a sixteenth of the planes within [8, 64] --
        a rank that holds 64 planes of an image shared by eight GPUs still overlaps its kernels with its PCIe copies"""
        zc = int(self.settings.get("b200_zchunk", 0) or 0)
        return zc if zc > 0 else max(8, min(64, -(-nz // 16)))

    def _voxel_launch(self, lev):
        """(launch(za, zb, buf) of voxel.maps_to_host, device status word or None) of the class's voxel kernel on the
        discretised volume `lev`: here the fused texture kernel (voxel.texture_launch)"""
        settings = self._voxel_settings()
        centers = self._centers_dev()
        alive = self._device.glcm_alive(settings, centers) if self.CLASS == "glcm" else None
        status = torch.zeros(1, dtype=torch.int32, device=lev.device)
        return voxel.texture_launch(self.CLASS, lev, settings, centers=centers, alive=alive, status=status), status

    def _calculateVoxels(self):
        """The class's voxel kernel in z-chunks; the ENABLED maps stream to page-locked host memory chunk by chunk while
        the next chunk computes (voxel.maps_to_host) -- replaces the voxelBatch loop and the per-voxel assignment of
        base.py:200-245.  `voxelBatch` is accepted and ignored."""
        lev = self._device.levels3d()
        names = _lib.feature_names(self.CLASS)
        idx = [k for k, n in enumerate(names) if self.enabledFeatures.get(n)]
        for n, enabled in self.enabledFeatures.items():
            if enabled and n not in names:
                self.logger.debug("Feature %s is deprecated / not computed in voxel-based mode", n)
        if not idx:
            return
        launch, status = self._voxel_launch(lev)
        # b200_zrange=(z0, z1): compute and return only these planes (a multi-GPU caller hands every rank the whole image --
        # so that bin edges, gray levels and the GLCM angle set are those of the whole ROI -- and takes one slab per rank)
        z0, z1 = self.settings.get("b200_zrange") or (0, int(lev.shape[0]))
        with self.progressReporter(total=int(z1 - z0), desc="planes") as pbar:
            host = voxel.maps_to_host(launch, len(names), lev.shape, lev.device, idx, z0=int(z0), z1=int(z1),
                                      zchunk=self._zchunk(int(z1 - z0)), out_dtype=self._map_dtype(), progress=pbar.update,
                                      map_dtypes=voxel.MAP_DTYPES if self.CLASS in _lib.CLASSES else (torch.float64,))
        st = 0 if status is None else int(status.item())
        if st & 2:
            raise _lib.B200Error("weighted GLCM entry list overflow")
        if st & 1:
            self.logger.warning("MCC eigen-problem too large for the in-kernel solver (more than 32 gray levels in one "
                                "matrix of a voxel's window): NaN stored as the MCC of those voxels")
        arrs = host.numpy()                      # views of ONE page-locked block the returned images keep alive
        for pos, k in enumerate(idx):
            arr = arrs[pos] if self._rawImageArray.ndim == 3 else arrs[pos][0]
            self.featureValues[names[k]] = I.like(self.inputImage, arr)

    def _calculateSegment(self):
        self._initCalculation()
        segment_feature_values(self._segment_features(), self.enabledFeatures, self.featureNames, self.logger,
                               self.featureValues)

    def _initCalculation(self, voxelCoordinates=None):
        setattr(self, self.MATRIX_ATTR, self._calculateMatrix(voxelCoordinates))

    def _matrix_args(self):
        return self.settings.get("force2D", False), self.settings.get("force2Ddimension", 0)

    def _batch_args(self, voxelCoordinates):
        return [self.settings.get("kernelRadius", 1), voxelCoordinates] if voxelCoordinates is not None else []

    def _single_roi(self, P):
        """the matrix of the one ROI out of the [batch, ...] a matrix builder returns"""
        if P.shape[0] != 1:
            raise NotImplementedError(f"{self.MATRIX_ATTR} of a voxel batch: the voxel-based path is fused (no per-voxel "
                                      f"matrices); use cmatrices.calculate_{self.CLASS} for dense per-voxel matrices")
        return P[0]

    def _value(self, name):
        """single feature (the reference's get<Name>FeatureValue entry points)."""
        if getattr(self, self.MATRIX_ATTR) is None:
            self._initCalculation()
        return np.float64(self._segment_features()[name])


def segment_feature_values(vals, enabledFeatures, featureNames, logger, out=None):
    """the enabled features of a segment-mode class out of `vals` (its formulas' {name: value}) into `out` (a new dict
    when None), in enabling order: deprecated ones without a value are skipped, a value that does not convert to a
    float64 becomes NaN with a logged error (per-feature isolation, reference base.py:258-273)"""
    out = {} if out is None else out
    for feature, enabled in enabledFeatures.items():
        if not enabled:
            continue
        if featureNames.get(feature) and feature not in vals:
            logger.debug("Feature %s is deprecated", feature)     # texture: the reference raises DeprecationWarning
            continue
        try:
            out[feature] = np.squeeze(np.float64(vals[feature]))
        except Exception:                                  # per-feature isolation (base.py:271-273)
            logger.error("FAILED: %s", feature, exc_info=True)
            out[feature] = np.nan
    return out


def _add_feature_getters(cls, names, deprecated=(), computable_deprecated=()):
    """get<Name>FeatureValue for every feature: `names` compute; `deprecated` [(name, why)] raise DeprecationWarning like
    the reference's; `computable_deprecated` [(name, why)] compute on request, but enableAllFeatures skips them"""
    def add(n, fn, doc, is_deprecated=False):
        fn.__name__, fn.__qualname__, fn.__doc__ = f"get{n}FeatureValue", f"{cls.__name__}.get{n}FeatureValue", doc
        fn._is_deprecated = is_deprecated
        setattr(cls, fn.__name__, fn)

    kind = cls.CLASS.upper()
    for n in names:
        add(n, lambda self, _n=n: self._value(_n),
            f"{kind} {n}: same definition as the reference's Radiomics{kind}.get{n}FeatureValue (see SURVEY.md Appendix C).")
    for n, why in computable_deprecated:
        add(n, lambda self, _n=n: self._value(_n), f"{kind} {n} (deprecated in the reference: {why}).", True)
    for n, why in deprecated:
        def dep(self, _why=why):
            raise DeprecationWarning(_why)
        add(n, dep, f"DEPRECATED in the reference: {why}", True)


class RadiomicsGLCM(RadiomicsFeaturesBase):
    """Gray Level Co-occurrence Matrix features (reference radiomics/glcm.py)."""
    CLASS, MATRIX_ATTR = "glcm", "P_glcm"

    def _configure(self, kwargs):
        self.symmetricalGLCM = kwargs.get("symmetricalGLCM", True)
        self.weightingNorm = kwargs.get("weightingNorm")
        super()._configure(kwargs)

    def _calculateMatrix(self, voxelCoordinates=None):
        f2, f2d = self._matrix_args()
        if voxelCoordinates is None:           # segment mode: the discretised image never leaves the GPU
            P, angles = self._device.segment_texture(self.settings.get("distances", [1]), self.settings.get("gldm_a", 0), f2, f2d)["glcm"]
        else:
            P, angles = cmatrices.calculate_glcm(self.imageArray, self.maskArray, np.array(self.settings.get("distances", [1])),
                                                 self.coefficients["Ng"], f2, f2d, *self._batch_args(voxelCoordinates))
        return MF.glcm_process(P, self.coefficients["grayLevels"], self.symmetricalGLCM,
                               _weights(angles, self._spacing_zyx(), self.weightingNorm, "glcm"))

    def _segment_features(self):
        return MF.glcm_features(self.P_glcm[0], self.coefficients["grayLevels"], self.coefficients["Ng"])


_add_feature_getters(RadiomicsGLCM, MF.GLCM_NAMES,
                     deprecated=[("Dissimilarity", "mathematically equal to Difference Average"),
                                 ("Homogeneity1", "mathematically equal to Inverse Difference"),
                                 ("Homogeneity2", "mathematically equal to Inverse Difference Moment"),
                                 ("SumVariance", "mathematically equal to Cluster Tendency")])


class RadiomicsGLRLM(RadiomicsFeaturesBase):
    """Gray Level Run Length Matrix features (reference radiomics/glrlm.py)."""
    CLASS, MATRIX_ATTR = "glrlm", "P_glrlm"

    def _configure(self, kwargs):
        self.weightingNorm = kwargs.get("weightingNorm")
        super()._configure(kwargs)

    def _calculateMatrix(self, voxelCoordinates=None):
        f2, f2d = self._matrix_args()
        if voxelCoordinates is None:
            P, angles = cmatrices.calculate_glrlm_device(self._device.levels, self.coefficients["Ng"],
                                                         int(np.max(self._image_shape())), f2, f2d)
        else:
            P, angles = cmatrices.calculate_glrlm(self.imageArray, self.maskArray, self.coefficients["Ng"],
                                                  int(np.max(self.imageArray.shape)), f2, f2d, *self._batch_args(voxelCoordinates))
        w = _weights(angles, self._spacing_zyx(), self.weightingNorm, "glrlm")
        M, j, Nr = MF.glrlm_process(self._single_roi(P), self.coefficients["grayLevels"], w)
        self.coefficients["jvector"], self.coefficients["Nr"] = j, Nr
        return M[None]

    def _segment_features(self):
        return MF.glrlm_features(self.P_glrlm[0], self.coefficients["jvector"], self.coefficients["Nr"], self.coefficients["grayLevels"])


_add_feature_getters(RadiomicsGLRLM, MF.GLRLM_NAMES)


class _SizeMatrixClass(RadiomicsFeaturesBase):
    NAMES = None

    def _segment_features(self):
        g = MF.size_matrix_features(getattr(self, self.MATRIX_ATTR)[0], self.coefficients["grayLevels"], self.coefficients["jvector"])
        return {self.NAMES[k]: v for k, v in g.items() if k in self.NAMES}


class RadiomicsGLSZM(_SizeMatrixClass):
    """Gray Level Size Zone Matrix features (reference radiomics/glszm.py)."""
    CLASS, MATRIX_ATTR, NAMES = "glszm", "P_glszm", MF.GLSZM_NAMES

    def _calculateMatrix(self, voxelCoordinates=None):
        f2, f2d = self._matrix_args()
        if voxelCoordinates is None:
            P = cmatrices.calculate_glszm_device(self._device.levels, self.coefficients["Ng"], f2, f2d)
        else:
            P = cmatrices.calculate_glszm(self.imageArray, self.maskArray, self.coefficients["Ng"], int(np.sum(self.maskArray)),
                                          f2, f2d, *self._batch_args(voxelCoordinates))
        M, j = MF.size_matrix_process(self._single_roi(P), self.coefficients["grayLevels"])
        self.coefficients["jvector"] = j
        return M[None]


_add_feature_getters(RadiomicsGLSZM, sorted(MF.GLSZM_NAMES.values()))


class RadiomicsGLDM(_SizeMatrixClass):
    """Gray Level Dependence Matrix features (reference radiomics/gldm.py)."""
    CLASS, MATRIX_ATTR, NAMES = "gldm", "P_gldm", MF.GLDM_NAMES

    def _configure(self, kwargs):
        self.gldm_a = kwargs.get("gldm_a", 0)
        super()._configure(kwargs)

    def _calculateMatrix(self, voxelCoordinates=None):
        f2, f2d = self._matrix_args()
        if voxelCoordinates is None:
            P = self._device.segment_texture(self.settings.get("distances", [1]), self.gldm_a, f2, f2d)["gldm"]
        else:
            P = cmatrices.calculate_gldm(self.imageArray, self.maskArray, np.array(self.settings.get("distances", [1])),
                                         self.coefficients["Ng"], self.gldm_a, f2, f2d, *self._batch_args(voxelCoordinates))
        M, j = MF.size_matrix_process(self._single_roi(P), self.coefficients["grayLevels"])
        self.coefficients["jvector"] = j
        return M[None]


_add_feature_getters(RadiomicsGLDM, sorted(MF.GLDM_NAMES.values()),
                     deprecated=[("GrayLevelNonUniformityNormalized", "mathematically equal to First Order - Uniformity"),
                                 ("DependencePercentage", "always computes 1")])


class RadiomicsNGTDM(RadiomicsFeaturesBase):
    """Neighbouring Gray Tone Difference Matrix features (reference radiomics/ngtdm.py)."""
    CLASS, MATRIX_ATTR = "ngtdm", "P_ngtdm"

    def _calculateMatrix(self, voxelCoordinates=None):
        f2, f2d = self._matrix_args()
        if voxelCoordinates is None:
            P = self._device.segment_texture(self.settings.get("distances", [1]), self.settings.get("gldm_a", 0), f2, f2d)["ngtdm"]
        else:
            P = cmatrices.calculate_ngtdm(self.imageArray, self.maskArray, np.array(self.settings.get("distances", [1])),
                                          self.coefficients["Ng"], f2, f2d, *self._batch_args(voxelCoordinates))
        keep = P[:, :, 0].sum(0) != 0
        return P[:, keep]

    def _segment_features(self):
        return MF.ngtdm_features(self.P_ngtdm[0])


_add_feature_getters(RadiomicsNGTDM, MF.NGTDM_NAMES)


class RadiomicsFirstOrder(RadiomicsFeaturesBase):
    """First-order statistics (reference radiomics/firstorder.py; SURVEY.md section 8f rank 2).  Voxel-
    based: one fused CUDA kernel (rb_firstorder_voxel_dev) over the raw intensities + discretised
    levels; segment-based: the ROI vector is reduced on the host like the reference does.

    Deviation (documented in DESIGN.md): voxel-based Entropy / Uniformity histogram the SAME window as
    the other features; the reference indexes its unpadded discretised array with padded coordinates
    (firstorder.py:109), i.e. a window shifted by +kernelRadius, or raises IndexError."""
    CLASS, MATRIX_ATTR = "firstorder", "_unused_matrix"
    FROM_DEVICE_REFUSED = "segment-mode first order of device tensors is voxel.firstorder_segment"
    NAMES = ["10Percentile", "90Percentile", "Energy", "Entropy", "InterquartileRange", "Kurtosis", "Maximum",
             "MeanAbsoluteDeviation", "Mean", "Median", "Minimum", "Range", "RobustMeanAbsoluteDeviation",
             "RootMeanSquared", "Skewness", "TotalEnergy", "Uniformity", "Variance"]

    def __init__(self, inputImage, inputMask, **kwargs):
        self.voxelArrayShift = kwargs.get("voxelArrayShift", 0)
        self.pixelSpacing = I.spacing_xyz(inputImage)
        super().__init__(inputImage, inputMask, **kwargs)
        self._imageArray = self._rawImageArray      # like the reference, imageArray stays the raw intensities here

    @property
    def discretizedImageArray(self):
        return self._device.binned_host()

    def _window_radii(self):
        nd = self._rawImageArray.ndim
        rad = voxel.firstorder_radii(self.settings.get("kernelRadius", 1), self._rawImageArray.shape,
                                     self._centerMask if self.masked else None, self.settings.get("force2D", False),
                                     self.settings.get("force2Ddimension", 0))
        return [0] * (3 - nd) + rad

    def _voxel_launch(self, lev):
        """voxel.firstorder_launch on the raw intensities (uploaded once), a chunk of planes per launch: every window reads
        the whole volume, so a chunk's maps are those of one whole-volume launch"""
        img = imageoperations._to_device(self._rawImageArray)
        msk = imageoperations._to_device(self.maskArray)
        if img.ndim == 2:
            img, msk = img[None], msk[None]
        vv = float(np.multiply.reduce(self.pixelSpacing))
        return voxel.firstorder_launch(img.contiguous(), lev, msk, self._window_radii(), centers=self._centers_dev(),
                                       voxelArrayShift=self.voxelArrayShift, voxel_volume=vv,
                                       initValue=self.settings.get("initValue", 0)), None

    def _initCalculation(self, voxelCoordinates=None):
        pass

    def _segment_features(self):
        x = np.sort(self._rawImageArray[self.maskArray].astype(np.float64))
        n = x.size
        sh = x + self.voxelArrayShift
        en = float(np.sum(sh ** 2))
        mean = float(x.mean())
        pct = lambda q: float(np.percentile(x, q))
        _, cnt = np.unique(self.discretizedImageArray[self.maskArray], return_counts=True)
        p = cnt / cnt.sum()
        d = x - mean
        m2, m3, m4 = float(np.mean(d ** 2)), float(np.mean(d ** 3)), float(np.mean(d ** 4))
        m2s = 1.0 if m2 == 0 else m2
        p10, p90 = pct(10), pct(90)
        kept = x[(x >= p10) & (x <= p90)]
        return {
            "10Percentile": p10, "90Percentile": p90, "Energy": en, "Entropy": float(-np.sum(p * np.log2(p + MF.EPS))),
            "InterquartileRange": pct(75) - pct(25), "Kurtosis": m4 / m2s ** 2, "Maximum": float(x[-1]),
            "MeanAbsoluteDeviation": float(np.mean(np.abs(d))), "Mean": mean, "Median": float(np.median(x)),
            "Minimum": float(x[0]), "Range": float(x[-1] - x[0]),
            "RobustMeanAbsoluteDeviation": float(np.mean(np.abs(kept - kept.mean()))), "RootMeanSquared": float(np.sqrt(en / n)),
            "Skewness": m3 / m2s ** 1.5, "TotalEnergy": en * float(np.multiply.reduce(self.pixelSpacing)),
            "Uniformity": float(np.sum(p ** 2)), "Variance": m2,
        }

    def _value(self, name):
        return np.float64(self._segment_features()[name])


_add_feature_getters(RadiomicsFirstOrder, RadiomicsFirstOrder.NAMES,
                     deprecated=[("StandardDeviation", "the square root of Variance")])


class _ShapeClass(RadiomicsFeaturesBase):
    """what RadiomicsShape and RadiomicsShape2D share: segment-based only (the reference raises while constructing,
    shape.py:50-52 via base.py:66), no binning (shape ignores intensities), coefficients computed on first use"""
    MATRIX_ATTR = "_unused_matrix"
    VOXEL_BASED_ERROR = None
    FROM_DEVICE_REFUSED = "shape2D is computed from a host mask only"

    def __init__(self, inputImage, inputMask, **kwargs):
        if kwargs.get("voxelBased", False):
            raise NotImplementedError(self.VOXEL_BASED_ERROR)
        super().__init__(inputImage, inputMask, **kwargs)

    def _initBinning(self):
        self._imageArray = self._rawImageArray

    def _calculateVoxels(self):
        raise NotImplementedError(self.VOXEL_BASED_ERROR)

    def _value(self, name):
        if not hasattr(self, "eigenValues"):          # the last thing _initCalculation sets
            self._initCalculation()
        return np.float64(self._segment_features()[name])


class RadiomicsShape(_ShapeClass):
    """3-D shape descriptors of the ROI (reference radiomics/shape.py; SURVEY.md section 8f rank 4): mesh
    surface area / volume / maximum diameters from the CUDA marching-cubes + all-pairs kernels
    (rb_shape_coefficients_dev), axis lengths from exact integer voxel moments (rb_shape_moments_dev).
    Segment-based only, like the reference (shape.py:50-52); independent of gray values (no binning)."""
    CLASS, VOXEL_BASED_ERROR = "shape", "Shape features are not available in voxel-based mode"
    NAMES = ["MeshVolume", "VoxelVolume", "SurfaceArea", "SurfaceVolumeRatio", "Sphericity", "Maximum3DDiameter",
             "Maximum2DDiameterSlice", "Maximum2DDiameterColumn", "Maximum2DDiameterRow", "MajorAxisLength",
             "MinorAxisLength", "LeastAxisLength", "Elongation", "Flatness"]

    def __init__(self, inputImage, inputMask, **kwargs):
        if np.ndim(I.as_array(inputMask)) != 3:
            raise AssertionError("Shape features are only available in 3D. If 2D, use shape2D instead")
        super().__init__(inputImage, inputMask, **kwargs)

    FROM_DEVICE_REFUSED = None

    @classmethod
    def from_device(cls, roi, spacing_zyx, **kwargs):
        """a segment-mode instance over the ROI `roi` (a 3-D CUDA tensor, non-zero = in the ROI; no host mask exists),
        cropped to its bounding box as the reference's flow crops the mask before shape (cropToTumorMask)"""
        self = super().from_device(None, spacing_zyx, **kwargs)
        self._roi_dev = roi[voxel.roi_box(roi)]
        return self

    def _padded_mask_dev(self):
        """the ROI padded with one plane of zeros on every side (shape.py:58-72), so every ROI voxel gets its 8 cubes,
        as a uint8 CUDA tensor (a copy: the ROI mask stays as it is however often this is called)"""
        roi = getattr(self, "_roi_dev", None)
        if roi is not None:
            return torch.nn.functional.pad((roi != 0).to(torch.uint8), (1, 1, 1, 1, 1, 1)).contiguous()
        return imageoperations._to_device(np.pad(np.asarray(self.maskArray, dtype=np.uint8), 1))

    def _initCalculation(self, voxelCoordinates=None):
        from . import cshape
        self.pixelSpacing = np.array(self._spacing_zyx(), dtype=np.float64)
        m_t = self._padded_mask_dev()
        self.SurfaceArea, self.Volume, self.diameters, self._n_vertices = cshape.coefficients_device(m_t, self.pixelSpacing)
        mom = cshape.moments_device(m_t)
        self._Np = mom[0]
        self.eigenValues = cshape.covariance_eigenvalues(mom, self.pixelSpacing)

    def _segment_features(self):
        sa, vol, ev = self.SurfaceArea, self.Volume, self.eigenValues
        with np.errstate(divide="ignore", invalid="ignore"):
            sph = np.float64(36 * np.pi * vol ** 2) ** (1.0 / 3.0)
            f = {"MeshVolume": vol, "VoxelVolume": self._Np * float(np.multiply.reduce(self.pixelSpacing)), "SurfaceArea": sa,
                 "SurfaceVolumeRatio": np.float64(sa) / vol, "Sphericity": sph / sa,
                 "Compactness1": vol / (np.float64(sa) ** 1.5 * np.sqrt(np.pi)),
                 "Compactness2": 36.0 * np.pi * vol ** 2 / np.float64(sa) ** 3, "SphericalDisproportion": sa / sph,
                 "Maximum3DDiameter": self.diameters[3], "Maximum2DDiameterSlice": self.diameters[0],
                 "Maximum2DDiameterColumn": self.diameters[1], "Maximum2DDiameterRow": self.diameters[2]}
            for name, k in (("MajorAxisLength", 2), ("MinorAxisLength", 1), ("LeastAxisLength", 0)):
                f[name] = np.nan if ev[k] < 0 else np.sqrt(ev[k]) * 4            # shape.py:313-371
            f["Elongation"] = np.nan if (ev[1] < 0 or ev[2] < 0) else np.sqrt(ev[1] / ev[2])
            f["Flatness"] = np.nan if (ev[0] < 0 or ev[2] < 0) else np.sqrt(ev[0] / ev[2])
        return f


# the deprecated ones are still computable on request, skipped by enableAllFeatures (shape.py:203-273)
_add_feature_getters(RadiomicsShape, RadiomicsShape.NAMES,
                     computable_deprecated=[(n, "correlated to Sphericity")
                                            for n in ("Compactness1", "Compactness2", "SphericalDisproportion")])


class RadiomicsShape2D(_ShapeClass):
    """2-D shape descriptors of a single-slice ROI (reference radiomics/shape2D.py): perimeter, mesh surface and maximum
    diameter from the CUDA marching-squares + all-pairs kernels (rb_calculate_coefficients2D), axis lengths from the pixel
    covariance.  Segment-based only; needs a 2-D mask or a 3-D one with force2D and size 1 in force2Ddimension."""
    CLASS, VOXEL_BASED_ERROR = "shape2D", "Shape features are not available in pixel-based mode"
    NAMES = ["MeshSurface", "PixelSurface", "Perimeter", "PerimeterSurfaceRatio", "Sphericity", "MaximumDiameter",
             "MajorAxisLength", "MinorAxisLength", "Elongation"]

    def _initCalculation(self, voxelCoordinates=None):
        from . import cshape
        m = np.asarray(self.maskArray, dtype=bool)
        sp = np.array(self._spacing_zyx(), dtype=np.float64)
        if m.ndim == 3:                       # shape2D.py:62-84
            if not self.settings.get("force2D", False):
                raise ValueError("Shape2D is can only be calculated when input is 2D or 3D with `force2D=True`")
            d = self.settings.get("force2Ddimension", 0)
            if m.shape[d] > 1:
                raise ValueError("Size of the mask in dimension %i is more than 1, cannot compute 2D shape" % d)
            m = np.squeeze(m, axis=d)
            sp = np.delete(sp, d)
        elif m.ndim != 2:
            raise ValueError("Shape2D is can only be calculated when input is 2D or 3D with `force2D=True`")
        self.pixelSpacing = sp
        padded = np.pad(m, 1)
        self.Perimeter, self.Surface, self.Diameter = cshape.calculate_coefficients2D(padded, sp)
        idx = np.array(np.where(padded), dtype=np.float64).T
        self._Np = len(idx)
        phys = idx * sp[None, :]
        phys -= phys.mean(0)
        phys /= np.sqrt(self._Np)
        ev = np.linalg.eigvals(phys.T.copy() @ phys).real
        ev[(ev < 0) & (ev > -1e-10)] = 0
        self.eigenValues = np.sort(ev)

    def _segment_features(self):
        ev = self.eigenValues
        with np.errstate(divide="ignore", invalid="ignore"):
            sph = (2 * np.sqrt(np.pi * self.Surface)) / self.Perimeter
            f = {"MeshSurface": self.Surface, "PixelSurface": self._Np * float(np.multiply.reduce(self.pixelSpacing)),
                 "Perimeter": self.Perimeter, "PerimeterSurfaceRatio": self.Perimeter / self.Surface, "Sphericity": sph,
                 "SphericalDisproportion": 1.0 / sph, "MaximumDiameter": self.Diameter,
                 "MajorAxisLength": np.nan if ev[1] < 0 else np.sqrt(ev[1]) * 4,
                 "MinorAxisLength": np.nan if ev[0] < 0 else np.sqrt(ev[0]) * 4,
                 "Elongation": np.nan if (ev[0] < 0 or ev[1] < 0) else np.sqrt(ev[0] / ev[1])}
        return f


_add_feature_getters(RadiomicsShape2D, RadiomicsShape2D.NAMES,
                     computable_deprecated=[("SphericalDisproportion", "the inverse of Sphericity")])


FEATURE_CLASSES = {"glcm": RadiomicsGLCM, "glrlm": RadiomicsGLRLM, "glszm": RadiomicsGLSZM, "gldm": RadiomicsGLDM,
                   "ngtdm": RadiomicsNGTDM}
# next row of the hot-path table (SURVEY.md section 8f): registered by install() as well
NEXT_CLASSES = {"firstorder": RadiomicsFirstOrder, "shape": RadiomicsShape, "shape2D": RadiomicsShape2D}


def install(radiomics_module=None):
    """Drop the CUDA engine under an importable pyradiomics: the feature classes replace the
    reference's in ``radiomics.getFeatureClasses()`` and ``cMatrices`` is rebound in every module
    that captured it at import time (SURVEY.md section 8b)."""
    import importlib

    rad = radiomics_module or importlib.import_module("radiomics")
    classes = rad.getFeatureClasses()
    for name, cls in {**FEATURE_CLASSES, **NEXT_CLASSES}.items():
        classes[name] = cls
    rad.cMatrices = cmatrices
    from . import cshape
    # radiomics.shape2D calls cShape.calculate_coefficients2D (shape2D.py:99): the replacement forwards every name it
    # does not implement to the reference's own _cshape, so a later import / reload of shape2D keeps working
    orig = getattr(rad, "cShape", None)
    if orig is not None and orig is not cshape and getattr(orig, "__name__", "") != cshape.__name__:
        cshape._fallback = orig
    rad.cShape = cshape
    for mod in ("shape", "shape2D"):
        try:
            importlib.import_module(f"{rad.__name__}.{mod}").cShape = cshape
        except ImportError:
            pass
    for mod in ("glcm", "glrlm", "glszm", "gldm", "ngtdm", "firstorder"):
        try:
            importlib.import_module(f"{rad.__name__}.{mod}").cMatrices = cmatrices
        except ImportError:
            pass
    return classes
