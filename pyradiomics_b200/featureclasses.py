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
    """One (image, ROI mask, binning) discretised ONCE on the GPU: rb_minmax_dev -> rb_digitize_dev ->
    rb_pack_levels_dev (reference: binImage in every class constructor, base.py:119-125, i.e. 5x per image)."""

    def __init__(self, imageArray, maskRaw, label, masked, settings):
        img_t = imageoperations._to_device(imageArray)
        # the ROI mask is formed on the device: label compare of the raw mask (or all ones for an unmasked kernel)
        raw_t = imageoperations._to_device(maskRaw)
        msk_t = (raw_t == label).to(torch.uint8) if masked else torch.ones(raw_t.shape, dtype=torch.uint8, device=raw_t.device)
        lev_t, self.edges = imageoperations.bin_image_device(img_t, msk_t, **settings)
        Ng = int(lev_t.max().item())
        self.levels, presence = voxel.pack_levels(lev_t, msk_t, max(Ng, 1))
        self.grayLevels = (torch.nonzero(presence).flatten() + 1).cpu().numpy().astype(np.int64)
        self.Ng = int(self.grayLevels.max()) if self.grayLevels.size else 0
        self.mask_dev = msk_t
        self._lev32 = lev_t                     # kept until the host copy has been asked for (or never)
        self._binned_host = None
        self._alive = {}
        self._segment = {}

    def binned_host(self):
        """the reference's ``self.imageArray`` after binning: int64 levels, 0 outside the ROI (lazy: voxel mode never needs it)"""
        if self._binned_host is None:
            self._binned_host = self._lev32.cpu().numpy().astype(np.int64)
            self._lev32 = None
        return self._binned_host

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
        self.progressReporter = getProgressReporter
        self.settings = kwargs
        self.label = kwargs.get("label", 1)
        self.voxelBased = kwargs.get("voxelBased", False)
        self.coefficients = {}
        self.enabledFeatures = {}
        self.featureValues = {}
        self.featureNames = self.getFeatureNames()
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
        setattr(self, self.MATRIX_ATTR, None)
        self._initBinning()

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

    @property
    def _levels_dev(self):
        return self._device.levels

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
        return tuple(I.spacing_xyz(self.inputImage))[::-1]

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

    def _calculateVoxels(self):
        """The fused kernel of the class in z-chunks; the ENABLED maps stream to page-locked host memory chunk by
        chunk while the next chunk computes (voxel.class_maps_to_host) -- replaces the voxelBatch loop and the
        per-voxel assignment of base.py:200-245.  `voxelBatch` is accepted and ignored."""
        lev = self._device.levels3d()
        names = _lib.feature_names(self.CLASS)
        idx = [k for k, n in enumerate(names) if self.enabledFeatures.get(n)]
        for n, enabled in self.enabledFeatures.items():
            if enabled and n not in names:
                self.logger.debug("Feature %s is deprecated / not computed in voxel-based mode", n)
        if not idx:
            return
        settings = self._voxel_settings()
        centers = self._centers_dev()
        alive = self._device.glcm_alive(settings, centers) if self.CLASS == "glcm" else None
        status = torch.zeros(1, dtype=torch.int32, device=lev.device)
        # b200_zrange=(z0, z1): compute and return only these planes (a multi-GPU caller hands every rank the whole image --
        # so that bin edges, gray levels and the GLCM angle set are those of the whole ROI -- and takes one slab per rank)
        z0, z1 = self.settings.get("b200_zrange") or (0, int(lev.shape[0]))
        with self.progressReporter(total=int(z1 - z0), desc="planes") as pbar:
            host = voxel.class_maps_to_host(self.CLASS, lev, settings, idx, centers=centers, alive=alive, status=status,
                                            z0=int(z0), z1=int(z1),
                                            zchunk=self._zchunk(int(z1 - z0)), out_dtype=self._map_dtype(),
                                            progress=pbar.update)
        st = int(status.item())
        if st & 2:
            raise _lib.B200Error("weighted GLCM entry list overflow")
        if st & 1:
            self.logger.warning("MCC eigen-problem too large for the in-kernel solver at some voxels: NaN stored")
        arrs = host.numpy()                      # views of ONE page-locked block the returned images keep alive
        for pos, k in enumerate(idx):
            arr = arrs[pos] if self._rawImageArray.ndim == 3 else arrs[pos][0]
            self.featureValues[names[k]] = I.like(self.inputImage, arr)

    def _calculateSegment(self):
        self._initCalculation()
        vals = self._segment_features()
        for feature, enabled in self.enabledFeatures.items():
            if not enabled:
                continue
            if self.featureNames.get(feature) and feature not in vals:
                self.logger.debug("Feature %s is deprecated", feature)     # texture: the reference raises DeprecationWarning
                continue
            try:
                self.featureValues[feature] = np.squeeze(np.float64(vals[feature]))
            except Exception:                                  # per-feature isolation (base.py:271-273)
                self.logger.error("FAILED: %s", feature, exc_info=True)
                self.featureValues[feature] = np.nan

    def _initCalculation(self, voxelCoordinates=None):
        setattr(self, self.MATRIX_ATTR, self._calculateMatrix(voxelCoordinates))

    def _matrix_args(self):
        return self.settings.get("force2D", False), self.settings.get("force2Ddimension", 0)

    def _batch_args(self, voxelCoordinates):
        return [self.settings.get("kernelRadius", 1), voxelCoordinates] if voxelCoordinates is not None else []

    def _value(self, name):
        """single feature (the reference's get<Name>FeatureValue entry points)."""
        if getattr(self, self.MATRIX_ATTR) is None:
            self._initCalculation()
        return np.float64(self._segment_features()[name])


def _add_feature_getters(cls, names, deprecated=()):
    for n in names:
        def getter(self, _n=n):
            return self._value(_n)
        getter.__name__ = f"get{n}FeatureValue"
        getter.__doc__ = (f"{cls.CLASS.upper()} {n}: same definition as the reference's "
                          f"Radiomics{cls.CLASS.upper()}.get{n}FeatureValue (see SURVEY.md Appendix C).")
        setattr(cls, getter.__name__, getter)
    for n, why in deprecated:
        def dep(self, _why=why):
            raise DeprecationWarning(_why)
        dep.__name__ = f"get{n}FeatureValue"
        dep.__doc__ = f"DEPRECATED in the reference: {why}"
        dep._is_deprecated = True
        setattr(cls, dep.__name__, dep)


class RadiomicsGLCM(RadiomicsFeaturesBase):
    """Gray Level Co-occurrence Matrix features (reference radiomics/glcm.py)."""
    CLASS, MATRIX_ATTR = "glcm", "P_glcm"

    def __init__(self, inputImage, inputMask, **kwargs):
        self.symmetricalGLCM = kwargs.get("symmetricalGLCM", True)
        self.weightingNorm = kwargs.get("weightingNorm")
        super().__init__(inputImage, inputMask, **kwargs)

    def _calculateMatrix(self, voxelCoordinates=None):
        f2, f2d = self._matrix_args()
        if voxelCoordinates is None:           # segment mode: the discretised image never leaves the GPU
            P, angles = self._device.segment_texture(self.settings.get("distances", [1]), self.settings.get("gldm_a", 0), f2, f2d)["glcm"]
        else:
            P, angles = cmatrices.calculate_glcm(self.imageArray, self.maskArray, np.array(self.settings.get("distances", [1])),
                                                 self.coefficients["Ng"], f2, f2d, *self._batch_args(voxelCoordinates))
        w = _weights(angles, self._spacing_zyx(), self.weightingNorm, "glcm")
        # symmetrise / weight / drop the angles that are empty for EVERY voxel of the batch (glcm.py:149-205): one
        # common angle axis, so the batch stacks
        idx = np.asarray(self.coefficients["grayLevels"], int) - 1
        P = P[:, idx][:, :, idx].astype(float)
        if self.symmetricalGLCM:
            P = P + P.transpose(0, 2, 1, 3)
        if w is not None:
            P = (P * w[None, None, None, :]).sum(3, keepdims=True)
        tot = P.sum((1, 2))
        if P.shape[3] > 1:
            keep = tot.sum(0) != 0
            P, tot = P[..., keep], tot[:, keep]
        tot = np.where(tot == 0, np.nan, tot)
        return P / tot[:, None, None, :]

    def _segment_features(self):
        return MF.glcm_features(self.P_glcm[0], self.coefficients["grayLevels"], self.coefficients["Ng"])


_add_feature_getters(RadiomicsGLCM, _lib_names := [
    "Autocorrelation", "ClusterProminence", "ClusterShade", "ClusterTendency", "Contrast", "Correlation",
    "DifferenceAverage", "DifferenceEntropy", "DifferenceVariance", "Id", "Idm", "Idmn", "Idn", "Imc1", "Imc2",
    "InverseVariance", "JointAverage", "JointEnergy", "JointEntropy", "MCC", "MaximumProbability", "SumAverage",
    "SumEntropy", "SumSquares"],
    deprecated=[("Dissimilarity", "mathematically equal to Difference Average"),
                ("Homogeneity1", "mathematically equal to Inverse Difference"),
                ("Homogeneity2", "mathematically equal to Inverse Difference Moment"),
                ("SumVariance", "mathematically equal to Cluster Tendency")])


class RadiomicsGLRLM(RadiomicsFeaturesBase):
    """Gray Level Run Length Matrix features (reference radiomics/glrlm.py)."""
    CLASS, MATRIX_ATTR = "glrlm", "P_glrlm"

    def __init__(self, inputImage, inputMask, **kwargs):
        self.weightingNorm = kwargs.get("weightingNorm")
        super().__init__(inputImage, inputMask, **kwargs)

    def _calculateMatrix(self, voxelCoordinates=None):
        f2, f2d = self._matrix_args()
        if voxelCoordinates is None:
            P, angles = cmatrices.calculate_glrlm_device(self._device.levels, self.coefficients["Ng"],
                                                         int(np.max(self._rawImageArray.shape)), f2, f2d)
        else:
            P, angles = cmatrices.calculate_glrlm(self.imageArray, self.maskArray, self.coefficients["Ng"],
                                                  int(np.max(self.imageArray.shape)), f2, f2d, *self._batch_args(voxelCoordinates))
        w = _weights(angles, self._spacing_zyx(), self.weightingNorm, "glrlm")
        if P.shape[0] != 1:
            raise NotImplementedError("P_glrlm of a voxel batch: the voxel-based path is fused (no per-voxel matrices); "
                                      "use cmatrices.calculate_glrlm for dense per-voxel matrices")
        M, j, Nr = MF.glrlm_process(P[0], self.coefficients["grayLevels"], w)
        self.coefficients["jvector"], self.coefficients["Nr"] = j, Nr
        return M[None]

    def _segment_features(self):
        return MF.glrlm_features(self.P_glrlm[0], self.coefficients["jvector"], self.coefficients["Nr"], self.coefficients["grayLevels"])


_add_feature_getters(RadiomicsGLRLM, [
    "GrayLevelNonUniformity", "GrayLevelNonUniformityNormalized", "GrayLevelVariance", "HighGrayLevelRunEmphasis",
    "LongRunEmphasis", "LongRunHighGrayLevelEmphasis", "LongRunLowGrayLevelEmphasis", "LowGrayLevelRunEmphasis",
    "RunEntropy", "RunLengthNonUniformity", "RunLengthNonUniformityNormalized", "RunPercentage", "RunVariance",
    "ShortRunEmphasis", "ShortRunHighGrayLevelEmphasis", "ShortRunLowGrayLevelEmphasis"])


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
        if P.shape[0] != 1:
            raise NotImplementedError("P_glszm of a voxel batch: use cmatrices.calculate_glszm for dense per-voxel matrices")
        M, j = MF.size_matrix_process(P[0], self.coefficients["grayLevels"])
        self.coefficients["jvector"] = j
        return M[None]


_add_feature_getters(RadiomicsGLSZM, sorted(MF.GLSZM_NAMES.values()))


class RadiomicsGLDM(_SizeMatrixClass):
    """Gray Level Dependence Matrix features (reference radiomics/gldm.py)."""
    CLASS, MATRIX_ATTR, NAMES = "gldm", "P_gldm", MF.GLDM_NAMES

    def __init__(self, inputImage, inputMask, **kwargs):
        self.gldm_a = kwargs.get("gldm_a", 0)
        super().__init__(inputImage, inputMask, **kwargs)

    def _calculateMatrix(self, voxelCoordinates=None):
        f2, f2d = self._matrix_args()
        if voxelCoordinates is None:
            P = self._device.segment_texture(self.settings.get("distances", [1]), self.gldm_a, f2, f2d)["gldm"]
        else:
            P = cmatrices.calculate_gldm(self.imageArray, self.maskArray, np.array(self.settings.get("distances", [1])),
                                         self.coefficients["Ng"], self.gldm_a, f2, f2d, *self._batch_args(voxelCoordinates))
        if P.shape[0] != 1:
            raise NotImplementedError("P_gldm of a voxel batch: use cmatrices.calculate_gldm for dense per-voxel matrices")
        M, j = MF.size_matrix_process(P[0], self.coefficients["grayLevels"])
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


_add_feature_getters(RadiomicsNGTDM, ["Busyness", "Coarseness", "Complexity", "Contrast", "Strength"])

class RadiomicsFirstOrder(RadiomicsFeaturesBase):
    """First-order statistics (reference radiomics/firstorder.py; SURVEY.md section 8f rank 2).  Voxel-
    based: one fused CUDA kernel (rb_firstorder_voxel_dev) over the raw intensities + discretised
    levels; segment-based: the ROI vector is reduced on the host like the reference does.

    Deviation (documented in DESIGN.md): voxel-based Entropy / Uniformity histogram the SAME window as
    the other features; the reference indexes its unpadded discretised array with padded coordinates
    (firstorder.py:109), i.e. a window shifted by +kernelRadius, or raises IndexError."""
    CLASS, MATRIX_ATTR = "firstorder", "_unused_matrix"
    NAMES = ["10Percentile", "90Percentile", "Energy", "Entropy", "InterquartileRange", "Kurtosis", "Maximum",
             "MeanAbsoluteDeviation", "Mean", "Median", "Minimum", "Range", "RobustMeanAbsoluteDeviation",
             "RootMeanSquared", "Skewness", "TotalEnergy", "Uniformity", "Variance"]

    def __init__(self, inputImage, inputMask, **kwargs):
        self.voxelArrayShift = kwargs.get("voxelArrayShift", 0)
        self.pixelSpacing = I.spacing_xyz(inputImage)
        self._raw = I.as_array(inputImage)
        super().__init__(inputImage, inputMask, **kwargs)
        self._imageArray = self._raw          # like the reference, imageArray stays the raw intensities here

    @property
    def discretizedImageArray(self):
        return self._device.binned_host()

    def _window_radii(self):
        r = int(self.settings.get("kernelRadius", 1))
        nd = self._raw.ndim
        if self.masked:
            m = self._centerMask
            size = []
            for d in range(m.ndim):
                on = np.flatnonzero(m.any(axis=tuple(k for k in range(m.ndim) if k != d)))
                size.append(int(on[-1] - on[0] + 1))
            size = np.array(size)
        else:
            size = np.array(self._raw.shape)
        rad = [int(min(r, s - 1)) for s in size]
        if self.settings.get("force2D", False):
            rad[self.settings.get("force2Ddimension", 0)] = 0
        return [0] * (3 - nd) + rad

    def _calculateVoxels(self):
        import ctypes as C
        img = imageoperations._to_device(self._raw)
        msk = imageoperations._to_device(self.maskArray)
        lev = self._levels_dev
        if img.ndim == 2:
            img, msk, lev = img[None], msk[None], lev[None]
        centers = None if self.masked else imageoperations._to_device(self._centerMask if self._centerMask.ndim == 3 else self._centerMask[None])
        Z, Y, X = img.shape
        rz, ry, rx = self._window_radii()
        nf = _lib.lib().rb_firstorder_num_features()
        out = torch.empty((nf, Z, Y, X), dtype=torch.float64, device=img.device)
        vv = float(np.multiply.reduce(self.pixelSpacing))
        idx = [k for k, n in enumerate(self.NAMES) if self.enabledFeatures.get(n)]
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        _lib.check(_lib.lib().rb_firstorder_voxel_dev(
            ptr(img), imageoperations._TORCH_DT[img.dtype], ptr(msk), ptr(centers), ptr(lev), voxel.level_bytes(lev), Z, Y, X,
            rz, ry, rx, C.c_double(float(self.voxelArrayShift)), C.c_double(vv), C.c_double(float(self.settings.get("initValue", 0))),
            ptr(out), C.c_longlong(out.stride(0)), 0, Z, 0, C.c_void_p(torch.cuda.current_stream().cuda_stream)), "firstorder")
        if not idx:
            return
        host = torch.empty((len(idx), Z, Y, X), dtype=torch.float64, pin_memory=True)     # enabled maps only
        for pos, k in enumerate(idx):
            host[pos].copy_(out[k], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        arrs = host.numpy()
        for pos, k in enumerate(idx):
            arr = arrs[pos] if self._raw.ndim == 3 else arrs[pos][0]
            self.featureValues[self.NAMES[k]] = I.like(self.inputImage, arr)

    def _initCalculation(self, voxelCoordinates=None):
        pass

    def _segment_features(self):
        x = np.sort(self._raw[self.maskArray].astype(np.float64))
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

class RadiomicsShape(RadiomicsFeaturesBase):
    """3-D shape descriptors of the ROI (reference radiomics/shape.py; SURVEY.md section 8f rank 4): mesh
    surface area / volume / maximum diameters from the CUDA marching-cubes + all-pairs kernels
    (rb_shape_coefficients_dev), axis lengths from exact integer voxel moments (rb_shape_moments_dev).
    Segment-based only, like the reference (shape.py:50-52); independent of gray values (no binning)."""
    CLASS, MATRIX_ATTR = "shape", "_unused_matrix"
    NAMES = ["MeshVolume", "VoxelVolume", "SurfaceArea", "SurfaceVolumeRatio", "Sphericity", "Maximum3DDiameter",
             "Maximum2DDiameterSlice", "Maximum2DDiameterColumn", "Maximum2DDiameterRow", "MajorAxisLength",
             "MinorAxisLength", "LeastAxisLength", "Elongation", "Flatness"]
    DEPRECATED = ["Compactness1", "Compactness2", "SphericalDisproportion"]

    def __init__(self, inputImage, inputMask, **kwargs):
        if np.ndim(I.as_array(inputMask)) != 3:
            raise AssertionError("Shape features are only available in 3D. If 2D, use shape2D instead")
        if kwargs.get("voxelBased", False):      # the reference raises while constructing (shape.py:50-52 via base.py:66)
            raise NotImplementedError("Shape features are not available in voxel-based mode")
        super().__init__(inputImage, inputMask, **kwargs)

    def _initBinning(self):                   # shape ignores intensities
        self._imageArray = self._rawImageArray

    def _calculateVoxels(self):
        raise NotImplementedError("Shape features are not available in voxel-based mode")

    def _initCalculation(self, voxelCoordinates=None):
        from . import cshape
        self.pixelSpacing = np.array(self._spacing_zyx(), dtype=np.float64)
        # pad with one plane of zeros on every side (shape.py:58-72): every ROI voxel gets its 8 cubes
        # (a local copy: self.maskArray stays the ROI mask however often this is called)
        padded = np.pad(np.asarray(self.maskArray, dtype=np.uint8), 1)
        m_t = imageoperations._to_device(padded)
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

    def _value(self, name):
        if not hasattr(self, "SurfaceArea"):
            self._initCalculation()
        return np.float64(self._segment_features()[name])


def _add_shape_getters():
    _add_feature_getters(RadiomicsShape, RadiomicsShape.NAMES)
    for n in RadiomicsShape.DEPRECATED:       # still computable on request, skipped by enableAllFeatures (shape.py:203-273)
        def getter(self, _n=n):
            return self._value(_n)
        getter.__name__ = f"get{n}FeatureValue"
        getter.__doc__ = f"SHAPE {n} (deprecated in the reference: correlated to Sphericity)."
        getter._is_deprecated = True
        setattr(RadiomicsShape, getter.__name__, getter)


_add_shape_getters()

class RadiomicsShape2D(RadiomicsFeaturesBase):
    """2-D shape descriptors of a single-slice ROI (reference radiomics/shape2D.py): perimeter, mesh surface and maximum
    diameter from the CUDA marching-squares + all-pairs kernels (rb_calculate_coefficients2D), axis lengths from the pixel
    covariance.  Segment-based only; needs a 2-D mask or a 3-D one with force2D and size 1 in force2Ddimension."""
    CLASS, MATRIX_ATTR = "shape2D", "_unused_matrix"
    NAMES = ["MeshSurface", "PixelSurface", "Perimeter", "PerimeterSurfaceRatio", "Sphericity", "MaximumDiameter",
             "MajorAxisLength", "MinorAxisLength", "Elongation"]
    DEPRECATED = ["SphericalDisproportion"]

    def __init__(self, inputImage, inputMask, **kwargs):
        if kwargs.get("voxelBased", False):
            raise NotImplementedError("Shape features are not available in pixel-based mode")
        super().__init__(inputImage, inputMask, **kwargs)

    def _initBinning(self):                   # shape ignores intensities
        self._imageArray = self._rawImageArray

    def _calculateVoxels(self):
        raise NotImplementedError("Shape features are not available in pixel-based mode")

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

    def _value(self, name):
        if not hasattr(self, "Surface"):
            self._initCalculation()
        return np.float64(self._segment_features()[name])


def _add_shape2d_getters():
    _add_feature_getters(RadiomicsShape2D, RadiomicsShape2D.NAMES)
    for n in RadiomicsShape2D.DEPRECATED:
        def getter(self, _n=n):
            return self._value(_n)
        getter.__name__ = f"get{n}FeatureValue"
        getter.__doc__ = f"SHAPE2D {n} (deprecated in the reference: the inverse of Sphericity)."
        getter._is_deprecated = True
        setattr(RadiomicsShape2D, getter.__name__, getter)


_add_shape2d_getters()

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
