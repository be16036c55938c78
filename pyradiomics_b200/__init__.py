"""pyradiomics_b200 -- H100-native (sm_90a) texture-matrix engine behind pyradiomics' feature-class API.

Python host code (this package) over a ctypes C ABI (include/b200radiomics.h) into hand-written
sm_90a CUDA kernels (pyradiomics_b200/csrc).  PyTorch is used only for device memory, streams
and torch.distributed.  There is no CPU fallback anywhere in the product path.
"""
from ._lib import B200Error, CLASSES, feature_names, lib  # noqa: F401

__version__ = "0.1.0"


def install(radiomics_module=None):
    """register the CUDA feature classes / cMatrices / cShape in an importable pyradiomics (featureclasses.install)"""
    from .featureclasses import install as _install
    return _install(radiomics_module)
