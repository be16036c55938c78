"""rb_firstorder_segment_dev refuses malformed arguments before anything reaches a device; from_device refuses the plugin
classes it cannot build."""
import ctypes as C

import pytest
import torch

from pyradiomics_b200 import _lib, featureclasses as FC


@pytest.mark.parametrize("args, msg", [((7, 1, 2, 2, 2), b"unknown dtype code"), ((-1, 1, 2, 2, 2), b"unknown dtype code"),
                                       ((0, 3, 2, 2, 2), b"level_bytes"), ((0, 1, 0, 2, 2), b"empty"),
                                       ((0, 2, 2, 0, 2), b"empty")])
def test_bad_arguments_are_refused_before_the_device(args, msg):
    if torch.cuda.is_available():
        pytest.skip("GPU present: placeholder device pointers must never reach a card")
    L = _lib.lib()
    code, lb, Z, Y, X = args
    out = (C.c_double * 18)()
    p = 16
    assert L.rb_firstorder_segment_dev(p, code, p, p, lb, Z, Y, X, 0.0, 1.0, out, None) == _lib.RB_ERR_ARG
    assert msg in L.rb_last_error()


@pytest.mark.parametrize("cls", [FC.RadiomicsFirstOrder, FC.RadiomicsShape2D])
def test_from_device_refuses_the_classes_it_cannot_build(cls):
    with pytest.raises(NotImplementedError):
        cls.from_device(None, (1.0, 1.0, 1.0))
