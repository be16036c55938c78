"""No-GPU checks of the Python side of the C ABI against include/b200radiomics.h: the ctypes prototype table, the pixel-type
codes, the layout of rb_voxel_settings, argument type checking, and the one dtype check every entry point runs before it
touches the device."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from pyradiomics_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200radiomics.h")


@pytest.fixture(scope="module")
def L():
    build.build()
    return _lib.lib()


def header_text():
    txt = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return "\n".join(line for line in txt.splitlines() if not line.lstrip().startswith("#"))


def header_prototypes():
    """{name: (return type, [parameter declarations])} of every function the header declares"""
    out = {}
    for decl in header_text().split(";"):
        m = re.fullmatch(r"\s*([\w\s*]+?)\s*\b(rb_\w+)\s*\(([^()]*)\)\s*", decl)
        if m:
            params = [p.strip() for p in m.group(3).split(",")]
            out[m.group(2)] = (" ".join(m.group(1).split()), [] if params == ["void"] else params)
    return out


def ctype_of_param(decl):
    if "*" in decl:
        return C.POINTER(_lib.VoxelSettings) if "rb_voxel_settings" in decl else C.c_void_p
    scalar = " ".join(decl.split()[:-1])
    return {"int": C.c_int, "long long": C.c_longlong, "unsigned long long": C.c_ulonglong, "double": C.c_double}[scalar]


def ctype_of_result(decl):
    return {"int": C.c_int, "void": None, "const char *": C.c_char_p}[decl]


def test_prototype_table_matches_header(L):
    protos = header_prototypes()
    assert len(protos) >= 40 and "rb_calculate_coefficients2D" in protos
    assert set(_lib.PROTOTYPES) == set(protos)
    for name, (res, params) in protos.items():
        want = (ctype_of_result(res), [ctype_of_param(p) for p in params])
        assert _lib.PROTOTYPES[name] == want, name
        f = getattr(L, name)
        assert f.restype is want[0] and tuple(f.argtypes) == tuple(want[1]), name


def test_dtype_codes_match_header():
    body = re.search(r"typedef enum \{([^}]*)\} rb_dtype;", header_text()).group(1)
    codes = {n.lower(): int(v) for n, v in re.findall(r"RB_DT_(\w+)\s*=\s*(\d+)", body)}
    assert len(codes) == 7
    assert _lib.DTYPE_CODE == {np.dtype(n): v for n, v in codes.items()}
    assert _lib.TORCH_DTYPE_CODE and all(codes[str(t).removeprefix("torch.")] == v for t, v in _lib.TORCH_DTYPE_CODE.items())
    for t, n in _lib.NP_OF_TORCH.items():
        assert _lib.TORCH_OF_NP[n] is t and _lib.DTYPE_CODE[np.dtype(n)] == _lib.TORCH_DTYPE_CODE[t]


def test_wrong_argument_type_is_refused(L):
    sz, d, buf = np.full(3, 5, np.int32), np.ones(1, np.int32), np.zeros((400, 3), np.int32)
    with pytest.raises(C.ArgumentError):
        L.rb_generate_angles(_lib.ptr(sz), 3.0, _lib.ptr(d), 1, 0, 0, 0, _lib.ptr(buf), 400)
    with pytest.raises(C.ArgumentError):
        L.rb_minmax_dev(None, 0, None, 8.0, None, None)
    assert L.rb_generate_angles(_lib.ptr(sz), 3, _lib.ptr(d), 1, 0, 0, 0, _lib.ptr(buf), 400) == 13


BUF = np.zeros(1 << 13)


def dtype_calls(L):
    """{(entry point, dtype parameter): call(code)} with every other argument valid; every pointer is real host memory"""
    p = _lib.ptr(BUF)
    n, sizes, start, step = 8, np.full(3, 2, np.int32), np.zeros(3), np.ones(3)
    verts, harm, w, rp = np.zeros((1, 3)), np.zeros((1, 1, 2)), np.ones(3), np.zeros(8)
    ok = _lib.DTYPE_CODE[np.dtype(np.float64)]
    return {
        ("rb_minmax_dev", "dtype"): lambda dt: L.rb_minmax_dev(p, dt, p, n, p, None),
        ("rb_digitize_dev", "dtype"): lambda dt: L.rb_digitize_dev(p, dt, p, n, p, 1, p, None),
        ("rb_pointwise_image_dev", "dtype"): lambda dt: L.rb_pointwise_image_dev(p, dt, n, 0, 1.0, p, None),
        ("rb_gradient_magnitude_dev", "dtype"): lambda dt: L.rb_gradient_magnitude_dev(p, dt, 2, 2, 2, _lib.ptr(w), p, None),
        ("rb_roi_moments_dev", "dtype"): lambda dt: L.rb_roi_moments_dev(p, dt, p, n, 1, p, p, None),
        ("rb_normalize_dev", "dtype"): lambda dt: L.rb_normalize_dev(p, dt, n, 0.0, 1.0, 0, 0.0, 1.0, p, None),
        ("rb_resegment_dev", "dtype"): lambda dt: L.rb_resegment_dev(p, dt, p, n, 0.0, 1.0, 1, p, p, None),
        ("rb_resample_dev", "src_dtype"): lambda dt: L.rb_resample_dev(
            p, dt, _lib.ptr(sizes), p, ok, _lib.ptr(sizes), _lib.ptr(start), _lib.ptr(step), 0, 0.0, None),
        ("rb_resample_dev", "dst_dtype"): lambda dt: L.rb_resample_dev(
            p, ok, _lib.ptr(sizes), p, dt, _lib.ptr(sizes), _lib.ptr(start), _lib.ptr(step), 0, 0.0, None),
        ("rb_lbp3d_dev", "img_dtype"): lambda dt: L.rb_lbp3d_dev(
            p, dt, ok, p, 2, 2, 2, _lib.ptr(verts), 1, _lib.ptr(harm), 1, p, p, None),
        ("rb_lbp3d_dev", "sample_dtype"): lambda dt: L.rb_lbp3d_dev(
            p, ok, dt, p, 2, 2, 2, _lib.ptr(verts), 1, _lib.ptr(harm), 1, p, p, None),
        ("rb_lbp2d_dev", "dtype"): lambda dt: L.rb_lbp2d_dev(p, dt, 2, 2, 2, 0, 8, _lib.ptr(rp), _lib.ptr(rp), 0, p, None),
        ("rb_firstorder_voxel_dev", "dtype"): lambda dt: L.rb_firstorder_voxel_dev(
            p, dt, p, p, p, 1, 2, 2, 2, 1, 1, 1, 0.0, 1.0, 0.0, p, n, 0, 2, 0, None),
    }


def test_dtype_calls_cover_every_dtype_parameter(L):
    declared = {(name, p.split()[-1]) for name, (_, params) in header_prototypes().items() for p in params
                if p.split()[-1].endswith("dtype")}
    assert set(dtype_calls(L)) == declared


@pytest.mark.parametrize("code", [-1, 7])
def test_unknown_dtype_code_is_refused_before_the_device(L, code):
    # placeholder device pointers must never reach a card: this runs only where there is none
    if torch.cuda.is_available() or L.rb_device_count() > 0:
        pytest.skip("GPU present")
    for key, call in dtype_calls(L).items():
        assert call(code) == _lib.RB_ERR_ARG, key
        assert b"unknown dtype code" in L.rb_last_error(), key
        assert call(_lib.DTYPE_CODE[np.dtype(np.float64)]) == _lib.RB_ERR_CUDA, key       # a valid code goes on to CUDA


def test_voxel_settings_offsets_match_header(tmp_path):
    body = re.search(r"typedef struct \{([^}]*)\} rb_voxel_settings;", header_text()).group(1)
    fields = [name for name, _ in _lib.VoxelSettings._fields_]
    assert re.findall(r"(\w+)(?:\[\d+\])?\s*;", body) == fields
    src = tmp_path / "offsets.cpp"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200radiomics.h"\nint main() {\n'
                   + "".join(f'  printf("%zu\\n", offsetof(rb_voxel_settings, {n}));\n' for n in fields) + "  return 0;\n}\n")
    exe = tmp_path / "offsets"
    subprocess.check_call(["g++", "-O2", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    offsets = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert offsets == [getattr(_lib.VoxelSettings, n).offset for n in fields]
