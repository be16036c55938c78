"""The shape kernels (csrc/shape.cu) at sizes where their loops run, against the vectorised exact oracle
(oracle/shape_np.mesh / mesh2d) and the compiled reference _cshape.

Launch rules, restated below from shape_coefficients_dev / shape2d_coefficients_dev / shape_moments_dev and
common.cuh::grid_for: the mesh, 2-D mesh and moments kernels run grid_for(n, 256, 8) blocks of 256 threads (at most
SMs x 8 blocks, one item per thread, grid-stride beyond); the diameter kernels run grid_for(tiles, 1, 8) blocks over
tiles of 256 vertices, so their outer loops run only above SMs x 8 x 256 vertices.  Every case asserts which loops it
makes run and prints its vertex count, grids and the worst area / volume error as a fraction of its bound.

Bounds.  With dyadic spacings (0.5, 0.75, 1.25, ...) every per-triangle term is exact (the oracle asserts it), so the
only rounding is in the sums: each thread adds its terms in order, a block adds its 256 partial sums in a tree of
log2(256) = 8 levels and the blocks meet in one atomicAdd each, so every term passes through at most
    depth = terms per thread + 8 + blocks
roundings, and |kernel sum - exact sum| <= depth * 2^-53 * sum|terms| (plus one rounding of the exact value itself and
of the final division by 6 for the volume).  Against the reference with other spacings the terms are rounded too: both
sides then also carry a per-term rounding scaled by shape_np.mesh's `area_mag` / `vol_mag`.  Diameters and vertex counts
are exact and order-free: they are compared bit for bit.  The area / volume sums are not deterministic (the blocks'
atomicAdd order varies), so two runs are held to twice the bound."""
from fractions import Fraction
import math
import time

import numpy as np
import pytest
import torch

import shape_np as S
from pyradiomics_b200 import cshape, featureclasses as FC, image as I
from pyradiomics_b200._lib import lib, ptr

pytestmark = pytest.mark.gpu

U = S.U
MAX_TRI = int(((S._TRI >= 0).sum(1) // 3).max())          # triangles of the fullest cube configuration (5)
SP3 = (0.75, 1.25, 0.5)
SP2 = (0.75, 1.25)


# ---------------------------------------------------------------------------------------------------- launch geometry
def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _grid_for(n, block, per_sm=8):
    """common.cuh grid_for: ceil(n / block) blocks, at least 1, at most SMs x per_sm"""
    return max(1, min(-(-n // block), _sms() * per_sm))


def _launch3d(shape, nverts):
    """(mesh blocks, terms per thread bound, diameter blocks, vertex tiles)"""
    ncubes = math.prod(s - 1 for s in shape)
    g = _grid_for(ncubes, 256)
    tiles = -(-nverts // 256)
    return g, MAX_TRI * -(-ncubes // (g * 256)), _grid_for(tiles, 1), tiles


def _launch2d(shape, nverts):
    nsq = (shape[0] - 1) * (shape[1] - 1)
    g = _grid_for(nsq, 256)
    tiles = -(-nverts // 256)
    return g, -(-nsq // (g * 256)), _grid_for(tiles, 1), tiles


def _exact_vol(o):
    return float(Fraction(o["vol6"]) * Fraction(o["vol6_unit"]) / 6)


# ---------------------------------------------------------------------------------------------------- masks
def _ellipsoid(n=200, seed=1, holes=0.03):
    """a noisy ellipsoid with interior holes filling most of an n^3 box, not touching its faces"""
    rng = np.random.default_rng(seed)
    z, y, x = np.ogrid[:n, :n, :n]
    c, r = (n - 1) / 2, (n - 8) / 2
    f = ((z - c - 0.3) / r) ** 2 + ((y - c + 0.2) / (0.92 * r)) ** 2 + ((x - c - 0.1) / (0.97 * r)) ** 2
    return (f < 1.0 + 0.05 * rng.standard_normal(f.shape)) & (rng.random(f.shape) > holes)


def _noise_box():
    return np.random.default_rng(2).random((72, 80, 88)) < 0.5


def _touching_faces():
    """an ellipsoid larger than its 150 x 140 x 160 box (it touches all six faces, unpadded) with 3 % holes"""
    rng = np.random.default_rng(3)
    z, y, x = np.ogrid[:150, :140, :160]
    f = ((z - 74.5) / 90) ** 2 + ((y - 69.5) / 85) ** 2 + ((x - 79.5) / 95) ** 2
    m = (f < 1.0) & (rng.random((150, 140, 160)) > 0.03)
    assert m[0].any() and m[-1].any() and m[:, 0].any() and m[:, -1].any() and m[:, :, 0].any() and m[:, :, -1].any()
    return m


CASES3D = {"ellipsoid_200_holes": _ellipsoid, "noise_box": _noise_box, "touching_six_faces": _touching_faces}


def _check_sums3d(what, area, vol, o, depth, log):
    """area and volume within the summation bound of the exact values; returns the worst error / bound"""
    exact_area = o["area_fsum"]
    ba = S.sum_bound(depth, exact_area) + U * exact_area
    bv = S.sum_bound(depth, o["vol_terms_abs"]) / 6 + 2 * U * abs(vol)
    ev, ea = abs(vol - _exact_vol(o)), abs(area - exact_area)
    assert ea <= ba, (what, "area", area, exact_area, ea, ba)
    assert ev <= bv, (what, "volume", vol, _exact_vol(o), ev, bv)
    log.append(f"{what}: area err/bound {ea / ba:.3f}, volume err/bound {ev / bv:.3f}")
    return max(ea / ba, ev / bv), ba, bv


@pytest.mark.parametrize("name", list(CASES3D))
def test_mesh_and_diameters_at_scale_match_exact_oracle(name):
    m = CASES3D[name]()
    o = S.mesh(m, SP3)
    assert o["exact"]
    g, tpt, dg, tiles = _launch3d(m.shape, o["n_verts"])
    depth = tpt + 8 + g
    log = [f"{name} {m.shape}: {o['n_verts']} vertices, {tiles} vertex tiles, diameter grid {dg}, mesh grid {g} "
           f"({tpt} terms per thread at most), depth {depth}"]
    assert dg < tiles, "the diameter kernel's tile loop must run"
    assert g * 256 < math.prod(s - 1 for s in m.shape), "the mesh kernel's grid-stride loop must run"
    expect_dia = [float(np.sqrt(v * o["dia2_unit"])) for v in o["dia2_exact"]]
    assert expect_dia == o["dia"]

    sa, vol, dia = cshape.calculate_coefficients(m, np.array(SP3))
    assert list(dia) == expect_dia
    _check_sums3d("host entry", sa, vol, o, depth, log)
    mt = torch.as_tensor(m.astype(np.uint8)).cuda()
    runs = []
    for r in range(2):
        a, v, d, nv = cshape.coefficients_device(mt, SP3)
        assert nv == o["n_verts"] and list(d) == expect_dia, (r, nv, d)
        _, ba, bv = _check_sums3d(f"device entry run {r}", a, v, o, depth, log)
        runs.append((a, v))
    (a0, v0), (a1, v1) = runs
    assert abs(a0 - a1) <= 2 * ba and abs(v0 - v1) <= 2 * bv
    log.append(f"run-to-run spread: area {abs(a0 - a1):.3g} ({abs(a0 - a1) / max(a0, 1e-300):.2g} rel), "
               f"volume {abs(v0 - v1):.3g} ({abs(v0 - v1) / max(abs(v0), 1e-300):.2g} rel)")
    print("\n" + "\n".join(log))


def _rough_disc():
    rng = np.random.default_rng(4)
    yy, xx = np.ogrid[:900, :900]
    f = ((yy - 449.5) / 420) ** 2 + ((xx - 449.5) / 400) ** 2
    return np.pad((f < 1.0 + 0.03 * rng.standard_normal((900, 900))) & (rng.random((900, 900)) > 0.02), 1)


def _touching_border_2d():
    rng = np.random.default_rng(5)
    yy, xx = np.ogrid[:700, :600]
    m = ((yy - 349.5) / 380) ** 2 + ((xx - 299.5) / 330) ** 2 < 1.0
    m &= rng.random((700, 600)) > 0.05
    assert m[0].any() and m[-1].any() and m[:, 0].any() and m[:, -1].any()
    return m


CASES2D = {"noise_1000_padded": lambda: np.pad(np.random.default_rng(6).random((1000, 1000)) < 0.5, 1),
           "rough_disc_padded": _rough_disc, "touching_border_unpadded": _touching_border_2d}


@pytest.mark.parametrize("name", list(CASES2D))
def test_mesh2d_at_scale_matches_exact_oracle(name):
    m = CASES2D[name]()
    o = S.mesh2d(m, SP2)
    assert o["dia2_exact"] is not None
    g, tpt, dg, tiles = _launch2d(m.shape, o["n_verts"])
    depth = tpt + 8 + g
    line = (f"{name} {m.shape}: {o['n_verts']} vertices, {tiles} vertex tiles, diameter grid {dg}, mesh grid {g}, "
            f"depth {depth}")
    if name.startswith("noise"):
        assert dg < tiles, "the 2-D diameter kernel's i0 loop must run"
    assert g * 256 < (m.shape[0] - 1) * (m.shape[1] - 1), "the 2-D mesh kernel's grid-stride loop must run"
    per, sur, dia = cshape.calculate_coefficients2D(m, np.array(SP2))
    assert sur == ((o["eighths"] * 0.125) * SP2[0]) * SP2[1]
    assert dia == float(np.sqrt(o["dia2_exact"] * 4.0 ** -(max(S._dyadic(s)[1] for s in SP2) + 1))) == o["dia"]
    bp = S.sum_bound(depth, o["per_fsum"]) + U * o["per_fsum"]
    assert abs(per - o["per_fsum"]) <= bp, (per, o["per_fsum"], bp)
    print(f"\n{line}; perimeter err/bound {abs(per - o['per_fsum']) / bp:.3f}")


# ---------------------------------------------------------------------------------------------------- axis limits
@pytest.mark.parametrize("axis", range(3))
def test_extent_32767_on_each_axis_gives_exact_diameters(axis):
    """(2, 3, 32767) and its permutations, full end planes of the long axis and a random one in the middle: half-index
    coordinates reach 65531, so a ushort that wrapped would show in the diameters"""
    shape = [2, 3, 3]
    shape[axis] = 32767
    m = np.zeros(shape, bool)
    idx = [slice(None)] * 3
    for k in (0, 16000, 32766):
        idx[axis] = k
        sub = m[tuple(idx)]
        sub[...] = True if k != 16000 else np.random.default_rng(k).random(sub.shape) < 0.6
    o = S.mesh(m, SP3)
    assert o["exact"] and o["n_verts"] > 0
    sa, vol, dia = cshape.calculate_coefficients(m, np.array(SP3))
    assert list(dia) == o["dia"]
    assert o["dia"][3] >= 32764 * SP3[axis] and o["verts"][:, axis].max() >= 65531
    a, v, d, nv = cshape.coefficients_device(torch.as_tensor(m.astype(np.uint8)).cuda(), SP3)
    assert list(d) == o["dia"] and nv == o["n_verts"]
    g, tpt, _, _ = _launch3d(m.shape, o["n_verts"])
    _check_sums3d(f"extent 32767 on axis {axis}", sa, vol, o, tpt + 8 + g, [])
    _check_sums3d(f"extent 32767 on axis {axis}, device", a, v, o, tpt + 8 + g, [])


@pytest.mark.parametrize("axis", range(2))
def test_2d_extent_32767_after_padding_gives_exact_diameter(axis):
    shape = [1, 1]
    shape[axis] = 32765
    m = np.zeros(shape, bool)
    m.flat[[0, 16000, 32764]] = True
    mp = np.pad(m, 1)
    assert mp.shape[axis] == 32767
    o = S.mesh2d(mp, SP2)
    per, sur, dia = cshape.calculate_coefficients2D(mp, np.array(SP2))
    assert dia == o["dia"] and dia > 32000 * min(SP2)
    assert sur == ((o["eighths"] * 0.125) * SP2[0]) * SP2[1]
    ref = FC.RadiomicsShape2D(I.ArrayImage(np.zeros(m.shape, np.int16), SP2[::-1]),
                              I.ArrayImage(m.astype(np.uint8), SP2[::-1])).execute()
    assert float(ref["MaximumDiameter"]) == o["dia"]


def test_extent_32768_is_refused_and_flat_masks_give_zeros():
    ref = _cshape()
    for shape in ((2, 2, 32768), (2, 32768, 2), (32768, 2, 2)):
        with pytest.raises(ValueError):
            cshape.calculate_coefficients(np.ones(shape, np.int8), np.array(SP3))
        with pytest.raises(ValueError):
            cshape.coefficients_device(torch.ones(shape, dtype=torch.uint8, device="cuda"), SP3)
    for shape in ((2, 32768), (32768, 2)):
        with pytest.raises(ValueError):
            cshape.calculate_coefficients2D(np.ones(shape, np.int8), np.array(SP2))
    for shape in ((1, 5, 6), (5, 1, 6), (5, 6, 1), (1, 1, 40000)):
        m = np.ones(shape, np.int8)
        got = cshape.calculate_coefficients(m, np.array(SP3))
        assert got == (0.0, 0.0, (0.0, 0.0, 0.0, 0.0)) == ref.calculate_coefficients(m, np.array(SP3))
        assert cshape.coefficients_device(torch.as_tensor(m.astype(np.uint8)).cuda(), SP3) == (0.0, 0.0, (0.0,) * 4, 0)
    for shape in ((1, 7), (7, 1)):
        m = np.ones(shape, np.int8)
        assert cshape.calculate_coefficients2D(m, np.array(SP2)) == (0.0, 0.0, 0.0) == ref.calculate_coefficients2D(m, np.array(SP2))


# ---------------------------------------------------------------------------------------------------- moments
def _exact_moments(m):
    """{N, z, y, x, zz, zy, zx, yy, yx, xx} as Python ints, from NumPy integer marginals"""
    m = m.astype(np.int64)
    ax = [np.arange(s, dtype=np.int64) for s in m.shape]
    c1 = [m.sum(axis=tuple(d for d in range(3) if d != k)) for k in range(3)]
    c2 = {(0, 1): m.sum(2), (0, 2): m.sum(1), (1, 2): m.sum(0)}
    s = [int(c1[0].sum())] + [int((ax[k] * c1[k]).sum()) for k in range(3)]
    for i, j in ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)):
        s.append(int((ax[i] ** 2 * c1[i]).sum()) if i == j else int((ax[i][:, None] * ax[j][None, :] * c2[(i, j)]).sum()))
    return s


@pytest.mark.parametrize("kind", ["random", "full", "empty", "last_voxel"])
def test_moments_with_grid_stride_loop_equal_exact_sums(kind):
    shape = (257, 263, 271)
    n = math.prod(shape)
    assert _grid_for(n, 256) * 256 < n, "the moments kernel's grid-stride loop must run"
    if kind == "random":
        m = np.random.default_rng(7).random(shape) < 0.5
    else:
        m = np.full(shape, kind == "full")
        if kind == "last_voxel":
            m[-1, -1, -1] = True
    got = cshape.moments_device(torch.as_tensor(m.astype(np.uint8)).cuda())
    assert got == _exact_moments(m)


def test_shape_class_on_large_roi_matches_oracle_features():
    """RadiomicsShape on the 200^3 ellipsoid (the class pads it): diameters and VoxelVolume exact, the other features
    within 1e-12 relative of features built from the oracle's exact area / volume and an exact-moment NumPy covariance
    (area and volume themselves are within ~1e-13 relative by the bound above; the derived features add a few
    roundings, and the eigenvalues of a 3 x 3 symmetric matrix agree to ~1e-15 between solvers)"""
    m = _ellipsoid()
    sp_xyz = SP3[::-1]
    got = FC.RadiomicsShape(I.ArrayImage(np.zeros(m.shape, np.int16), sp_xyz), I.ArrayImage(m.astype(np.uint8), sp_xyz)).execute()
    o = S.mesh(np.pad(m, 1), SP3)
    sa, vol = o["area_fsum"], _exact_vol(o)
    mo = _exact_moments(m)
    N = mo[0]
    s2 = {(0, 0): mo[4], (0, 1): mo[5], (0, 2): mo[6], (1, 1): mo[7], (1, 2): mo[8], (2, 2): mo[9]}
    cov = np.array([[float(Fraction(N * s2[min(i, j), max(i, j)] - mo[1 + i] * mo[1 + j], N * N)) * SP3[i] * SP3[j]
                     for j in range(3)] for i in range(3)])
    ev = np.sort(np.linalg.eigvalsh(cov))
    sph = (36 * np.pi * vol ** 2) ** (1.0 / 3.0)
    ref = {"MeshVolume": vol, "SurfaceArea": sa, "SurfaceVolumeRatio": sa / vol, "Sphericity": sph / sa,
           "MajorAxisLength": np.sqrt(ev[2]) * 4, "MinorAxisLength": np.sqrt(ev[1]) * 4, "LeastAxisLength": np.sqrt(ev[0]) * 4,
           "Elongation": np.sqrt(ev[1] / ev[2]), "Flatness": np.sqrt(ev[0] / ev[2])}
    for k, v in ref.items():
        assert float(got[k]) == pytest.approx(v, rel=1e-12, abs=0), k
    assert float(got["VoxelVolume"]) == N * math.prod(SP3)
    for k, q in (("Maximum2DDiameterSlice", 0), ("Maximum2DDiameterColumn", 1), ("Maximum2DDiameterRow", 2),
                 ("Maximum3DDiameter", 3)):
        assert float(got[k]) == o["dia"][q], k


# ---------------------------------------------------------------------------------------------------- compiled reference
def _cshape():
    import build_ref
    try:
        return build_ref.load("_cshape")
    except ImportError as e:
        pytest.fail(f"the compiled reference _cshape is missing ({e}); build() compiles it into oracle/_ref/")


def test_compiled_reference_on_non_dyadic_spacings():
    """meshes of up to ~4e4 vertices (the reference's O(V^2) loop takes seconds): diameters bit-identical, area and
    volume within the sum of both implementations' bounds (each: its summation depth plus per-term rounding)"""
    ref = _cshape()
    rng = np.random.default_rng(8)
    z, y, x = np.ogrid[:70, :80, :90]
    ell = (((z - 34.5) / 33) ** 2 + ((y - 39.5) / 37) ** 2 + ((x - 44.5) / 42) ** 2 < 1) & (rng.random((70, 80, 90)) > 0.01)
    cases = {"ellipsoid_70x80x90": (np.pad(ell, 1), (2.1, 0.7, 1.3)),
             "noise_32x30x28": (rng.random((32, 30, 28)) < 0.4, (0.83, 1.17, 2.9))}
    worst_v = 0
    for name, (m, sp) in cases.items():
        o = S.mesh(m, sp)
        assert not o["exact"]
        t = time.perf_counter()
        r = ref.calculate_coefficients(m.astype(np.int8), np.array(sp))
        t = time.perf_counter() - t
        k = cshape.calculate_coefficients(m, np.array(sp))
        assert list(k[2]) == list(r[2]) == o["dia"], name
        g, tpt, dg, tiles = _launch3d(m.shape, o["n_verts"])
        n = o["n_tri"]
        ba = S.sum_bound(tpt + 8 + g, o["area_fsum"], o["area_mag"], 4) + S.sum_bound(n, o["area_fsum"], 2 * o["area_mag"], 4)
        bv = (S.sum_bound(tpt + 8 + g, o["vol_terms_abs"], o["vol_mag"], 8)
              + S.sum_bound(n, o["vol_terms_abs"], 2 * o["vol_mag"], 8)) / 6
        assert abs(k[0] - r[0]) <= ba and abs(k[1] - r[1]) <= bv, (name, k, r, ba, bv)
        worst_v = max(worst_v, o["n_verts"])
        print(f"\n{name}: {o['n_verts']} vertices (reference {t:.1f} s); area err/bound {abs(k[0] - r[0]) / ba:.3g}, "
              f"volume err/bound {abs(k[1] - r[1]) / bv:.3g}")
    rng = np.random.default_rng(9)
    yy, xx = np.ogrid[:300, :260]
    cases2 = {"noise_200x180": (np.pad(rng.random((200, 180)) < 0.5, 1), (2.1, 0.7)),
              "disc_300x260": (np.pad(((yy - 149.5) / 140) ** 2 + ((xx - 129.5) / 125) ** 2 < 1, 1), (0.83, 1.17))}
    for name, (m, sp) in cases2.items():
        o = S.mesh2d(m, sp)
        r = ref.calculate_coefficients2D(m.astype(np.int8), np.array(sp))
        k = cshape.calculate_coefficients2D(m, np.array(sp))
        assert k[2] == r[2] == o["dia"], name
        nseg = o["n_diag"] + o["n_x"] + o["n_y"]
        g, tpt, _, _ = _launch2d(m.shape, o["n_verts"])
        pmax = float(np.hypot(m.shape[0] * sp[0], m.shape[1] * sp[1]))
        bp = S.sum_bound(tpt + 8 + g + nseg, o["per_fsum"]) + 6 * U * pmax * nseg
        assert abs(k[0] - r[0]) <= bp, (name, k, r, bp)
        exact_sur = o["eighths"] * 0.125 * sp[0] * sp[1]
        assert k[1] == ((o["eighths"] * 0.125) * sp[0]) * sp[1]
        bs = S.sum_bound(nseg + 5, o["cross_mag"]) / 2 + 3 * U * exact_sur     # the reference's signed-cross sum
        assert abs(r[1] - exact_sur) <= bs, (name, r[1], exact_sur, bs)
        worst_v = max(worst_v, o["n_verts"])
        print(f"{name}: {o['n_verts']} vertices; perimeter err/bound {abs(k[0] - r[0]) / bp:.3g}, "
              f"reference surface err/bound {abs(r[1] - exact_sur) / bs:.3g}")
    print(f"largest mesh against the compiled reference: {worst_v} vertices")


# ---------------------------------------------------------------------------------------------------- C ABI
def _host_call3d(view, sp):
    import ctypes as C
    base = np.ascontiguousarray(np.asarray(sp, np.float64))
    size = np.array(view.shape, np.int32)
    strides = np.array([s // view.itemsize for s in view.strides], np.int32)
    sa, vol, dia = C.c_double(), C.c_double(), (C.c_double * 4)()
    assert lib().rb_calculate_coefficients(ptr(view), ptr(size), ptr(strides), ptr(base), C.byref(sa), C.byref(vol), dia) == 0
    return sa.value, vol.value, tuple(dia)


def _host_call2d(view, sp):
    import ctypes as C
    base = np.ascontiguousarray(np.asarray(sp, np.float64))
    size = np.array(view.shape, np.int32)
    strides = np.array([s // view.itemsize for s in view.strides], np.int32)
    per, sur, dia = C.c_double(), C.c_double(), C.c_double()
    assert lib().rb_calculate_coefficients2D(ptr(view), ptr(size), ptr(strides), ptr(base), C.byref(per), C.byref(sur),
                                             C.byref(dia)) == 0
    return per.value, sur.value, dia.value


def test_host_entry_points_gather_strided_views():
    """rb_calculate_coefficients / rb_calculate_coefficients2D on step slices, transposes and reversed views give what
    the contiguous copy gives (diameters bit for bit, area / volume / perimeter within two runs' bounds)"""
    rng = np.random.default_rng(10)
    base = (rng.random((70, 80, 90)) < 0.5).astype(np.int8)
    for view in (base[::2, 1::3, ::2], base.transpose(2, 0, 1), base[::-1, :, ::-3], base[5:60:3].transpose(1, 2, 0)):
        assert not view.flags.c_contiguous
        got, want = _host_call3d(view, SP3), _host_call3d(np.ascontiguousarray(view), SP3)
        o = S.mesh(np.ascontiguousarray(view), SP3)
        g, tpt, _, _ = _launch3d(view.shape, o["n_verts"])
        assert got[2] == want[2] == tuple(o["dia"])
        _check_sums3d("strided view", got[0], got[1], o, tpt + 8 + g, [])
        _check_sums3d("contiguous copy", want[0], want[1], o, tpt + 8 + g, [])
    base2 = (rng.random((300, 400)) < 0.5).astype(np.int8)
    for view in (base2[::2, 1::3], base2.T, base2[::-1, ::-2]):
        got, want = _host_call2d(view, SP2), _host_call2d(np.ascontiguousarray(view), SP2)
        o = S.mesh2d(np.ascontiguousarray(view), SP2)
        assert got[1] == want[1] and got[2] == want[2] == o["dia"]
        g, tpt, _, _ = _launch2d(view.shape, o["n_verts"])
        assert abs(got[0] - o["per_fsum"]) <= S.sum_bound(tpt + 8 + g, o["per_fsum"]) + U * o["per_fsum"]


def _stream_case():
    """a mask written on the current stream, then coefficients and moments on it; nothing waits on the host between"""
    g = torch.Generator(device="cuda").manual_seed(12)
    m = (torch.rand((60, 64, 72), generator=g, device="cuda") < 0.5).to(torch.uint8)
    m[:, :, :9] = 0
    return cshape.coefficients_device(m, SP3), cshape.moments_device(m), m.cpu().numpy()


def test_device_entry_points_on_a_side_stream_equal_the_default_stream():
    (a0, v0, d0, n0), mom0, m = _stream_case()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        (a1, v1, d1, n1), mom1, _ = _stream_case()
    assert mom1 == mom0 == _exact_moments(m)
    assert d1 == d0 and n1 == n0
    o = S.mesh(m, SP3)
    assert list(d0) == o["dia"] and n0 == o["n_verts"]
    g, tpt, _, _ = _launch3d(m.shape, o["n_verts"])
    for a, v in ((a0, v0), (a1, v1)):
        _check_sums3d("stream", a, v, o, tpt + 8 + g, [])
