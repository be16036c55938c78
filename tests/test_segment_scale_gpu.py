"""Segment-mode matrices (one GLCM / GLDM / NGTDM / GLRLM / GLSZM per ROI) at sizes where every block of every kernel
loops: the tile kernel walks several 4x8x64 tiles per block (TMA prefetch of the next box, mbarrier phase flip,
cooperative restage into the other buffer, shared-memory histograms carried across tiles), and the grid-stride kernels
(direct texture kernel, run-end GLRLM, union-find GLSZM labelling) sweep their volume several times.

Every input is compared, matrix by matrix, with the C oracle (integer entries bit for bit), through the host API and the
device-resident entry points (bit-identical to each other and to a second call). NGTDM's s_i is also compared with an
exact rational restatement. Every case also shows, from the dispatch rules restated below, which kernel builds its
matrices and that the grid of each kernel is at most a third of its work items. The last test runs one case of the
batch-of-cases benchmark (64 independent 256^3 cases) through the plugin classes and compares every feature with the
oracle pipeline."""
from fractions import Fraction

import numpy as np
import pytest
import scipy.ndimage as ndi
import torch

import cmatrices_oracle as O
import pipeline as PL
from pyradiomics_b200 import cmatrices as B, featureclasses as FC, voxel

pytestmark = pytest.mark.gpu

ALPHA = 1                                       # GLDM's dependence threshold in the matrix cases
TILE_TMA, TILE_COOP = "seg_tile_kernel<true>", "seg_tile_kernel<false>"
DIRECT8, DIRECT16 = "seg_direct_kernel<unsigned char>", "seg_direct_kernel<unsigned short>"


# ---------------------------------------------------------------------------------------------------- seeded volumes
def _iid(shape, Ng, keep, seed):
    """i.i.d. levels 1..Ng, each voxel in the ROI with probability `keep`"""
    rng = np.random.default_rng(seed)
    lev = rng.integers(1, Ng + 1, shape).astype(np.int32)
    msk = rng.random(shape) < keep if keep < 1 else np.ones(shape, bool)
    return lev, msk


def _smooth_with_holes(shape, Ng, seed):
    """a smoothed noise field quantised to Ng levels; the ROI loses smooth blobs (~15 %) and 2 % scattered voxels"""
    rng = np.random.default_rng(seed)
    f = ndi.gaussian_filter(rng.normal(size=shape), 4.0)
    lev = (1 + np.floor((f - f.min()) / (f.max() - f.min()) * Ng).clip(0, Ng - 1)).astype(np.int32)
    h = ndi.gaussian_filter(rng.normal(size=shape), 3.0)
    msk = (h > np.quantile(h, 0.15)) & (rng.random(shape) > 0.02)
    return lev, msk


def _blocky_lines(shape, Ng, seed, block=8):
    """levels constant on block^nd cubes, crossed by whole lines of one level along every axis and the main diagonal:
    runs reach the full length of each axis, most runs are longer than 4, and the lines join into one zone that spans the
    volume; the whole volume is the ROI"""
    rng = np.random.default_rng(seed)
    lev = rng.integers(1, Ng + 1, [-(-s // block) for s in shape])
    for ax in range(len(shape)):
        lev = np.repeat(lev, block, axis=ax)
    lev = np.ascontiguousarray(lev[tuple(slice(0, s) for s in shape)]).astype(np.int32)
    g = max(1, Ng // 2)
    if len(shape) == 3:
        lev[2::11, 4::13, :] = g
        lev[2::11, :, 6::19] = g
        lev[:, 4::13, 6::19] = g
        k = np.arange(min(shape))
        lev[k, k, k] = g
    else:
        lev[4::13, :] = g
        lev[:, 6::19] = g
        k = np.arange(min(shape))
        lev[k, k] = g
    return lev, np.ones(shape, bool)


def _config5ii_levels(k=0, n=256):
    """the gray levels of case k of the batch-of-cases benchmark (bench.py secondary_config5ii): i.i.d. 1..32 from a CUDA
    generator seeded 1000 + k; its raw image is (levels - 1) * 25 + 3, which binWidth 25 bins back to these levels"""
    g = torch.Generator(device="cuda").manual_seed(1000 + k)
    return torch.randint(1, 33, (n, n, n), generator=g, device="cuda", dtype=torch.int16)


# name: (volume, Ng, distances, force2Ddimension or None, texture kernel).  The texture kernel is one name, or a pair
# (the host API's GLCM call, its GLDM / NGTDM calls and the fused device pass) when only the GLCM plan fits the tile kernel.
CASES = {
    # seg_tile_kernel staged by TMA; each of these also runs with B200_SEG_TMA=0 (cooperative staging)
    "tma_iid32_1024_tiles": (lambda: _iid((64, 128, 256), 32, 0.8, 1), 32, [1], None, TILE_TMA),
    "tma_ragged_smooth_holes_d12": (lambda: _smooth_with_holes((66, 123, 144), 32, 2), 32, [1, 2], None, TILE_TMA),
    "tma_ng48_one_block_per_sm": (lambda: _iid((64, 128, 256), 48, 0.8, 3), 48, [1], None, TILE_TMA),
    "tma_d123_glcm_in_global_memory": (lambda: _iid((42, 70, 528), 24, 0.8, 4), 24, [1, 2, 3], None, TILE_TMA),
    "tma_2d_2048_d123": (lambda: _iid((2048, 2048), 32, 0.8, 5), 32, [1, 2, 3], None, TILE_TMA),
    "tma_force2d_dim0": (lambda: _blocky_lines((64, 128, 256), 32, 6), 32, [1], 0, TILE_TMA),
    "tma_force2d_dim2": (lambda: _blocky_lines((64, 128, 256), 32, 6), 32, [1], 2, TILE_TMA),
    # seg_tile_kernel staged cooperatively: by shape (X % 16 != 0), or by a level tensor that is not 16-byte aligned
    "coop_x_not_multiple_of_16": (lambda: _iid((67, 125, 250), 32, 0.8, 7), 32, [1], None, TILE_COOP),
    "coop_misaligned_device_levels": (lambda: _iid((64, 128, 256), 32, 0.8, 8), 32, [1], None, TILE_TMA),
    # seg_direct_kernel: 16-bit levels; GLDM / NGTDM histograms beyond shared memory; offsets beyond 3 (GLCM privatised)
    "direct_16bit_ng300": (lambda: _iid((64, 128, 256), 300, 0.8, 9), 300, [1], None, DIRECT16),
    "direct_ng200_d123": (lambda: _iid((42, 70, 528), 200, 0.8, 10), 200, [1, 2, 3], None, (TILE_TMA, DIRECT8)),
    "direct_2d_d14_glcm_privatised": (lambda: _iid((1024, 1024), 24, 0.8, 11), 24, [1, 4], None, DIRECT8),
    # GLRLM: full-length runs, the global long-run histogram; 16-bit levels without the shared short-run histogram;
    # a sparse ROI (long walk-backs, the "line holds two voxels" rule); 2-D
    "blocky_lines": (lambda: _blocky_lines((64, 128, 256), 32, 12), 32, [1], None, TILE_TMA),
    "blocky_lines_16bit_ng600": (lambda: _blocky_lines((32, 128, 256), 600, 13), 600, [1], None, DIRECT16),
    "sparse_roi_5pct_128": (lambda: _iid((128, 128, 128), 4, 0.05, 14), 4, [1], None, TILE_TMA),
    "blocky_lines_2d_2048": (lambda: _blocky_lines((2048, 2048), 8, 15), 8, [1], None, TILE_TMA),
    # GLSZM: many small zones at 256^3 (the benchmark's case 0); a percolating zone of ~1 M voxels; one zone of 2 M
    "config5ii_case0_256": (lambda: ((_config5ii_levels().cpu().numpy()).astype(np.int32), np.ones((256,) * 3, bool)),
                            32, [1], None, TILE_TMA),
    "percolating_ng2_128": (lambda: _iid((128, 128, 128), 2, 1.0, 16), 2, [1], None, TILE_TMA),
    "one_zone_ng1_128": (lambda: (np.ones((128, 128, 128), np.int32), np.ones((128, 128, 128), bool)), 1, [1], None, TILE_TMA),
}


# ---------------------------------------------------------------------------------------------------- launch geometry
# The dispatch of segment_kernels.cu (segment_matrices, tile_plan, launch_tile, launch_direct, segment_glrlm, and the
# GLSZM labelling in segment_glszm), restated: which kernel builds a matrix and with how many blocks.
# (torch.profiler does record these kernels, but over the many sessions of one test process it lost kernel records of
# some sessions on an H100, so the launches are computed from the same rules instead of read back.)
def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _grid_for(n, per_sm):
    """common.cuh grid_for(n, 256, per_sm): 256-thread blocks, one item per thread, at most per_sm blocks per SM"""
    return max(1, min(-(-n // 256), _sms() * per_sm))


def _tiles(shape):
    """seg_tile_kernel's work items: tiles of tz x ty x ST_TX = 4 x 8 x 64 voxels, 1 x 32 x 64 in 2-D (tile_plan)"""
    Z, Y, X = (1,) * (3 - len(shape)) + tuple(shape)
    tz, ty = (1, 32) if Z == 1 else (4, 8)
    return -(-X // 64) * -(-Y // ty) * -(-Z // tz)


def _texture_launch(shape, level_bytes, dist, f2, f2d, Ng, flags, tma):
    """(kernel, blocks, work items) of one segment_matrices call; flags 1 = GLCM, 2 = GLDM, 4 = NGTDM; `tma`: the
    level tensor admits a tensor map (B200_SEG_TMA not 0, 16-byte aligned data pointer)"""
    ang = O.generate_angles(shape, dist, 0, f2, f2d)
    na, H = len(ang), int(np.abs(ang).max())
    n = int(np.prod(shape))
    smem = 0
    if level_bytes == 1 and H <= 3 and na <= 172:             # tile_plan: two staged boxes of ST_BX = 96 bytes per row
        tz, ty = (1, 32) if len(shape) == 2 else (4, 8)
        box = (96 * (ty + 2 * H) * (tz + 2 * H) + 127) & ~127
        smem = 2 * box + (Ng * (2 * na + 2) * 8 if flags & 4 else 0) + (Ng * (4 * na + 1) * 4 if flags & 2 else 0)
        if flags & 1 and smem + Ng * Ng * na * 4 <= 200 * 1024:           # GLCM histogram in shared memory
            smem += Ng * Ng * na * 4
        smem = 0 if smem > 220 * 1024 else smem
    if smem:                                                   # launch_tile: one block per SM above 110 KB, else two
        kernel = TILE_TMA if tma and shape[-1] % 16 == 0 else TILE_COOP
        return kernel, min(_tiles(shape), _sms() * (1 if smem > 110 * 1024 else 2)), _tiles(shape)
    privatised = flags & 1 and Ng * Ng * na * 4 <= 160 * 1024   # launch_direct: GLCM in shared memory, one block per SM
    return DIRECT8 if level_bytes == 1 else DIRECT16, _grid_for(n, 1 if privatised else 8), -(-n // 256)


def _assert_launches(expect, shape, level_bytes, dist, f2, f2d, Ng, tma):
    """each texture call ({call: kernel}; "texture" = the fused device pass) runs the kernel `expect` names with at most a
    third as many blocks as work items, and so do seg_glrlm_ends_kernel and ccl_merge_kernel (grid_for(n, 256, 8))"""
    for call, flags in (("glcm", 1), ("gldm", 2), ("ngtdm", 4), ("texture", 7)):
        if call in expect:
            kernel, blocks, work = _texture_launch(shape, level_bytes, dist, f2, f2d, Ng, flags, tma[call])
            assert kernel == expect[call], (call, kernel, expect[call])
            assert 3 * blocks <= work, (call, kernel, blocks, work)
    n = int(np.prod(shape))
    assert 3 * _grid_for(n, 8) <= -(-n // 256), (n, _sms())


# ---------------------------------------------------------------------------------------------------- matrices
def _host_calls(lev, msk, Ng, dist, f2, f2d, texture_only=False):
    calls = {"glcm": lambda: B.calculate_glcm(lev, msk, dist, Ng, f2, f2d),
             "gldm": lambda: B.calculate_gldm(lev, msk, dist, Ng, ALPHA, f2, f2d),
             "ngtdm": lambda: B.calculate_ngtdm(lev, msk, dist, Ng, f2, f2d)}
    if not texture_only:
        calls["glrlm"] = lambda: B.calculate_glrlm(lev, msk, Ng, max(lev.shape), f2, f2d)
        calls["glszm"] = lambda: B.calculate_glszm(lev, msk, Ng, int(msk.sum()), f2, f2d)
    return calls


def _device_calls(levd, Ng, dist, f2, f2d, texture_only=False):
    calls = {"texture": lambda: B.segment_texture_device(levd, dist, Ng, ALPHA, f2, f2d)}      # GLCM + GLDM + NGTDM, one pass
    if not texture_only:
        calls["glrlm"] = lambda: B.calculate_glrlm_device(levd, Ng, max(levd.shape), f2, f2d)
        calls["glszm"] = lambda: B.calculate_glszm_device(levd, Ng, f2, f2d)
    return calls


def _run(calls):
    """{matrix: array} of every call"""
    out = {}
    for call, fn in calls.items():
        r = fn()
        if call == "texture":
            out.update(glcm=r["glcm"][0], glcm_angles=r["glcm"][1], gldm=r["gldm"], ngtdm=r["ngtdm"])
        elif call in ("glcm", "glrlm"):
            out[call], out[call + "_angles"] = r
        else:
            out[call] = r
    return out


def _oracle(lev, msk, Ng, dist, f2, f2d):
    P, ang = O.calculate_glcm(lev, msk, dist, Ng, f2, f2d)
    R, ang_r = O.calculate_glrlm(lev, msk, Ng, max(lev.shape), f2, f2d)
    return {"glcm": P, "glcm_angles": ang, "gldm": O.calculate_gldm(lev, msk, dist, Ng, ALPHA, f2, f2d),
            "ngtdm": O.calculate_ngtdm(lev, msk, dist, Ng, f2, f2d), "glrlm": R, "glrlm_angles": ang_r,
            "glszm": O.calculate_glszm(lev, msk, Ng, int(msk.sum()), f2, f2d)}


def _assert_identical(a, b, what):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), (what, k)


def _assert_matches_oracle(got, ref):
    for k, r in ref.items():
        g = got[k]
        assert g.shape == r.shape, (k, g.shape, r.shape)
        if k == "ngtdm":          # n_i, level exact; s_i: the oracle sums a double per voxel (see _assert_ngtdm_exact)
            assert np.array_equal(g[..., [0, 2]], r[..., [0, 2]])
            assert np.allclose(g[..., 1], r[..., 1], rtol=1e-12, atol=1e-12)
        else:
            assert np.array_equal(g, r), k


def _ngtdm_exact(lev, msk, Ng, dist, f2, f2d):
    """segment NGTDM restated in integers: (n_i, exact s_i as Fractions, ncnt).  s_i = sum_c T[g][c] / c, where T[g][c]
    sums |g * c - (sum of the c ROI neighbours)| over the ROI voxels of level g with c ROI neighbours, c = 1..ncnt"""
    ang = O.generate_angles(lev.shape, dist, 1, f2, f2d)      # both directions of every offset
    ncnt = len(ang)
    L = np.where(msk, lev, 0).astype(np.int32)
    cnt = np.zeros(L.shape, np.int16)
    tot = np.zeros(L.shape, np.int32)
    for off in ang:
        nb = L[tuple(slice(max(o, 0), s + min(o, 0)) for o, s in zip(off, L.shape))]     # the neighbour p + off ...
        at = tuple(slice(max(-o, 0), s - max(o, 0)) for o, s in zip(off, L.shape))      # ... of every p that has one
        cnt[at] += nb > 0
        tot[at] += nb
    g, c = L[msk].astype(np.int64), cnt[msk].astype(np.int64)
    d = np.abs(g * c - tot[msk])
    assert int(d.sum()) < 2 ** 53                                  # the float64 bincount below sums integers exactly
    T = np.rint(np.bincount((g - 1) * (ncnt + 1) + c, weights=d, minlength=Ng * (ncnt + 1))).astype(np.int64)
    T = T.reshape(Ng, ncnt + 1).tolist()
    s = [sum((Fraction(t, k) for k, t in enumerate(row) if t), Fraction(0)) for row in T]
    return np.bincount(g - 1, minlength=Ng), s, ncnt


def _assert_ngtdm_exact(P, lev, msk, Ng, dist, f2, f2d):
    """n_i exact and s_i within (ncnt + 1) * 2^-53 relative of the exact s_i: the GPU divides its integer accumulators
    once per count c and sums the ncnt quotients in double"""
    n, s, ncnt = _ngtdm_exact(lev, msk, Ng, dist, f2, f2d)
    assert np.array_equal(P[0, :, 0], n)
    assert np.array_equal(P[0, :, 2], np.arange(1, Ng + 1))
    tol = Fraction(ncnt + 1, 2 ** 53)
    for gi, exact in enumerate(s):
        assert abs(Fraction(float(P[0, gi, 1])) - exact) <= tol * exact, (gi, float(P[0, gi, 1]), float(exact))


def _device_levels(lev, msk, Ng, misalign=False):
    levd, _ = voxel.pack_levels(torch.as_tensor(lev).cuda(), torch.as_tensor(msk).cuda(), Ng)
    if not misalign:
        return levd
    # the same packed levels one byte into a larger allocation: a contiguous tensor whose data pointer is not 16-byte
    # aligned, which no tensor map can address
    assert levd.dtype == torch.uint8
    buf = torch.zeros(levd.numel() + 16, dtype=torch.uint8, device=levd.device)
    view = buf[1:1 + levd.numel()].view(levd.shape)
    view.copy_(levd)
    assert view.is_contiguous() and view.data_ptr() % 16 == 1
    return view


@pytest.mark.parametrize("name", list(CASES))
def test_segment_matrices_at_scale_match_oracle(name, monkeypatch):
    volume, Ng, dist, f2d, texture = CASES[name]
    f2, f2d = (True, f2d) if f2d is not None else (False, 0)
    glcm_kernel, fused_kernel = texture if isinstance(texture, tuple) else (texture, texture)
    misalign = name == "coop_misaligned_device_levels"
    expect = {"glcm": glcm_kernel, "gldm": fused_kernel, "ngtdm": fused_kernel,
              "texture": TILE_COOP if misalign else fused_kernel}
    lev, msk = volume()
    monkeypatch.setenv("B200_SEG_TMA", "1")
    levd = _device_levels(lev, msk, Ng, misalign)
    lb = levd.element_size()
    assert lb == (1 if Ng <= 255 else 2)
    tma = {"glcm": True, "gldm": True, "ngtdm": True, "texture": levd.data_ptr() % 16 == 0}
    _assert_launches(expect, lev.shape, lb, dist, f2, f2d, Ng, tma)

    host = _run(_host_calls(lev, msk, Ng, dist, f2, f2d))
    dev = _run(_device_calls(levd, Ng, dist, f2, f2d))
    _assert_matches_oracle(host, _oracle(lev, msk, Ng, dist, f2, f2d))
    _assert_ngtdm_exact(host["ngtdm"], lev, msk, Ng, dist, f2, f2d)
    _assert_identical(dev, host, "device API vs host API")
    _assert_identical(_run(_host_calls(lev, msk, Ng, dist, f2, f2d)), host, "host API, second call")
    _assert_identical(_run(_device_calls(levd, Ng, dist, f2, f2d)), dev, "device API, second call")

    if TILE_TMA in expect.values():       # the same boxes staged by cooperative loads: the same bits
        monkeypatch.setenv("B200_SEG_TMA", "0")
        expect = {k: TILE_COOP if v == TILE_TMA else v for k, v in expect.items()}
        _assert_launches(expect, lev.shape, lb, dist, f2, f2d, Ng, dict.fromkeys(tma, False))
        coop = _run(_host_calls(lev, msk, Ng, dist, f2, f2d, texture_only=True))
        _assert_identical(coop, {k: host[k] for k in coop}, "cooperative staging, host API")
        coop = _run(_device_calls(levd, Ng, dist, f2, f2d, texture_only=True))
        _assert_identical(coop, {k: dev[k] for k in coop}, "cooperative staging, device API")


def test_tile_kernel_equals_direct_kernel_at_scale():
    """levels 1..24 as an 8-bit volume (Ng = 24: tile kernel) and as a 16-bit one (Ng = 300: direct kernel), both looping:
    the leading 24 levels of the Ng = 300 matrices are the Ng = 24 matrices bit for bit, NGTDM s_i included"""
    lev, msk = _iid((64, 128, 256), 24, 0.8, 21)
    dist = [1, 2]
    got = {}
    for Ng, kernel in ((24, TILE_TMA), (300, DIRECT16)):
        levd = _device_levels(lev, msk, Ng)
        expect = dict.fromkeys(("glcm", "gldm", "ngtdm", "texture"), kernel)
        _assert_launches(expect, lev.shape, levd.element_size(), dist, False, 0, Ng, dict.fromkeys(expect, True))
        got[Ng] = (_run(_host_calls(lev, msk, Ng, dist, False, 0, texture_only=True)),
                   _run(_device_calls(levd, Ng, dist, False, 0, texture_only=True)))
    for api in range(2):
        small, big = got[24][api], got[300][api]
        assert np.array_equal(big["glcm"][:, :24, :24], small["glcm"]) and not big["glcm"][:, 24:].any()
        assert not big["glcm"][:, :, 24:].any()
        assert np.array_equal(big["gldm"][:, :24], small["gldm"]) and not big["gldm"][:, 24:].any()
        assert np.array_equal(big["ngtdm"][:, :24], small["ngtdm"]) and not big["ngtdm"][:, 24:, :2].any()


def test_glrlm_nr_below_longest_run_raises():
    """runs of the full x length (256) do not fit Nr = 255: IndexError from the host API and the device entry point, as
    from the oracle"""
    lev, msk = _blocky_lines((64, 128, 256), 32, 12)
    with pytest.raises(IndexError):
        O.calculate_glrlm(lev, msk, 32, 255, False, 0)
    with pytest.raises(IndexError):
        B.calculate_glrlm(lev, msk, 32, 255, False, 0)
    with pytest.raises(IndexError):
        B.calculate_glrlm_device(_device_levels(lev, msk, 32), 32, 255, False, 0)


def test_config5ii_case_features_match_oracle():
    """case 0 of the batch-of-cases benchmark (64 independent 256^3 cases, segment-based full suite), generated as the
    benchmark generates it, through the five plugin classes: every feature within 1e-9 relative of the oracle pipeline"""
    raw = ((_config5ii_levels() - 1) * 25 + 3).cpu().numpy()
    mask = np.ones(raw.shape, np.uint8)
    FC.clear_device_cache()
    for c in PL.CLASS_NAMES:
        got = FC.FEATURE_CLASSES[c](raw, mask, binWidth=25).execute()
        ref = PL.extract(c, raw, mask.astype(bool), binWidth=25)
        assert set(got) == set(ref), (c, set(got) ^ set(ref))
        for f, v in ref.items():
            assert abs(float(got[f]) - v) <= max(1e-9 * abs(v), 1e-12), (c, f, float(got[f]), v)
