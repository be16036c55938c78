"""The GLSZM and GLDM kernelRadius-1 kernels on their full/deferred tile frame (csrc/voxel_fast.cu,
tiles_fast_kernel): the full-window body and the general body against the window oracle and the generic kernel, both
bodies inside one tile, slab / whole-volume bit identity, and the launch rules that make blocks take several tiles and
fill the deferred list."""
import numpy as np
import pytest
import torch

from helpers import FAST_NAMES, GLDM_ALPHAS, compare_window_maps, plant, window_at, window_features
from pyradiomics_b200 import _lib, voxel

pytestmark = pytest.mark.gpu

CLASSES = ("glszm", "gldm")


def _refs(wins, Ng, alphas=GLDM_ALPHAS):
    out = {}
    for cname in CLASSES:
        for a in (alphas if cname == "gldm" else (0,)):
            ref = np.empty((len(FAST_NAMES[cname]), len(wins)))
            for i, w in enumerate(wins):
                f = window_features(w, Ng, cname, a)
                ref[:, i] = [f[n] for n in FAST_NAMES[cname]]
            out[(cname, a)] = ref
    return out


def _settings(vol, Ng, a=0):
    return _lib.make_settings(Ng, len(np.unique(vol[vol > 0])), gldm_a=a)


def _at(out, cen):
    idx = tuple(torch.as_tensor(cen[:, d], device=out.device) for d in range(3))
    return out[(slice(None),) + idx].cpu().numpy()


def _maps(cname, lev, s, generic, monkeypatch, **kw):
    if generic:
        monkeypatch.setenv("B200_RADIOMICS_FORCE_GENERIC", "1")
    try:
        return voxel.voxel_features(cname, lev, s, **kw)
    finally:
        monkeypatch.delenv("B200_RADIOMICS_FORCE_GENERIC", raising=False)


def _single_zero_windows(rng, Ng):
    """full windows, then a single zero at each of the 26 positions other than the centre (a zero centre is no centre)"""
    wins = [rng.integers(1, Ng + 1, 27) for _ in range(40)] + [rng.integers(1, min(Ng, 3) + 1, 27) for _ in range(20)]
    for pos in range(27):
        if pos == 13:
            continue
        for k in range(3):
            w = rng.integers(1, (Ng if k else min(Ng, 3)) + 1, 27)
            w[pos] = 0
            wins.append(w)
    return wins


@pytest.mark.parametrize("Ng", [2, 32, 255])
def test_full_and_general_bodies_against_oracle_and_generic(Ng, monkeypatch):
    rng = np.random.default_rng(500 + Ng)
    wins = _single_zero_windows(rng, Ng)
    vol, cen = plant(wins)
    vol[vol > 0] = np.minimum(vol[vol > 0], Ng)
    refs = _refs(wins, Ng)
    lev = torch.as_tensor(vol.astype(np.uint8)).cuda()
    for cname in CLASSES:
        for a in (GLDM_ALPHAS if cname == "gldm" else (0,)):
            s = _settings(vol, Ng, a)
            for generic in (False, True):
                got = _at(_maps(cname, lev, s, generic, monkeypatch), cen)
                compare_window_maps(got, refs, cname, a, f"Ng={Ng}/gldm_a={a}/{'generic' if generic else 'fast'}", generic)


def _mixed_volume():
    """faces and holes: full and deferred centres side by side in the same tiles"""
    rng = np.random.default_rng(41)
    lev = rng.integers(1, 33, (9, 37, 301)).astype(np.uint8)
    lev[rng.random(lev.shape) < 0.02] = 0
    lev[4, 10:20, 50:90] = 0
    return lev


def test_both_bodies_in_one_tile(monkeypatch):
    lev_np = _mixed_volume()
    Z, Y, X = lev_np.shape
    pad = np.pad(lev_np, 1)
    full = np.ones(lev_np.shape, bool)
    for dz in range(3):
        for dy in range(3):
            for dx in range(3):
                full &= pad[dz:dz + Z, dy:dy + Y, dx:dx + X] != 0
    centre = lev_np != 0
    deferred, fast = (centre & ~full).reshape(-1), (centre & full).reshape(-1)
    for nt in (128, 256):
        t = np.arange(deferred.size) // nt
        mixed = np.bincount(t, deferred) * np.bincount(t, fast) > 0
        assert mixed.sum() > 100, nt
    rng = np.random.default_rng(42)
    cen = np.argwhere(centre)[rng.choice(int(centre.sum()), 300, replace=False)]
    wins = [window_at(lev_np, c) for c in cen]
    refs = _refs(wins, 32, alphas=(0, 3))
    lev = torch.as_tensor(lev_np).cuda()
    for cname in CLASSES:
        for a in ((0, 3) if cname == "gldm" else (0,)):
            s = _lib.make_settings(32, 32, gldm_a=a)
            fast_maps = _maps(cname, lev, s, False, monkeypatch)
            gen_maps = _maps(cname, lev, s, True, monkeypatch)
            compare_window_maps(_at(fast_maps, cen), refs, cname, a, f"mixed/{cname}/{a}", False)
            ok = fast_maps.isnan() == gen_maps.isnan()
            assert bool(ok.all()), cname
            d = (fast_maps - gen_maps).abs().nan_to_num(0)
            assert bool((d <= 1e-9 * gen_maps.abs().nan_to_num(0) + 1e-12).all()), (cname, a, float(d.max()))
            # non-centres hold the init value
            assert bool((fast_maps[:, ~torch.as_tensor(centre).cuda()] == s.initValue).all()), cname


def test_slabs_at_arbitrary_planes_are_bit_identical():
    lev_np = _mixed_volume()
    lev = torch.as_tensor(lev_np).cuda()
    for cname in CLASSES:
        s = _lib.make_settings(32, 32)
        whole = voxel.voxel_features(cname, lev, s).nan_to_num(nan=-7.0)
        for cuts in ((0, 1, 9), (0, 3, 4, 8, 9), (0, 5, 9)):
            parts = [voxel.voxel_features(cname, lev, s, z0=a, z1=b) for a, b in zip(cuts[:-1], cuts[1:])]
            assert torch.equal(torch.cat(parts, 1).nan_to_num(nan=-7.0), whole), (cname, cuts)


# ------------------------------------------------------------------------------------------------------------ launch
SCALE_SHAPE = (7, 1024, 1024)
# (threads per block, resident blocks per SM) of tiles_fast_kernel: 120 / 128 registers (ptxas, sm_90a)
TILE_LAUNCH = {"glszm": (128, 4), "gldm": (256, 2)}


def _tile_launch_rules(shape, sms):
    """restated from voxel_fast.cu: a resident grid (at most one wave) of NT-voxel tiles, tile b, b + grid, ... to
    block b; per class the fewest tiles any block takes and the most entries any block's deferred list holds before
    it drains NT of them (full_window_tiles, voxel_tiles.cuh) on a volume whose every voxel is a centre"""
    Z, Y, X = shape
    total = Z * Y * X
    z, rem = np.divmod(np.arange(total), Y * X)
    y, x = np.divmod(rem, X)
    deferred = (z == 0) | (z == Z - 1) | (y == 0) | (y == Y - 1) | (x == 0) | (x == X - 1)
    out = {}
    for cname, (nt, per_sm) in TILE_LAUNCH.items():
        ntiles = -(-total // nt)
        grid = max(1, min(ntiles, sms * per_sm))
        per_tile = np.bincount(np.arange(total) // nt, deferred, minlength=ntiles).astype(int)
        fill = 0
        for b in range(grid):
            nd = 0
            for c in per_tile[b::grid]:
                nd += c
                fill = max(fill, nd)
                if nd >= nt:
                    nd -= nt
        out[cname] = dict(nt=nt, min_tiles=ntiles // grid, max_fill=fill)
    return out


def test_launch_rules_at_scale():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rules = _tile_launch_rules(SCALE_SHAPE, sms)
    for cname, r in rules.items():
        assert r["min_tiles"] >= 3, (cname, r)
        assert r["max_fill"] >= r["nt"], (cname, r)
