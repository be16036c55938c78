"""The kernelRadius-1 fast voxel kernels (csrc/voxel_fast.cu: GLCM phase A + MCC eigen-tasks, GLRLM, GLSZM, GLDM, NGTDM)
against the window oracle (tests/helpers.py: window_features, window_mcc) on the GPU:

(a) planted corpora -- volumes whose 3x3x3 blocks are seeded, structured and adversarial windows, their levels sent into
    1..Ng for Ng in {2, 3, 32, 33, 128, 254, 255} -- through the fast dispatch and through the generic kernels;
(b) the per-Ng GLCM table cache across runs of different level counts;
(c) two (7, 1024, 1024) volumes at which every block of these kernels takes several tiles and the GLCM eigen-task queue
    runs in z-chunks, against the oracle on sampled centres and against the generic kernel on the whole volume.
MCC is held to 1e-9 absolute on both paths, every other feature to 1e-9 relative (helpers.window_bound states the
exceptions).  That the corpus reaches every eigen-task class is shown on the CPU (test_fast_voxel_windows_cpu.py)."""
import numpy as np
import pytest
import torch

from helpers import (FAST_NAMES, GLDM_ALPHAS, MCC_ATOL, assert_within_window_bounds, compare_window_maps, ng_corpus, plant,
                     planted_corpus, window_at, window_mcc, window_references)
from pyradiomics_b200 import _lib, voxel

pytestmark = pytest.mark.gpu

NGS = (2, 3, 32, 33, 128, 254, 255)
N_BASE = 10500
N_CORPUS = {32: N_BASE, 255: N_BASE}     # every planted centre is checked for MCC; 3 000 windows at the other Ng
N_ORACLE = {32: 2000, 255: 2000}         # centres checked for the other features (the oracle's ~5 ms per window)


def _solver_kind(per):
    """the largest eigen-task of a window (mcc_angle results per slot): 0 none, else its node count"""
    return max([r[1] for r in per if r is not None and r[2] and not r[3] and r[1] > 1] or [0])


KINDS = {"dense <= 8": (2, 8), "dense 9-12": (9, 12), "Lanczos 13-18": (13, 18), "no task": (0, 0)}


@pytest.fixture(scope="module")
def cases():
    base = planted_corpus(N_BASE, seed=0)
    mcc0, kind0 = [], []
    for w in base:
        m, per = window_mcc(w)
        mcc0.append(m)
        kind0.append(_solver_kind(per))
    cache = {}

    def get(Ng):
        if Ng not in cache:
            rng = np.random.default_rng(100 + Ng)
            wins, kept = ng_corpus(base, Ng, N_CORPUS.get(Ng, 3000), rng)
            mcc, kind = [], []
            for w, k in zip(wins, kept):
                if k >= 0:
                    mcc.append(mcc0[k]); kind.append(kind0[k])
                else:
                    m, per = window_mcc(w)
                    mcc.append(m); kind.append(_solver_kind(per))
            vol, cen = plant(wins)
            m = N_ORACLE.get(Ng, 500)
            cache[Ng] = dict(wins=wins, mcc=np.array(mcc), kind=np.array(kind), vol=vol, cen=cen,
                             refs=window_references(wins[:m], Ng, mcc[:m]))
        return cache[Ng]
    return get


def _settings(vol, Ng, a=0):
    return _lib.make_settings(Ng, len(np.unique(vol[vol > 0])), gldm_a=a)


def _at(out, cen):
    idx = tuple(torch.as_tensor(cen[:, d], device=out.device) for d in range(3))
    return out[(slice(None),) + idx].cpu().numpy()


def _check_mcc(got, mcc, kind, what):
    """MCC of every planted centre within MCC_ATOL; the worst error per solver kind goes into the message"""
    err = np.abs(got - mcc)
    assert np.array_equal(np.isnan(got), np.isnan(mcc)), what
    err = np.where(np.isnan(mcc), 0.0, err)
    per = {name: (float(err[(kind >= lo) & (kind <= hi)].max(initial=0)), int(((kind >= lo) & (kind <= hi)).sum()))
           for name, (lo, hi) in KINDS.items()}
    print(what, "MCC worst |error| (windows) per largest eigen-task:", per)
    assert err.max() <= MCC_ATOL, (what, per)
    return per


@pytest.mark.parametrize("path", ["fast", "generic"])
@pytest.mark.parametrize("Ng", NGS)
def test_planted_windows_against_window_oracle(Ng, path, cases, monkeypatch):
    c = cases(Ng)
    vol, cen = c["vol"], c["cen"]
    assert vol.max() == Ng and vol[tuple(cen.T)].min() > 0
    if path == "generic":
        monkeypatch.setenv("B200_RADIOMICS_FORCE_GENERIC", "1")
    lev = torch.as_tensor(vol.astype(np.uint8)).cuda()
    for cname, names in FAST_NAMES.items():
        for a in (GLDM_ALPHAS if cname == "gldm" else (0,)):
            out = voxel.voxel_features(cname, lev, _settings(vol, Ng, a))
            got = _at(out, cen)
            what = f"Ng={Ng}/{path}/gldm_a={a}"
            worst = compare_window_maps(got, c["refs"], cname, a, what, path == "generic")
            print(what, cname, "worst |error| / bound:", {f: f"{v:.2g}" for f, v in worst.items() if v > 1e-3})
            if cname == "glcm":
                _check_mcc(got[names.index("MCC")], c["mcc"], c["kind"], what)
            if path == "fast" and Ng == 255 and cname in ("glcm", "ngtdm"):
                # a centres mask: the planted centres see exactly their own blocks either way
                centers = torch.zeros(lev.shape, dtype=torch.uint8, device=lev.device)
                centers[tuple(torch.as_tensor(cen[:, d]).cuda() for d in range(3))] = 1
                masked = voxel.voxel_features(cname, lev, _settings(vol, Ng), centers=centers)
                assert np.array_equal(_at(masked, cen), got, equal_nan=True), cname


def test_glcm_table_cache_across_level_counts(cases):
    """the per-Ng GLCM table block (device_table keyed by Ng): 255, then 32, then 255 again in one process"""
    runs = []
    for Ng in (255, 32, 255):
        c = cases(Ng)
        lev = torch.as_tensor(c["vol"].astype(np.uint8)).cuda()
        runs.append(voxel.voxel_features("glcm", lev, _settings(c["vol"], Ng)).nan_to_num(nan=-7.0))
        torch.cuda.synchronize()
    assert torch.equal(runs[0], runs[2])


# ------------------------------------------------------------------------------------------------------------ (c) scale
SCALE_SHAPE = (7, 1024, 1024)
THREADS_PER_SM = 2048                     # H100: a resident grid never holds more than this per SM


def _launch_rules(shape, sms):
    """restated from voxel_fast.cu's launch code: the GLCM queue's z-chunks, and the fewest tiles (or grid-stride
    steps) any block of each kernel takes"""
    Z, Y, X = shape
    plane = Y * X
    total = Z * plane
    zchunk = min(max((48 << 20) // (plane * 13), 1), Z)                 # glcm_fast_launch: max_entries / (plane * GF_NA)
    chunks = [min(zchunk, Z - z) for z in range(0, Z, zchunk)]

    def grid_for(n, block, per_sm):                                     # common.cuh
        return max(1, min(-(-n // block), sms * per_sm))

    def min_tiles(n, block, grid):
        return (-(-n // block)) // grid

    resident = lambda n, nt: grid_for(n, nt, THREADS_PER_SM // nt)      # resident_grid: at most one wave
    tiles = {
        "glcm phase A": min(min_tiles(c * plane, 512, resident(c * plane, 512)) for c in chunks),
        "ngtdm": min_tiles(total, 128, resident(total, 128)),
        "glrlm": min_tiles(total, 128, grid_for(total, 128, 32)),
        "glszm": min_tiles(total, 128, grid_for(total, 128, 32)),
        "gldm": min_tiles(total, 256, grid_for(total, 256, 16)),
    }
    return chunks, tiles


def _scale_volume(kind):
    rng = np.random.default_rng(31)
    if kind == "uniform":
        return rng.integers(1, 33, SCALE_SHAPE).astype(np.uint8), 32
    zz, yy, xx = np.meshgrid(*[np.arange(s, dtype=np.float64) for s in SCALE_SHAPE], indexing="ij", sparse=True)
    f = np.sin(zz / 2.7) + np.cos(yy / 3.1) + np.sin(xx / 2.3 + 1) + 0.25 * rng.normal(size=SCALE_SHAPE)
    lev = np.digitize(f, np.quantile(f, np.linspace(0, 1, 256)[1:-1])) + 1
    return lev.astype(np.uint8), 255


def _sample_centres(shape, chunks, rng, n=2000):
    """a quarter on faces / edges / corners, a quarter on the planes either side of each queue-chunk boundary, the rest
    anywhere"""
    Z, Y, X = shape
    c = np.stack([rng.integers(0, s, n) for s in shape], 1)
    q = n // 4
    for i in range(q):                                  # snap 1..3 coordinates onto a face
        for d in rng.choice(3, int(rng.integers(1, 4)), replace=False):
            c[i, d] = 0 if rng.random() < 0.5 else shape[d] - 1
    cuts = np.cumsum(chunks)[:-1]
    band = np.concatenate([cuts - 1, cuts])
    c[q:2 * q, 0] = rng.choice(band, q)
    return c


@pytest.fixture(scope="module")
def scale_case():
    cache = {}

    def get(kind):
        if kind not in cache:
            lev, Ng = _scale_volume(kind)
            sms = torch.cuda.get_device_properties(0).multi_processor_count
            chunks, tiles = _launch_rules(lev.shape, sms)
            cen = _sample_centres(lev.shape, chunks, np.random.default_rng(7))
            wins = [window_at(lev, c) for c in cen]
            cache[kind] = dict(lev=lev, Ng=Ng, chunks=chunks, tiles=tiles, cen=cen, wins=wins,
                               refs=window_references(wins, Ng, alphas=(0,)))
        return cache[kind]
    return get


@pytest.mark.parametrize("kind", ["uniform", "smooth"])
def test_scale_against_oracle_generic_and_itself(kind, scale_case, monkeypatch):
    c = scale_case(kind)
    lev_np, Ng = c["lev"], c["Ng"]
    assert c["chunks"] == [3, 3, 1], c["chunks"]
    assert min(c["tiles"].values()) >= 3, c["tiles"]
    lev = torch.as_tensor(lev_np).cuda()
    s = _settings(lev_np, Ng)
    cen = c["cen"]
    for cname, names in FAST_NAMES.items():
        fast = voxel.voxel_features(cname, lev, s)
        worst = compare_window_maps(_at(fast, cen), c["refs"], cname, 0, f"{kind}/fast", False)
        print(kind, cname, "fast, worst |error| / bound:", {f: f"{v:.2g}" for f, v in worst.items() if v > 1e-3})
        # bit-identical on a second run, and over z-slabs cut inside a queue chunk (z = 2) and at its end (z = 3)
        again = voxel.voxel_features(cname, lev, s)
        assert torch.equal(again.nan_to_num(nan=-7.0), fast.nan_to_num(nan=-7.0)), cname
        parts = [voxel.voxel_features(cname, lev, s, z0=a, z1=b) for a, b in ((0, 2), (2, 3), (3, 7))]
        assert torch.equal(torch.cat(parts, 1).nan_to_num(nan=-7.0), fast.nan_to_num(nan=-7.0)), cname
        del again, parts
        # the whole volume against the generic kernel at the same bounds (Imc2: against the oracle on the sampled
        # centres only, see _compare -- the two kernels' conventions differ on exactly independent angles)
        monkeypatch.setenv("B200_RADIOMICS_FORCE_GENERIC", "1")
        gen = voxel.voxel_features(cname, lev, s)
        monkeypatch.delenv("B200_RADIOMICS_FORCE_GENERIC")
        compare_window_maps(_at(gen, cen), c["refs"], cname, 0, f"{kind}/generic", True)
        cpg = gen[names.index("ClusterProminence")].reshape(-1).cpu().numpy() if cname == "glcm" else None
        for k, f in enumerate(names):
            if f != "Imc2":
                assert_within_window_bounds(fast[k].reshape(1, -1).cpu().numpy(), gen[k].reshape(1, -1).cpu().numpy(),
                                            cname, [f], f"{kind}/fast vs generic", cpg)
        del fast, gen
        torch.cuda.empty_cache()


def test_glcm_queue_cache_grow_and_release(scale_case):
    """the eigen-task queue grows on demand and rb_release_device_caches gives it back: a small volume gives the same
    maps before the large one, after it, and after the release"""
    rng = np.random.default_rng(5)
    small = torch.as_tensor(rng.integers(1, 33, (12, 40, 44)).astype(np.uint8)).cuda()
    s_small = _lib.make_settings(32, 32)
    big_np = scale_case("uniform")["lev"]
    big = torch.as_tensor(big_np).cuda()
    runs = [voxel.voxel_features("glcm", small, s_small)]
    voxel.voxel_features("glcm", big, _settings(big_np, 32))
    runs.append(voxel.voxel_features("glcm", small, s_small))
    torch.cuda.synchronize()
    _lib.check(_lib.lib().rb_release_device_caches(), "release_device_caches")
    runs.append(voxel.voxel_features("glcm", small, s_small))
    for r in runs[1:]:
        assert torch.equal(r.nan_to_num(nan=-7.0), runs[0].nan_to_num(nan=-7.0))
