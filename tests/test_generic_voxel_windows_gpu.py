"""The generic voxel kernels (csrc/voxel_kernels.cu running csrc/vox_features.cuh) against the general window oracle
(tests/helpers.py: WindowRun, box_features, box_mcc) on the GPU, on every setting the r = 1 fast path declines:
kernelRadius 2 and 3, distances other than {1}, symmetricalGLCM=False, weighted GLCM and GLRLM, force2D on each axis and
a 2-D image, 16-bit levels, a `centers` mask with ROI holes, clipped windows on the faces of a volume, and a volume large
enough that every thread of the kernel's grid-stride loop runs three times.

Volumes are planted with 5^3 / 7^3 blocks (helpers.plant_boxes) so that every planted centre's window is exactly its
block, and run with the planted centres as the `centers` mask: the status word then speaks of those windows alone and is
asserted exactly (bit 0: an MCC problem over the dense solve's capacity, NaN MCC exactly there; bit 1: never, the
weighted corpora leave out windows over the entry-list limits, which tests/test_generic_voxel_windows_cpu.py and the
capacity test below cover).  Bounds are those of the r = 1 file (helpers.window_bound), with the entropy floor scaled to
the window's entry count (helpers.entropy_atol).  The MCC of every window of helpers.reach_corpus (3 300 blocks at r = 2,
3 600 at r = 3) is checked here too, with the same reach assertion the CPU file makes on it: >= 100 eigen-problems of
every row count 2..32, >= 100 over capacity, bipartite and disconnected."""
import numpy as np
import pytest
import torch

from helpers import (FAST_NAMES, GLDM_ALPHAS, MCC_ATOL, WindowRun, assert_mcc_reach, block_corpus, box_mcc, box_references,
                     compare_box_maps, mcc_reach, plant_boxes, reach_corpus, remap_boxes, weighted_overflow, window_box)
from pyradiomics_b200 import _lib, voxel

pytestmark = pytest.mark.gpu

SPACING_ZYX = (2.0, 0.8, 0.6)          # xyz (0.6, 0.8, 2.0)
NORMS = ("manhattan", "euclidean", "infinity", "no_weighting")


def _cuda(a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a if dtype is None else a.astype(dtype))).cuda()


def _pack(vol):
    Ng = int(vol.max())
    lev, _ = voxel.pack_levels(_cuda(vol, np.int32), _cuda(vol != 0), Ng)
    return lev


def _at(out, cen):
    idx = tuple(torch.as_tensor(cen[:, d], device=out.device) for d in range(3))
    return out[(slice(None),) + idx].cpu().numpy()


def _boxes(side, n, seed, Ng=None, K_max=None, shape=None):
    """n seeded side^3 blocks, levels sent into 1..Ng when given, cut to `shape` (force2D: one plane of each block)"""
    boxes = block_corpus(n, side, seed=seed, K_max=K_max)
    if Ng is not None:
        boxes, _ = remap_boxes(boxes, Ng, np.random.default_rng(seed + Ng))
    if shape is not None:
        c = side // 2
        boxes = [b[tuple(slice(c - s // 2, c + s // 2 + 1) for s in shape)] for b in boxes]
        boxes = [b for b in boxes if b[tuple(s // 2 for s in shape)] > 0]
    return boxes


def run_planted(boxes, what, Ng=None, classes=FAST_NAMES, alphas=GLDM_ALPHAS, **kw):
    """plant `boxes`, run every class through voxel.voxel_features with the planted centres as `centers` and compare
    their maps with the oracle; returns {class: worst ratio per feature}"""
    vol, cen = plant_boxes(boxes)
    Ng = Ng or int(vol.max())
    assert vol.max() == Ng, (what, vol.max(), Ng)
    run = WindowRun(vol.shape, Ng, **kw)
    centers = np.zeros(vol.shape, bool)
    centers[tuple(cen.T)] = True
    run.alive_from(vol, centers)
    boxes = [window_box(vol, c, run.radii) for c in cen]
    if run.weights is not None:
        keep = np.array([not weighted_overflow(b, run) for b in boxes])
        boxes, cen = [b for b, k in zip(boxes, keep) if k], cen[keep]
        centers[:] = False
        centers[tuple(cen.T)] = True
        run.alive_from(vol, centers)
    lev = _pack(vol)
    assert lev.dtype == (torch.int16 if Ng > 255 else torch.uint8)
    centers_t = _cuda(centers, np.uint8)
    worst_all = {}
    for cname in classes:
        for a in (alphas if cname == "gldm" else (0,)):
            run.gldm_a = a
            refs = box_references(boxes, run, classes=[cname], mcc=cname == "glcm")
            status = torch.zeros(1, dtype=torch.int32, device="cuda")
            out = voxel.voxel_features(cname, lev, run.settings(len(np.unique(vol[vol > 0]))), centers=centers_t,
                                       status=status)
            got = _at(out, cen)
            st = int(status.item())
            want = int(refs["mcc_over"].any()) if cname == "glcm" else 0
            assert st == want, (what, cname, st, want)
            w = compare_box_maps(got, refs, cname, a, f"{what}/gldm_a={a}", run)
            print(what, cname, a, "worst |error| / bound:", {f: f"{v:.2g}" for f, v in w.items() if v > 1e-3})
            worst_all[(cname, a)] = w
    return worst_all


# ------------------------------------------------------------------------------------------------- default settings
@pytest.mark.parametrize("r", [2, 3])
def test_default_settings(r):
    side = 2 * r + 1
    run_planted(_boxes(side, 88, seed=r), f"r{r}", kernelRadius=r)


# ------------------------------------------------------------------------------------------------ MCC at every size
@pytest.mark.parametrize("r", [2, 3])
def test_mcc_of_the_reach_corpus(r):
    """every window of helpers.reach_corpus(r) planted and run through the generic GLCM kernel: MCC within MCC_ATOL of
    box_mcc, NaN exactly on the windows with a problem over capacity, status bit 0 exactly when there is one"""
    boxes = reach_corpus(r)
    vol, cen = plant_boxes(boxes)
    run = WindowRun(vol.shape, int(vol.max()), kernelRadius=r)
    centers = np.zeros(vol.shape, bool)
    centers[tuple(cen.T)] = True
    run.alive_from(vol, centers)
    mccs = [box_mcc(b, run) for b in boxes]
    assert_mcc_reach(mcc_reach(per for _, per in mccs), f"r{r}")
    ref = np.array([m for m, _ in mccs])
    over = np.array([any(m is not None and m[5] for m in per) for _, per in mccs])
    largest = np.array([max([m[1] for m in per if m is not None and m[3] and min(m[1], m[2]) >= 2 and not m[5]]
                            or [0]) for _, per in mccs])
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = voxel.voxel_features("glcm", _pack(vol), run.settings(len(np.unique(vol[vol > 0]))),
                               centers=_cuda(centers, np.uint8), status=status)
    got = _at(out, cen)[FAST_NAMES["glcm"].index("MCC")]
    assert int(status.item()) == int(over.any())
    assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.isnan(ref[over]).all()
    err = np.where(np.isnan(ref), 0.0, np.abs(got - ref))
    per = {f"{lo}-{hi} rows": float(err[(largest >= lo) & (largest <= hi)].max(initial=0))
           for lo, hi in ((0, 1), (2, 8), (9, 18), (19, 32))}
    print(f"reach r{r}: MCC worst |error| per largest solved problem:", per, "over capacity:", int(over.sum()))
    assert err.max() <= MCC_ATOL, per


# ------------------------------------------------------------------------------------------------------ distances
@pytest.mark.parametrize("r,distances", [(3, (2,)), (3, (1, 3)), (3, (1, 2, 3)), (2, (3,))],
                         ids=["r3-d2", "r3-d13", "r3-d123", "r2-d3"])
def test_distances(r, distances):
    side = 2 * r + 1
    run_planted(_boxes(side, 33, seed=10 + r, K_max=64), f"r{r}/d{distances}", kernelRadius=r, distances=distances,
                alphas=(0, 3))


# ------------------------------------------------------------------------------------------------ asymmetric GLCM
@pytest.mark.parametrize("r", [1, 2, 3])
def test_asymmetric_glcm(r):
    side = 2 * r + 1
    n = 600 if r == 1 else 88
    run_planted(_boxes(side, n, seed=20 + r, Ng=64 if r == 1 else 255), f"asym/r{r}", classes=["glcm"], kernelRadius=r,
                symmetricalGLCM=False)


# ------------------------------------------------------------------------------------------------ weighted GLCM / GLRLM
@pytest.mark.parametrize("norm", NORMS)
@pytest.mark.parametrize("r", [1, 2, 3])
def test_weighted(r, norm):
    side = 2 * r + 1
    run_planted(_boxes(side, 44, seed=30 + r, K_max=60), f"weighted/{norm}/r{r}", classes=["glcm", "glrlm"],
                kernelRadius=r, weightingNorm=norm, spacing_zyx=SPACING_ZYX)


# ------------------------------------------------------------------------------------------------ force2D and 2-D
@pytest.mark.parametrize("dim", [0, 1, 2])
@pytest.mark.parametrize("r", [2, 3])
def test_force2d(r, dim):
    """whole side^3 blocks planted: the window is the centre plane of each, the other planes must not count"""
    side = 2 * r + 1
    run_planted(_boxes(side, 80, seed=40 + r + dim), f"force2D{dim}/r{r}", kernelRadius=r, force2D=True,
                force2Ddimension=dim, alphas=(0, 3))


@pytest.mark.parametrize("r", [2, 3])
def test_two_d_image(r):
    """a 2-D image runs as one plane (Z = 1): its windows are boxes of one plane, the z offsets drop out"""
    side = 2 * r + 1
    run_planted(_boxes(side, 80, seed=50 + r, shape=(1, side, side)), f"2D/r{r}", kernelRadius=r, alphas=(0, 3))


# ------------------------------------------------------------------------------------------------ 16-bit levels
@pytest.mark.parametrize("Ng", [256, 4096, 65535])
@pytest.mark.parametrize("r", [1, 2, 3])
def test_sixteen_bit_levels(r, Ng):
    """Ng > 255 stores levels as uint16: the generic kernel at every radius, r = 1 included"""
    side = 2 * r + 1
    run_planted(_boxes(side, 44 if r > 1 else 300, seed=60 + r, Ng=Ng), f"Ng{Ng}/r{r}", Ng=Ng, kernelRadius=r)


# ------------------------------------------------------------------------------------- masks, faces, capacity, scale
def test_unmasked_run_equals_centers_run():
    """the same planted volume without `centers` (every ROI voxel a centre, windows straddling blocks too): the planted
    centres' maps are bit for bit those of the `centers` run, JointAverage aside (more angles alive in the run)"""
    boxes = _boxes(5, 60, seed=70, K_max=40)
    vol, cen = plant_boxes(boxes)
    lev = _pack(vol)
    centers = np.zeros(vol.shape, np.uint8)
    centers[tuple(cen.T)] = 1
    s = _lib.make_settings(int(vol.max()), len(np.unique(vol[vol > 0])), kernelRadius=2)
    for cname in FAST_NAMES:
        a = _at(voxel.voxel_features(cname, lev, s, centers=_cuda(centers)), cen)
        b = _at(voxel.voxel_features(cname, lev, s), cen)
        if cname == "glcm":
            k = FAST_NAMES["glcm"].index("JointAverage")
            ok = ~np.isnan(a[k]) & ~np.isnan(b[k])
            assert np.array_equal(a[k][ok], b[k][ok])
            a, b = np.delete(a, k, 0), np.delete(b, k, 0)
        assert np.array_equal(a, b, equal_nan=True), cname


@pytest.mark.parametrize("r", [2, 3])
def test_clipped_windows_on_faces(r):
    """sampled centres on the faces, edges and corners of a random (9, 64, 64) volume with ROI holes, the unmasked
    kernel's `centers` choosing them: every window is clipped by the volume"""
    rng = np.random.default_rng(80 + r)
    shape = (9, 64, 64)
    vol = rng.integers(1, 25, shape)
    vol[rng.random(shape) < 0.15] = 0
    vol[0, 0, 0], vol[-1, -1, -1] = 1, 24
    n = 60
    c = np.stack([rng.integers(0, s, n) for s in shape], 1)
    for i in range(n):
        for d in rng.choice(3, int(rng.integers(1, 4)), replace=False):
            c[i, d] = 0 if rng.random() < 0.5 else shape[d] - 1 - int(rng.integers(0, 2)) * (i % 2)
    c = np.unique(c, axis=0)
    c = c[vol[tuple(c.T)] > 0]
    run = WindowRun(shape, 24, kernelRadius=r)
    centers = np.zeros(shape, bool)
    centers[tuple(c.T)] = True
    run.alive_from(vol, centers)
    boxes = [window_box(vol, x, run.radii) for x in c]
    lev = _pack(vol)
    refs = box_references(boxes, run)
    for cname in FAST_NAMES:
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        out = voxel.voxel_features(cname, lev, run.settings(24), centers=_cuda(centers, np.uint8), status=status)
        assert int(status.item()) == (int(refs["mcc_over"].any()) if cname == "glcm" else 0)
        w = compare_box_maps(_at(out, c), refs, cname, 0, f"faces/r{r}", run)
        print("faces", r, cname, "worst |error| / bound:", {f: f"{v:.2g}" for f, v in w.items() if v > 1e-3})


def _weighted_limit_volume(kind, rng):
    """one 7^3 block at r = 3, weighted over distances {1, 2, 3}: 'sums' 45 spread 16-bit levels (2025 pairs fit the
    list, up to 1035 distinct sums do not fit KCAP), 'entries' 48 levels (more than 2048 pairs), 'fits' 40 levels"""
    n = {"sums": 45, "entries": 48, "fits": 40}[kind]
    levels = np.sort(rng.choice(np.arange(1, 65536), n, replace=False))
    levels[0], levels[-1] = 1, 65535
    return levels[rng.permutation(np.arange(343) % n)].reshape(7, 7, 7)


@pytest.mark.parametrize("kind", ["sums", "entries", "fits"])
def test_weighted_capacity_status_exact(kind):
    """status bit 1 exactly when a window's pooled entry list or its |i - j| / i + j lists overflow, computed from every
    voxel's (clipped) window in the test; bit 0 exactly when a pooled MCC problem is over capacity"""
    vol = _weighted_limit_volume(kind, np.random.default_rng(90))
    run = WindowRun(vol.shape, 65535, kernelRadius=3, distances=(1, 2, 3), weightingNorm="euclidean",
                    spacing_zyx=SPACING_ZYX)
    boxes = [window_box(vol, c, run.radii) for c in np.ndindex(vol.shape)]
    over1 = any(weighted_overflow(b, run) for b in boxes)
    over0 = any(any(m is not None and m[5] for m in box_mcc(b, run)[1]) for b in boxes)
    assert over1 == (kind != "fits")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    voxel.voxel_features("glcm", _pack(vol), run.settings(len(np.unique(vol))), status=status)
    assert int(status.item()) & 2 == 2 * int(over1)
    if not over1:
        assert int(status.item()) & 1 == int(over0)


# the generic kernel's launch (voxel_kernels.cu launch_cls, common.cuh grid_for): 128 threads per block, at most 64
# resident-or-queued blocks per SM, one thread per voxel in a grid-stride loop
def _grid_for(n, block, per_sm, sms):
    return max(1, min(-(-n // block), sms * per_sm))


def test_large_volume_grid_stride():
    """(14, 512, 512) at r = 2: every thread loops at least three times; sampled centres against the oracle, the whole
    volume bit for bit against a second run and against z-slab calls"""
    shape = (14, 512, 512)
    total = int(np.prod(shape))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grid = _grid_for(total, 128, 64, sms)
    assert total >= 3 * grid * 128, (total, grid)
    rng = np.random.default_rng(95)
    zz, yy, xx = np.meshgrid(*[np.arange(s, dtype=np.float64) for s in shape], indexing="ij", sparse=True)
    f = np.sin(zz / 2.1) + np.cos(yy / 3.3) + np.sin(xx / 2.7 + 1) + 0.4 * rng.normal(size=shape)
    vol = np.digitize(f, np.quantile(f, np.linspace(0, 1, 20)[1:-1])) + 1
    vol[rng.random(shape) < 0.05] = 0
    vol[0, 0, 0] = 1
    run = WindowRun(shape, int(vol.max()), kernelRadius=2)
    c = np.stack([rng.integers(0, s, 160) for s in shape], 1)
    c[:40, 0] = rng.choice([0, 1, shape[0] - 2, shape[0] - 1], 40)
    c = c[vol[tuple(c.T)] > 0]
    run.alive_from(vol[:, :40, :40])            # every angle has pairs in this corner already: all alive
    assert run.alive.all()
    boxes = [window_box(vol, x, run.radii) for x in c]
    refs = box_references(boxes, run)
    lev = _pack(vol)
    s = run.settings(len(np.unique(vol[vol > 0])))
    for cname in FAST_NAMES:
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        out = voxel.voxel_features(cname, lev, s, status=status)
        assert int(status.item()) & 2 == 0
        w = compare_box_maps(_at(out, c), refs, cname, 0, "large/r2", run)
        print("large", cname, "worst |error| / bound:", {f: f"{v:.2g}" for f, v in w.items() if v > 1e-3})
        again = voxel.voxel_features(cname, lev, s)
        assert torch.equal(again.nan_to_num(nan=-7.0), out.nan_to_num(nan=-7.0)), cname
        del again
        parts = [voxel.voxel_features(cname, lev, s, z0=a, z1=b) for a, b in ((0, 3), (3, 10), (10, 14))]
        assert torch.equal(torch.cat(parts, 1).nan_to_num(nan=-7.0), out.nan_to_num(nan=-7.0)), cname
        del out, parts
        torch.cuda.empty_cache()
