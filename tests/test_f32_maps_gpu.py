"""Float32 feature maps written by the texture voxel kernels themselves (rb_voxel_features_dev with out_is_f32 = 1).

Every comparison is bit for bit: the float32 maps of a call equal the float64 maps of the same call rounded to float32
(the kernels compute in float64 and round once, at the store), NaN at the same positions.  Covered: every class on every
dispatch path and settings variant, GLCM voxels whose MCC is finished by the eigen-task phase (planted windows of every
task size in a volume whose queue runs in three z-chunks), slab arguments and strided outputs, status words, the
host-copy driver, the filter pipeline and the NRRD writer."""
import numpy as np
import pytest
import torch

from helpers import envelope_volume, planted_corpus
from pyradiomics_b200 import _lib, featureclasses as FC, image as I, pipeline, voxel

pytestmark = pytest.mark.gpu

SENTINEL = -12345.0


def assert_rounded(f32, f64, what=""):
    """f32 == f64 rounded to float32, bit for bit, NaN where f64 is NaN"""
    assert f32.dtype == torch.float32 and f64.dtype == torch.float64 and f32.shape == f64.shape, what
    ref = f64.to(torch.float32)
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(f32), nan), what
    assert torch.equal(f32.masked_fill(nan, 0).view(torch.int32), ref.masked_fill(nan, 0).view(torch.int32)), what


def _levels(shape, n_levels, seed, holes=True):
    rng = np.random.default_rng(seed)
    img = rng.integers(1, n_levels + 1, shape).astype(np.int32)
    mask = np.ones(shape, bool)
    if holes:
        mask &= rng.random(shape) > 0.15                  # ROI holes, and windows cut by the volume's faces
        mask[:, :2, :3] = False
    img[~mask] = 0
    Ng = int(img.max())
    lev, presence = voxel.pack_levels(torch.as_tensor(img).cuda(), torch.as_tensor(mask.astype(np.uint8)).cuda(), Ng)
    return lev, Ng, int((presence > 0).sum().item())


def _both(cname, lev, s, **kw):
    a = voxel.voxel_features(cname, lev, s, **kw)
    b = voxel.voxel_features(cname, lev, s, dtype=torch.float32, **kw)
    return a, b


# (id, level volume (shape, levels, seed), settings, force the generic kernels, centres mask)
CONFIGS = [
    ("r1-fast", ((9, 20, 22), 32, 1), {}, False, False),
    ("r1-fast-init-centers", ((9, 20, 22), 32, 2), dict(initValue=-3.25), False, True),
    ("r1-generic", ((9, 20, 22), 32, 1), {}, True, False),
    ("r1-generic-init-centers", ((9, 20, 22), 32, 3), dict(initValue=7.5), True, True),
    ("r2", ((8, 14, 15), 24, 4), dict(kernelRadius=2), False, False),
    ("r3", ((8, 11, 12), 16, 5), dict(kernelRadius=3, initValue=1.0), False, False),
    ("weighted-euclidean", ((8, 14, 15), 16, 6), dict(weightingNorm="euclidean", spacing_zyx=(2.0, 0.7, 1.0)), False, False),
    ("weighted-manhattan-r2", ((8, 14, 15), 16, 7), dict(kernelRadius=2, weightingNorm="manhattan",
                                                          spacing_zyx=(2.0, 0.7, 1.0)), False, False),
    ("asymmetric", ((8, 14, 15), 24, 8), dict(symmetricalGLCM=False), False, False),
    ("force2D-z", ((8, 14, 15), 24, 9), dict(force2D=True, force2Ddimension=0), False, False),
    ("force2D-y", ((8, 14, 15), 24, 10), dict(force2D=True, force2Ddimension=1), False, False),
    ("force2D-x", ((8, 14, 15), 24, 11), dict(force2D=True, force2Ddimension=2), False, True),
    ("distances-1-2", ((8, 14, 15), 24, 12), dict(distances=[1, 2], kernelRadius=2), False, False),
    ("ng300-u16", ((8, 14, 15), 300, 13), dict(), False, False),
    ("ng300-u16-r2-generic", ((8, 14, 15), 300, 14), dict(kernelRadius=2), True, False),
]


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c[0] for c in CONFIGS])
@pytest.mark.parametrize("cname", _lib.CLASSES)
def test_float32_maps_are_the_rounded_float64_maps(cname, cfg, monkeypatch):
    _, (shape, n_levels, seed), kw, generic, with_centers = cfg
    if generic:
        monkeypatch.setenv("B200_RADIOMICS_FORCE_GENERIC", "1")
    lev, Ng, nlev = _levels(shape, n_levels, seed)
    assert lev.dtype == (torch.int16 if Ng > 255 else torch.uint8)
    s = _lib.make_settings(Ng, nlev, **kw)
    centers = None
    if with_centers:                                     # an unmasked kernel: centres independent of the ROI
        rng = np.random.default_rng(seed + 100)
        centers = torch.as_tensor((rng.random(shape) > 0.3).astype(np.uint8)).cuda()
    a, b = _both(cname, lev, s, centers=centers)
    assert_rounded(b, a, f"{cname}/{cfg[0]}")
    if kw.get("initValue") and cname == "glcm":
        assert (b == float(kw["initValue"])).any()


def _planted_large():
    """(7, 1024, 1024) levels whose 3x3x3 blocks are planted windows reaching every eigen-task size (dense <= 8, 9-12 and
    Lanczos 13-18): the GLCM queue of this volume runs in three z-chunks"""
    blocks = np.asarray(planted_corpus(6000, seed=3), np.int32)
    nb = 2 * 341 * 341
    tiled = blocks[np.arange(nb) % len(blocks)]
    tiled = tiled.reshape(2, 341, 341, 3, 3, 3).transpose(0, 3, 1, 4, 2, 5).reshape(6, 1023, 1023)
    lev = np.zeros((7, 1024, 1024), np.int32)
    lev[:6, :1023, :1023] = tiled
    return lev


@pytest.fixture(scope="module")
def planted_large():
    lev = _planted_large()
    Ng = int(lev.max())
    lev_t, presence = voxel.pack_levels(torch.as_tensor(lev).cuda(), torch.as_tensor((lev != 0).astype(np.uint8)).cuda(), Ng)
    return lev_t, _lib.make_settings(Ng, int((presence > 0).sum().item()))


def test_glcm_mcc_from_the_eigen_tasks_in_z_chunks(planted_large):
    lev, s = planted_large
    a, b = _both("glcm", lev, s)
    mcc = _lib.feature_names("glcm").index("MCC")
    assert_rounded(b, a, "glcm")
    # the planted windows do need eigen-solves: MCC strictly between 0 and 1 somewhere
    m = a[mcc]
    assert ((m > 0.01) & (m < 0.99)).sum().item() > 1000
    again = voxel.voxel_features("glcm", lev, s, dtype=torch.float32)
    assert torch.equal(again.view(torch.int32), b.view(torch.int32))
    parts = [voxel.voxel_features("glcm", lev, s, z0=z0, z1=z1, dtype=torch.float32) for z0, z1 in ((0, 2), (2, 3), (3, 7))]
    assert torch.equal(torch.cat(parts, 1).view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("cname", _lib.CLASSES)
@pytest.mark.parametrize("generic", [False, True], ids=["fast", "generic"])
def test_slab_into_a_strided_view(cname, generic, monkeypatch):
    if generic:
        monkeypatch.setenv("B200_RADIOMICS_FORCE_GENERIC", "1")
    lev, Ng, nlev = _levels((11, 18, 20), 32, 21)
    s = _lib.make_settings(Ng, nlev)
    whole = voxel.voxel_features(cname, lev, s, dtype=torch.float32)
    assert torch.equal(voxel.voxel_features(cname, lev, s, dtype=torch.float32).view(torch.int32), whole.view(torch.int32))
    nf = whole.shape[0]
    base = torch.full((nf, 9, 18, 20), SENTINEL, dtype=torch.float32, device="cuda")
    out = base[:, :6]                                    # feature stride 9 planes, 6 planes per map
    assert out.stride(0) == 9 * 18 * 20
    z0, z1, out_z0 = 4, 8, 3                             # planes 4..7 -> out[:, 1:5]
    got = voxel.voxel_features(cname, lev, s, z0=z0, z1=z1, out=out, out_z0=out_z0)
    assert got is out
    assert torch.equal(base[:, 1:5].view(torch.int32), whole[:, 4:8].view(torch.int32))
    written = torch.zeros(base.shape, dtype=torch.bool, device="cuda")
    written[:, 1:5] = True
    assert (base[~written] == SENTINEL).all()


def test_status_words_are_the_same_in_both_modes():
    lev = envelope_volume(48)                            # r = 2: MCC eigen-problems over 32 levels
    Ng = int(lev.max())
    lev_t, _ = voxel.pack_levels(torch.as_tensor(lev.astype(np.int32)).cuda(), torch.as_tensor((lev != 0).astype(np.uint8)).cuda(), Ng)
    s = _lib.make_settings(Ng, len(np.unique(lev[lev > 0])), kernelRadius=2)
    st = [torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(2)]
    a = voxel.voxel_features("glcm", lev_t, s, status=st[0])
    b = voxel.voxel_features("glcm", lev_t, s, status=st[1], dtype=torch.float32)
    assert int(st[0].item()) == int(st[1].item()) == 1
    assert_rounded(b, a, "glcm over capacity")
    # the weighted GLCM entry-list overflow (r = 3, 64 levels) is loud in float32 too
    lev = envelope_volume(64)
    sp = (2.0, 0.7, 1.0)
    with pytest.raises(_lib.B200Error, match="entry list overflow"):
        FC.RadiomicsGLCM(I.ArrayImage(lev, sp[::-1]), I.ArrayImage((lev != 0).astype(np.uint8), sp[::-1]), voxelBased=True,
                         binWidth=1, kernelRadius=3, weightingNorm="euclidean", b200_map_dtype="float32").execute()


@pytest.mark.parametrize("cname", _lib.CLASSES)
@pytest.mark.parametrize("zchunk", [1, 3, 64])
def test_class_maps_to_host_float32_ring(cname, zchunk):
    lev, Ng, nlev = _levels((10, 64, 96), 32, 31)
    s = _lib.make_settings(Ng, nlev)
    Z, Y, X = lev.shape
    ref = voxel.voxel_features(cname, lev, s).cpu()
    nf = ref.shape[0]
    idx = [0, 2, 3, nf - 1]                              # runs of consecutive features and a gap
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    host = voxel.class_maps_to_host(cname, lev, s, idx, zchunk=zchunk, out_dtype=torch.float32)
    torch.cuda.synchronize()
    grown = torch.cuda.max_memory_allocated() - base
    zc = min(zchunk, Z)
    ring = (2 if Z > zc else 1) * nf * zc * Y * X * 4
    assert grown <= ring + (1 << 20), (grown, ring)      # one float32 ring, no float64 ring
    assert host.dtype == torch.float32 and host.shape == (len(idx), Z, Y, X)
    assert_rounded(host, ref[idx], cname)
    sub = voxel.class_maps_to_host(cname, lev, s, idx, z0=3, z1=9, zchunk=zchunk, out_dtype=torch.float32)
    assert torch.equal(sub.view(torch.int32), host[:, 3:9].view(torch.int32))


def test_suite_with_filters_and_nrrd_in_float32(tmp_path):
    from pyradiomics_b200 import nrrd
    rng = np.random.default_rng(41)
    img = torch.as_tensor(rng.normal(100, 20, (12, 24, 26))).cuda()
    mask = torch.zeros(img.shape, dtype=torch.uint8, device="cuda")
    mask[2:10, 3:21, 4:22] = 1
    got = {}
    for dt in (torch.float64, torch.float32):
        maps = {}
        pipeline.voxel_suite_with_filters(img, mask, sigmas=(1.0,), binWidth=10, map_dtype=dt,
                                          consume=lambda name, c, m: maps.__setitem__((name, c), m.clone()))
        got[dt] = maps
    assert got[torch.float64].keys() == got[torch.float32].keys() and len(got[torch.float32]) == 10 * 5
    for k, m in got[torch.float32].items():
        assert_rounded(m, got[torch.float64][k], str(k))
    # extract_to_nrrd: float32 maps written as `type: float` files holding those values
    lev, Ng, nlev = _levels((6, 10, 12), 16, 42)
    s = _lib.make_settings(Ng, nlev)
    paths = voxel.extract_to_nrrd(lev, s, tmp_path, classes=("ngtdm",), out_dtype=torch.float32, compress=False)
    ref = voxel.voxel_features("ngtdm", lev, s)
    for k, name in enumerate(_lib.feature_names("ngtdm")):
        raw = open(paths[f"original_ngtdm_{name}"], "rb").read()
        head, data = raw.split(b"\n\n", 1)
        assert b"\ntype: float\n" in head and b"encoding: raw" in head
        arr = torch.as_tensor(np.frombuffer(data, "<f4").reshape(lev.shape).copy())
        assert_rounded(arr, ref[k].cpu(), name)


def test_other_map_types_raise():
    lev, Ng, nlev = _levels((4, 6, 7), 8, 51)
    s = _lib.make_settings(Ng, nlev)
    for dt in (torch.float16, torch.int32, torch.bfloat16):
        with pytest.raises(TypeError):
            voxel.voxel_features("glrlm", lev, s, out=torch.empty((16, 4, 6, 7), dtype=dt, device="cuda"))
        with pytest.raises(TypeError):
            voxel.voxel_features("glrlm", lev, s, dtype=dt)
        with pytest.raises(TypeError):
            pipeline.voxel_suite_with_filters(lev.to(torch.float64), lev != 0, map_dtype=dt)
