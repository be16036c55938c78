"""The voxel-map path on the caller's stream and from concurrent host threads (include/b200radiomics.h, the threading
contract by rb_release_device_caches).

Ordering on the caller's stream is made visible, not left to timing: the inputs hold a *sentinel* volume (the real
one mirrored in x, its levels shifted cyclically) and the maps NaN, written on the default stream and synchronised.
Then on a fresh side stream `s` (torch's streams are non-blocking, so nothing orders them with the legacy stream) a
bounded delay kernel is queued, the real volume is copied over the inputs in place, and the entry point is called with
no host synchronisation in between.  A launch, memset or copy that went to any other stream would run during the delay
on the sentinel (or write before the real maps), so the maps are compared bit for bit, NaN payloads and status words
included, with the same call on the default stream.  Where a driver synchronises the host before its launches, what it
would compute there is passed in (the GLCM alive angles, the first-order radii, the binning range), or the delay is put
after that synchronisation (pack_levels inside HostExtractor; the discretisation's min / max and digitisation, whose
inputs are uploaded by synchronous copies, through DelayedEntry).

Then three host threads, each on its own stream, run this pattern at once while the shared state changes under them
(device_table's first use of a level count, a GLCM queue and a wide workspace that grow), and two host threads share
the default stream while a third releases the device caches: every map equals the serial default-stream run."""
import threading

import numpy as np
import pytest
import torch

from helpers import (FAST_NAMES, WindowRun, box_references, compare_box_maps, compare_window_maps, window_at,
                     window_references, window_box)
from pyradiomics_b200 import _lib, imageoperations as IO, voxel

pytestmark = pytest.mark.gpu

# torch.cuda._sleep spins for this many clock cycles: 20 ms at 2.0 GHz, 40 ms at 1.0 GHz
DELAY_CYCLES = 40_000_000
MAP_DTYPES = (torch.float64, torch.float32)
_BITS = {8: torch.int64, 4: torch.int32, 2: torch.int16, 1: torch.uint8}


def _bits(t):
    t = t.contiguous()
    return t.view(_BITS[t.element_size()])


def assert_same_bits(got, ref, what):
    assert got.shape == ref.shape and got.dtype == ref.dtype, (what, got.shape, ref.shape, got.dtype, ref.dtype)
    g, r = _bits(got), _bits(ref.to(got.device))
    if not torch.equal(g, r):
        bad = (g != r).nonzero()
        raise AssertionError(f"{what}: {bad.shape[0]} of {g.numel()} values differ, first at {tuple(bad[0].tolist())}")


def _cuda(a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a if dtype is None else a.astype(dtype))).cuda()


def _volume(shape, Ng, seed, holes=0.05):
    """seeded int levels 1..Ng (a smooth field plus noise, so windows repeat levels), 0 on a share of holes"""
    rng = np.random.default_rng(seed)
    zz, yy, xx = np.meshgrid(*[np.arange(s, dtype=np.float64) for s in shape], indexing="ij", sparse=True)
    f = np.sin(zz / 1.7) + np.cos(yy / 2.3) + np.sin(xx / 1.9 + 1) + 0.8 * rng.normal(size=shape)
    vol = np.digitize(f, np.quantile(f, np.linspace(0, 1, Ng + 1)[1:-1])) + 1
    vol[rng.random(shape) < holes] = 0
    vol[0, 0, 0] = Ng
    return vol.astype(np.int32)


def _pack(vol):
    Ng = int(vol.max())
    lev, _ = voxel.pack_levels(_cuda(vol), _cuda(vol != 0, np.uint8), Ng)
    return lev


def _settings(vol, **kw):
    return _lib.make_settings(int(vol.max()), len(np.unique(vol[vol > 0])), **kw)


def _sentinel(t, Ng=None):
    """the real tensor mirrored in x; levels (Ng given) also shifted cyclically, 1..Ng stays 1..Ng and 0 stays 0"""
    s = t.flip(-1)
    if Ng is not None:
        s = torch.where(s > 0, s % Ng + 1, s).to(t.dtype)
    return s.contiguous()


def on_side_stream(call, pairs):
    """call() on a fresh side stream behind the delay and the in-place copies `pairs` [(held input, real input)], the
    held inputs already holding the sentinel; returns its result once the stream is done"""
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(DELAY_CYCLES)
        for held, real in pairs:
            held.copy_(real)
        out = call()
    s.synchronize()
    return out


def _nan_maps(nf, shape, dtype):
    return torch.full((nf,) + tuple(shape), float("nan"), dtype=dtype, device="cuda")


# ------------------------------------------------------------------------------------------------------- volumes
@pytest.fixture(scope="module")
def fast_case():
    """(16, 48, 64), 12 levels with ROI holes: every r = 1 class runs its fast kernel"""
    vol = _volume((16, 48, 64), 12, seed=3)
    lev = _pack(vol)
    s = _settings(vol)
    alive = voxel.glcm_alive_angles(lev, s)
    assert bin(int(alive[0])).count("1") == 13
    return {"vol": vol, "lev": lev, "settings": s, "alive": alive, "Ng": int(vol.max())}


# ------------------------------------------------------------------------------- discretisation and alive angles
def test_pack_levels_on_the_callers_stream():
    vol = _volume((9, 40, 56), 30, seed=5)
    img, msk = _cuda(vol), _cuda(vol != 0, np.uint8)
    ref_lev, ref_pres = voxel.pack_levels(img, msk, 30)
    held_img, held_msk = _sentinel(img, 30), _sentinel(msk)
    sent_lev, sent_pres = voxel.pack_levels(held_img, held_msk, 30)
    assert not torch.equal(sent_lev, ref_lev) and not torch.equal(sent_pres, ref_pres)
    lev, pres = on_side_stream(lambda: voxel.pack_levels(held_img, held_msk, 30), [(held_img, img), (held_msk, msk)])
    assert_same_bits(lev, ref_lev, "levels")
    assert_same_bits(pres, ref_pres, "presence")


class DelayedEntry:
    """the library with entry point `name` delayed: right before each call of it, the delay kernel and the in-place
    copies `pairs` [(held input, real input)] are queued on the current stream -- after any host synchronisation the
    driver made on its way there (torch's pageable uploads of `keys` and the bin edges are such synchronisations)"""

    def __init__(self, name, pairs):
        self._lib, self._name, self._pairs, self.calls = _lib.lib(), name, pairs, 0

    def __getattr__(self, attr):
        f = getattr(self._lib, attr)
        if attr != self._name:
            return f

        def delayed(*args):
            self.calls += 1
            torch.cuda._sleep(DELAY_CYCLES)
            for held, real in self._pairs:
                held.copy_(real)
            return f(*args)
        return delayed


@pytest.mark.parametrize("binning", [{"binWidth": 25}, {"binCount": 19}], ids=["binWidth", "binCount"])
@pytest.mark.parametrize("entry", ["rb_minmax_dev", "rb_digitize_dev"], ids=["minmax", "digitize"])
def test_discretize_on_the_callers_stream(monkeypatch, binning, entry):
    """the delay and the copy of the real image and mask go in right before the ROI min / max, or (the binning range
    passed in, so the min / max is not run) right before the digitisation; the sentinel image has another range"""
    rng = np.random.default_rng(17)
    raw = (rng.normal(size=(10, 36, 44)) * 120 + 40).astype(np.float64)
    mask = (rng.random(raw.shape) < 0.9).astype(np.uint8)
    img, msk = _cuda(raw), _cuda(mask)
    ref = voxel.discretize(img, msk, **binning)
    held_img, held_msk = (_sentinel(img) * 1.5 + 10).contiguous(), _sentinel(msk)
    assert not np.array_equal(voxel.discretize(held_img, held_msk, **binning)[1], ref[1])
    if entry == "rb_digitize_dev":
        rng_real = IO._binning_range(img, msk)
        monkeypatch.setattr(IO, "_binning_range", lambda *a, **k: rng_real)
    proxy = DelayedEntry(entry, [(held_img, img), (held_msk, msk)])
    monkeypatch.setattr(IO, "lib", lambda: proxy)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = voxel.discretize(held_img, held_msk, **binning)
    s.synchronize()
    assert proxy.calls == 1, proxy.calls
    assert_same_bits(got[0], ref[0], "int32 levels")
    assert np.array_equal(got[1], ref[1]), "edges"
    assert_same_bits(got[2], ref[2], "packed levels")
    assert np.array_equal(got[3], ref[3]) and got[4] == ref[4]


@pytest.mark.parametrize("with_centers", [False, True])
def test_glcm_alive_angles_on_the_callers_stream(with_centers):
    """the real ROI is one plane (4 of 13 angles alive), the sentinel the whole volume (all alive)"""
    vol = np.zeros((6, 30, 34), np.int32)
    vol[3] = _volume((1, 30, 34), 9, seed=8, holes=0.0)[0]
    lev = _pack(vol)
    full = _pack(_volume(vol.shape, 9, seed=9, holes=0.0))
    s = _settings(vol)
    cen = _cuda(vol != 0, np.uint8) if with_centers else None
    held_cen = torch.ones_like(cen) if with_centers else None
    ref = voxel.glcm_alive_angles(lev, s, cen)
    sent = voxel.glcm_alive_angles(full, s, held_cen)
    assert bin(int(ref[0])).count("1") == 4 and bin(int(sent[0])).count("1") == 13
    held = full.clone()
    pairs = [(held, lev)] + ([(held_cen, cen)] if with_centers else [])
    got = on_side_stream(lambda: voxel.glcm_alive_angles(held, s, held_cen), pairs)
    assert np.array_equal(got, ref), (got, ref)


# ---------------------------------------------------------------------------------------------- texture maps
def _run_side(cls, lev, settings, Ng, dtype, alive=None, centers=None, held_centers=None, z0=0, z1=None, out=None,
              out_z0=None):
    """voxel_features on the side stream: held levels (and centres) start as the sentinel; returns (maps, status)"""
    Z, Y, X = lev.shape
    z1 = Z if z1 is None else z1
    nf = _lib.lib().rb_num_features(_lib.CLASS_ID[cls])
    out = _nan_maps(nf, (z1 - z0, Y, X), dtype) if out is None else out
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    held = _sentinel(lev, Ng)
    pairs = [(held, lev)]
    if centers is not None:
        pairs.append((held_centers, centers))
    on_side_stream(lambda: voxel.voxel_features(cls, held, settings, centers=held_centers if centers is not None else None,
                                                z0=z0, z1=z1, out=out, out_z0=z0 if out_z0 is None else out_z0,
                                                alive=alive, status=status), pairs)
    return out, status


def _run_default(cls, lev, settings, dtype, alive=None, centers=None, z0=0, z1=None):
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = voxel.voxel_features(cls, lev, settings, centers=centers, z0=z0, z1=z1, alive=alive, status=status, dtype=dtype)
    return out, status


def _at(out, cen):
    idx = tuple(torch.as_tensor(cen[:, d], device=out.device) for d in range(3))
    return out[(slice(None),) + idx].double().cpu().numpy()


@pytest.mark.parametrize("dtype", MAP_DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("cls", list(FAST_NAMES))
def test_fast_path_on_the_callers_stream(fast_case, cls, dtype):
    c = fast_case
    alive = c["alive"] if cls == "glcm" else None
    ref, ref_st = _run_default(cls, c["lev"], c["settings"], dtype, alive)
    got, st = _run_side(cls, c["lev"], c["settings"], c["Ng"], dtype, alive)
    assert_same_bits(got, ref, f"{cls}/{dtype}")
    assert_same_bits(st, ref_st, f"{cls}/{dtype} status")
    if dtype == torch.float64:                # a sample of centres against the r = 1 window oracle
        vol = c["vol"]
        rng = np.random.default_rng(21)
        cen = np.argwhere(vol > 0)
        cen = cen[rng.choice(len(cen), 24, replace=False)]
        wins = [window_at(vol, x) for x in cen]
        refs = window_references(wins, c["Ng"], alphas=(0,))
        compare_window_maps(_at(got, cen), refs, cls, 0, f"side stream/{cls}", False)


# GLCM's eigen-task queue (voxel_fast.cu glcm_fast_run): at most 48 Mi entries of 13 per voxel, the planes spread evenly
# over the chunks
def _glcm_chunks(Z, Y, X):
    plane = Y * X
    zchunk = max(1, (48 << 20) // (plane * 13))
    zchunk = min(zchunk, Z)
    n = -(-Z // zchunk)
    zchunk = -(-Z // n)
    return [(a, min(a + zchunk, Z)) for a in range(0, Z, zchunk)]


@pytest.fixture(scope="module")
def big_glcm():
    shape = (7, 1024, 1024)
    assert _glcm_chunks(*shape) == [(0, 3), (3, 6), (6, 7)]
    vol = _volume(shape, 16, seed=31, holes=0.03)
    lev = _pack(vol)
    s = _settings(vol)
    return {"vol": vol, "lev": lev, "settings": s, "alive": voxel.glcm_alive_angles(lev, s), "Ng": 16}


@pytest.mark.parametrize("dtype", MAP_DTYPES, ids=["f64", "f32"])
def test_multi_chunk_glcm_on_the_callers_stream(big_glcm, dtype):
    c = big_glcm
    ref, ref_st = _run_default("glcm", c["lev"], c["settings"], dtype, c["alive"])
    got, st = _run_side("glcm", c["lev"], c["settings"], c["Ng"], dtype, c["alive"])
    assert_same_bits(got, ref, f"glcm 3 chunks/{dtype}")
    assert_same_bits(st, ref_st, "status")
    del ref, got
    torch.cuda.empty_cache()


GENERIC_CASES = [(c, {}) for c in FAST_NAMES] + [("glcm", {"weightingNorm": "manhattan"}),
                                                  ("glrlm", {"weightingNorm": "euclidean"})]


@pytest.mark.parametrize("dtype", MAP_DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("cls,kw", GENERIC_CASES, ids=[f"{c}-{kw.get('weightingNorm', 'plain')}" for c, kw in GENERIC_CASES])
def test_generic_kernel_on_the_callers_stream(cls, kw, dtype):
    vol = _volume((10, 28, 36), 8, seed=41)
    lev = _pack(vol)
    s = _settings(vol, kernelRadius=2, spacing_zyx=(2.0, 0.8, 0.6), **kw)
    alive = voxel.glcm_alive_angles(lev, s) if cls == "glcm" else None
    ref, ref_st = _run_default(cls, lev, s, dtype, alive)
    got, st = _run_side(cls, lev, s, 8, dtype, alive)
    assert_same_bits(got, ref, f"r2 {cls} {kw}/{dtype}")
    assert_same_bits(st, ref_st, "status")
    if dtype == torch.float64 and not kw:     # a sample of centres against the general window oracle
        run = WindowRun(vol.shape, 8, kernelRadius=2).alive_from(vol)
        rng = np.random.default_rng(43)
        cen = np.argwhere(vol > 0)
        cen = cen[rng.choice(len(cen), 12, replace=False)]
        refs = box_references([window_box(vol, x, run.radii) for x in cen], run, classes=[cls], mcc=cls == "glcm")
        compare_box_maps(_at(got, cen), refs, cls, 0, f"side stream r2/{cls}", run)


def _wide_case(Ng, seed):
    vol = _volume((11, 22, 24), Ng, seed=seed)       # Ng > 255: 16-bit levels
    centers = np.zeros(vol.shape, bool)
    centers[1::3, 1::5, 2::5] = True
    centers &= vol > 0
    return vol, centers


@pytest.mark.parametrize("dtype", MAP_DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("Ng", [10, 300], ids=["8bit", "16bit"])
@pytest.mark.parametrize("cls", list(FAST_NAMES))
def test_wide_kernel_on_the_callers_stream(cls, Ng, dtype):
    vol, centers = _wide_case(Ng, seed=51)
    lev = _pack(vol)
    assert lev.dtype == (torch.int16 if Ng > 255 else torch.uint8)
    s = _settings(vol, kernelRadius=5)
    cen = _cuda(centers, np.uint8)
    alive = voxel.glcm_alive_angles(lev, s, cen) if cls == "glcm" else None
    ref, ref_st = _run_default(cls, lev, s, dtype, alive, centers=cen)
    held_cen = _sentinel(cen)
    got, st = _run_side(cls, lev, s, int(vol.max()), dtype, alive, centers=cen, held_centers=held_cen)
    assert_same_bits(got, ref, f"r5 {cls} Ng={Ng}/{dtype}")
    assert_same_bits(st, ref_st, "status")


@pytest.mark.parametrize("cls", list(FAST_NAMES))
def test_z_slab_into_strided_out_on_the_callers_stream(fast_case, cls):
    """planes [5, 11) into planes [2, 8) of a 9-plane buffer whose feature stride is 9 planes"""
    c = fast_case
    Z, Y, X = c["lev"].shape
    alive = c["alive"] if cls == "glcm" else None
    ref, _ = _run_default(cls, c["lev"], c["settings"], torch.float64, alive)
    nf = ref.shape[0]
    big = _nan_maps(nf, (9, Y, X), torch.float64)
    got = big[:, 2:8]
    assert got.stride(0) == 9 * Y * X
    _run_side(cls, c["lev"], c["settings"], c["Ng"], torch.float64, alive, z0=5, z1=11, out=got, out_z0=5)
    assert_same_bits(got, ref[:, 5:11], f"slab {cls}")
    assert big[:, :2].isnan().all() and big[:, 8:].isnan().all()


# --------------------------------------------------------------------------------------------------- first order
@pytest.mark.parametrize("dtype", MAP_DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("r", [1, 2, 5])
def test_firstorder_on_the_callers_stream(fast_case, monkeypatch, r, dtype):
    """float32 maps go through the float64 scratch, four planes at a time"""
    c = fast_case
    rng = np.random.default_rng(61)
    image = _cuda((c["vol"] * 7.5 + rng.normal(size=c["vol"].shape) * 3).astype(np.float64))
    roi = _cuda(c["vol"] != 0, np.uint8)
    lev = c["lev"]
    kw = dict(kernelRadius=r, voxelArrayShift=3, dtype=dtype, zchunk=4)
    ref = voxel.firstorder_features(image, lev, roi, **kw)
    radii = voxel.firstorder_radii(r, lev.shape, roi)
    monkeypatch.setattr(voxel, "firstorder_radii", lambda *a, **k: radii)     # its ROI box synchronises the host
    held = [_sentinel(image), _sentinel(lev, c["Ng"]), _sentinel(roi)]
    got = on_side_stream(lambda: voxel.firstorder_features(*held, **kw), list(zip(held, (image, lev, roi))))
    assert_same_bits(got, ref, f"firstorder r={r}/{dtype}")


# -------------------------------------------------------------------------------------------- host-facing drivers
@pytest.mark.parametrize("dtype", MAP_DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("cls,idx", [("glcm", [0, 1, 2, 5, 19, 23]), ("glszm", [3, 4, 5, 6, 15])])
def test_class_maps_to_host_ring_on_the_callers_stream(fast_case, cls, idx, dtype):
    """zchunk 5 of 16 planes: four chunks through both ring slots, a feature subset of several runs"""
    c = fast_case
    alive = c["alive"] if cls == "glcm" else None
    kw = dict(alive=alive, zchunk=5, out_dtype=dtype)
    ref = voxel.class_maps_to_host(cls, c["lev"], c["settings"], idx, **kw)
    held = _sentinel(c["lev"], c["Ng"])
    host = torch.empty(ref.shape, dtype=ref.dtype, pin_memory=True)      # allocated before: no page-locked allocation inside the call
    got = on_side_stream(lambda: voxel.class_maps_to_host(cls, held, c["settings"], idx, host=host, **kw),
                         [(held, c["lev"])])
    assert_same_bits(got, ref, f"maps_to_host {cls}/{dtype}")


def test_host_extractor_on_the_callers_stream(fast_case, monkeypatch):
    """run() uploads and packs the levels, which synchronises the host (pack_levels' status word); the delay and the
    sentinel go in after that, so every class's launches and copies are behind them"""
    c = fast_case
    vol = c["vol"]
    args = (vol, (vol != 0).astype(np.uint8), c["Ng"], len(np.unique(vol[vol > 0])))
    ref = {k: v.clone() for k, v in voxel.HostExtractor(vol.shape, zchunk=5).run(*args, alive=c["alive"]).items()}
    real_pack = voxel.pack_levels

    def delayed_pack(image, mask, Ng):
        lev, presence = real_pack(image, mask, Ng)
        held = _sentinel(lev, Ng)
        torch.cuda.current_stream().synchronize()
        torch.cuda._sleep(DELAY_CYCLES)
        held.copy_(lev)
        return held, presence
    monkeypatch.setattr(voxel, "pack_levels", delayed_pack)
    ex = voxel.HostExtractor(vol.shape, zchunk=5)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = ex.run(*args, alive=c["alive"])
    s.synchronize()
    assert got.keys() == ref.keys()
    for k in ref:
        assert_same_bits(got[k], ref[k], f"HostExtractor {k}")


@pytest.mark.parametrize("cls", ["gldm", "glszm", "glrlm", "ngtdm", "glcm", "firstorder"])
def test_extract_to_nrrd_on_the_callers_stream(fast_case, monkeypatch, tmp_path, cls):
    """one class per call (each class ends with a host synchronisation): its files equal the default stream's byte for
    byte"""
    c = fast_case
    lev = c["lev"][:8, :24, :32].contiguous()
    vol = c["vol"][:8, :24, :32]
    s = _settings(vol)
    rng = np.random.default_rng(71)
    image = _cuda((vol * 7.5 + rng.normal(size=vol.shape) * 3).astype(np.float64))
    alive = voxel.glcm_alive_angles(lev, s)
    kw = dict(classes=(cls,), image=image, zchunk=3, workers=2, spacing_xyz=(0.7, 0.8, 2.0))
    ref = voxel.extract_to_nrrd(lev, s, str(tmp_path / "ref"), **kw)
    radii = voxel.firstorder_radii(1, lev.shape, lev != 0)
    monkeypatch.setattr(voxel, "glcm_alive_angles", lambda *a, **k: alive)
    monkeypatch.setattr(voxel, "firstorder_radii", lambda *a, **k: radii)
    held_lev, held_img = _sentinel(lev, int(vol.max())), _sentinel(image)
    got = on_side_stream(lambda: voxel.extract_to_nrrd(held_lev, s, str(tmp_path / "side"), **dict(kw, image=held_img)),
                         [(held_lev, lev), (held_img, image)])
    assert sorted(got) == sorted(ref) and ref
    for k, p in ref.items():
        with open(p, "rb") as a, open(got[k], "rb") as b:
            assert a.read() == b.read(), k


# ------------------------------------------------------------------------------------------ concurrent host threads
def _run_threads(workers, parties=None):
    """start the workers together (threading.Barrier), join them all, re-raise the first failure"""
    barrier = threading.Barrier(parties or len(workers))
    errors = []

    def wrap(fn):
        def go():
            try:
                fn(barrier)
            except BaseException as e:       # noqa: BLE001 -- reported after the join
                errors.append(e)
                barrier.abort()
        return go
    threads = [threading.Thread(target=wrap(fn)) for fn in workers]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    torch.cuda.synchronize()
    if errors:
        raise errors[0]


def test_different_streams_from_concurrent_threads():
    """three threads, a stream each, the step-by-step pattern of the tests above on their own volumes, while the shared
    state changes: threads 0 and 1 are the first to use GLCM's fast tables for 241 levels (no other test uses that
    level count, and the serial runs come after the threads), thread 1 then grows its
    GLCM queue (a 4-plane 64^2 volume, then 5 planes of 384^2), thread 2 grows its wide workspace.  The workspace is
    grid x block bytes (voxel_wide.cu wide_layout / wide_grid), the grid at most one block per voxel and at least one
    per SM: NGTDM at r = 4 on a (3, 9, 9) volume takes at most 243 blocks of 8 944 + 5 200 bytes (an angle slot's lists of
    729 entries, the block's per-angle results), 3.4 MB; NGTDM at r = 7 takes at least 132 blocks (the H100's SMs) of
    40 696 + 5 200 bytes, 6.1 MB, so that call grows it whatever its occupancy; GLSZM at r = 7 follows on the same
    workspace"""
    assert _lib.lib().rb_release_device_caches() == 0     # every queue and workspace starts empty: both must grow
    assert torch.cuda.get_device_properties(0).multi_processor_count * (40696 + 5200) > 243 * (8944 + 5200)
    jobs = []                                            # per thread: [(cls, lev, settings, alive, centers)]

    def job(vol, cls, centers=None, **kw):
        lev = _pack(vol)
        s = _settings(vol, **kw)
        cen = None if centers is None else _cuda(centers, np.uint8)
        alive = voxel.glcm_alive_angles(lev, s, cen) if cls == "glcm" else None
        return cls, lev, s, alive, cen

    ng = 241
    jobs.append([job(_volume((6, 80, 96), ng, seed=81), "glcm"), job(_volume((6, 80, 96), 40, seed=82), "glrlm")])
    jobs.append([job(_volume((4, 64, 64), ng, seed=83), "glcm"), job(_volume((5, 384, 384), 30, seed=84), "glcm")])
    wv = _volume((15, 24, 26), 12, seed=85)
    cen = np.zeros(wv.shape, bool)
    cen[2::4, 1::4, 1::4] = True
    cen &= wv > 0
    jobs.append([job(_volume((3, 9, 9), 12, seed=86), "ngtdm", kernelRadius=4), job(wv, "ngtdm", cen, kernelRadius=7),
                 job(wv, "glszm", cen, kernelRadius=7)])
    streams = [torch.cuda.Stream() for _ in jobs]
    results = [[None] * len(j) for j in jobs]
    prepared = []
    for j in jobs:
        prepared.append([])
        for cls, lev, s, alive, cen in j:
            nf = _lib.lib().rb_num_features(_lib.CLASS_ID[cls])
            prepared[-1].append((_sentinel(lev, s.Ng), None if cen is None else _sentinel(cen), _nan_maps(nf, lev.shape,
                                 torch.float64), torch.zeros(1, dtype=torch.int32, device="cuda")))
    torch.cuda.synchronize()

    def worker(t):
        def run(barrier):
            barrier.wait()
            with torch.cuda.stream(streams[t]):
                for i, ((cls, lev, s, alive, cen), (held, held_cen, out, st)) in enumerate(zip(jobs[t], prepared[t])):
                    torch.cuda._sleep(DELAY_CYCLES)
                    held.copy_(lev)
                    if cen is not None:
                        held_cen.copy_(cen)
                    voxel.voxel_features(cls, held, s, centers=held_cen, out=out, alive=alive, status=st)
                    results[t][i] = (out, st)
            streams[t].synchronize()
        return run
    _run_threads([worker(t) for t in range(len(jobs))])
    for t, j in enumerate(jobs):
        for i, (cls, lev, s, alive, cen) in enumerate(j):
            ref, ref_st = _run_default(cls, lev, s, torch.float64, alive, centers=cen)
            assert_same_bits(results[t][i][0], ref, f"thread {t} job {i} {cls}")
            assert_same_bits(results[t][i][1], ref_st, f"thread {t} job {i} status")


def test_same_stream_from_concurrent_threads(big_glcm):
    """two threads on the default stream (a thread pool's default), two rounds: each enqueues a multi-chunk GLCM, then
    two wide r = 5 calls, the second needing a larger workspace than the first (GLSZM / GLDM, then GLCM; 16-bit levels
    in one thread); a third thread releases the device caches as round two starts"""
    c = big_glcm
    v8, cen8 = _wide_case(10, seed=91)
    v16, cen16 = _wide_case(300, seed=92)
    sub = c["vol"][:4]                                   # (4, 1024, 1024): two queue chunks of 2 planes
    assert len(_glcm_chunks(*sub.shape)) == 2

    def job(vol, cls, centers=None, **kw):
        lev = _pack(vol)
        s = _settings(vol, **kw)
        cen = None if centers is None else _cuda(centers, np.uint8)
        alive = voxel.glcm_alive_angles(lev, s, cen) if cls == "glcm" else None
        return cls, lev, s, alive, cen

    jobs = [[("glcm", c["lev"], c["settings"], c["alive"], None), job(v8, "glszm", cen8, kernelRadius=5),
             job(v8, "glcm", cen8, kernelRadius=5)],
            [job(sub, "glcm"), job(v16, "gldm", cen16, kernelRadius=5), job(v16, "glcm", cen16, kernelRadius=5)]]
    rounds = 2
    results = [[[None] * len(j) for j in jobs] for _ in range(rounds)]
    assert _lib.lib().rb_release_device_caches() == 0
    torch.cuda.synchronize()

    def worker(t):
        def run(barrier):
            for rd in range(rounds):
                barrier.wait()
                for i, (cls, lev, s, alive, cen) in enumerate(jobs[t]):
                    st = torch.zeros(1, dtype=torch.int32, device="cuda")
                    out = voxel.voxel_features(cls, lev, s, centers=cen, alive=alive, status=st)
                    results[rd][t][i] = (out, st)
                torch.cuda.current_stream().synchronize()
        return run

    def releaser(barrier):
        for rd in range(rounds):
            barrier.wait()
            if rd > 0:
                assert _lib.lib().rb_release_device_caches() == 0
    _run_threads([worker(0), worker(1), releaser])
    for t, j in enumerate(jobs):
        for i, (cls, lev, s, alive, cen) in enumerate(j):
            ref, ref_st = _run_default(cls, lev, s, torch.float64, alive, centers=cen)
            for rd in range(rounds):
                assert_same_bits(results[rd][t][i][0], ref, f"round {rd} thread {t} job {i} {cls}")
                assert_same_bits(results[rd][t][i][1], ref_st, f"round {rd} thread {t} job {i} status")
            del ref
    del results
    torch.cuda.empty_cache()
