"""Voxel-based first order at kernelRadius 1 on the GPU: one JSON line.

* 256^3 uniform and smooth volumes (bench.py's levels, raw int16 intensities (level - 1) * 25 + 3, every voxel in the
  ROI): CUDA-event time of rb_firstorder_voxel_dev with the generic kernel (B200_RADIOMICS_FORCE_GENERIC=1) and with the
  tile kernel, alternating in one process, --reps runs each; the spread (max - min) of each; whether the two write the
  same bits.
* BASELINE.json config 4 at 256^3 (bench.py's smoothed float volume, original + wavelet + LoG -> binWidth 25) through
  pipeline.voxel_suite_with_filters with and without "firstorder": ms per image, alternating.
* The 512^3 float32 suite (75 texture maps) plus the 18 first-order maps of the original image on one GPU: time, peak
  torch.cuda.max_memory_allocated, --oracle-voxels sampled centres (a quarter on faces / edges / corners) against the
  oracle's window statistics (oracle/firstorder_np.py), and a repeat of the first-order maps slab by slab compared bit
  for bit.

    python scripts/bench_firstorder.py [--reps 3] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import bench  # noqa: E402  (the bench volumes, the sampled centres, the card's name and power limit)

ENV = "B200_RADIOMICS_FORCE_GENERIC"


def _set_generic(on):
    os.environ[ENV] = "1" if on else "0"


def kernel_times(vol, reps):
    import torch
    from pyradiomics_b200 import voxel
    lev = torch.from_numpy(vol.astype(np.uint8)).cuda()
    raw = torch.from_numpy(bench.raw_from_levels(vol)).cuda()
    roi = torch.ones(vol.shape, dtype=torch.uint8, device="cuda")
    launch = voxel.firstorder_launch(raw, lev, roi, (1, 1, 1))
    outs = {k: torch.empty((voxel.FIRSTORDER_NF,) + vol.shape, dtype=torch.float64, device="cuda") for k in ("generic", "tiles")}
    ms = {"generic": [], "tiles": []}
    for rep in range(reps + 1):                     # rep 0 warms both up
        for name in ("generic", "tiles"):
            _set_generic(name == "generic")
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            launch(0, vol.shape[0], outs[name])
            b.record()
            b.synchronize()
            if rep:
                ms[name].append(a.elapsed_time(b))
    os.environ.pop(ENV, None)
    same = bool(torch.equal(outs["generic"].view(torch.int64), outs["tiles"].view(torch.int64)))
    row = {"bit_identical": same}
    for k, v in ms.items():
        v = np.array(v)
        row[k] = {"median_ms": float(np.median(v)), "spread_ms": float(v.max() - v.min()),
                  "runs": [round(float(x), 3) for x in v]}
    row["tiles_over_generic"] = row["tiles"]["median_ms"] / row["generic"]["median_ms"]
    # faster by more than the spread: the slowest tile run beats the fastest generic run by more than either spread
    gap = min(ms["generic"]) - max(ms["tiles"])
    row["faster_by_more_than_spread"] = bool(gap > max(row["generic"]["spread_ms"], row["tiles"]["spread_ms"]))
    del outs
    torch.cuda.empty_cache()
    return row


def config4_volume(n):
    """bench.secondary_config4's volume: Gaussian-smoothed noise (sigma 2) scaled to 0..800, float64"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((n, n, n), generator=g, device="cuda", dtype=torch.float32)
    k = torch.tensor([np.exp(-0.5 * (i / 2.0) ** 2) for i in range(-6, 7)], device="cuda")
    k = (k / k.sum()).to(torch.float32)
    for ax in range(3):
        shape = [1, 1, 1, 1, 1]
        shape[2 + ax] = 13
        pad = [0, 0, 0]
        pad[ax] = 6
        x = torch.nn.functional.conv3d(x[None, None], k.view(shape), padding=pad)[0, 0]
    return ((x - x.min()) / (x.max() - x.min()) * 800.0).to(torch.float64)


def config4(n, rounds):
    import torch
    from pyradiomics_b200 import pipeline as PL
    from pyradiomics_b200._lib import CLASSES
    x = config4_volume(n)
    mask = torch.ones(x.shape, dtype=torch.uint8, device="cuda")
    variants = {"texture": CLASSES, "texture+firstorder": CLASSES + ("firstorder",)}
    for cl in variants.values():                     # warm-up
        PL.voxel_suite_with_filters(x[:64, :64, :64].contiguous(), mask[:64, :64, :64].contiguous(), classes=cl, binWidth=25)
    ms = {k: [] for k in variants}
    nimg = 0
    for _ in range(rounds):
        for k, cl in variants.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            info = PL.voxel_suite_with_filters(x, mask, classes=cl, binWidth=25)
            b.record()
            b.synchronize()
            nimg = len(info)
            ms[k].append(a.elapsed_time(b) / nimg)
    res = {"workload": f"original + wavelet coif1 (8) + LoG sigma 1,2,3 -> binWidth 25, synthetic {n}^3 float volume",
           "images": nimg}
    for k, v in ms.items():
        res[k] = {"ms_per_image": float(np.median(v)), "runs_ms_per_image": [round(float(t), 2) for t in v]}
    res["firstorder_ms_per_image"] = res["texture+firstorder"]["ms_per_image"] - res["texture"]["ms_per_image"]
    del x, mask
    torch.cuda.empty_cache()
    return res


def oracle_windows(raw, lev, vox, shift=0.0, vv=1.0):
    """the oracle's first-order statistics of the r = 1 windows of centres vox [3, V] (every voxel in the ROI)"""
    import firstorder_np as FO
    n = raw.shape[0]
    off = np.array([(a, b, c) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1)])
    idx = vox.T[:, None, :] + off[None]
    inside = ((idx >= 0) & (idx < n)).all(-1)
    cl = np.clip(idx, 0, n - 1)
    T = np.where(inside, raw[cl[..., 0], cl[..., 1], cl[..., 2]].astype(np.float64), np.nan)
    L = np.where(inside, lev[cl[..., 0], cl[..., 1], cl[..., 2]], 0)
    p = np.stack([(L == g).sum(1) for g in range(1, int(lev.max()) + 1)], 1).astype(float)
    p /= p.sum(1, keepdims=True)
    f = FO._features(T, p, shift, vv)
    return np.stack([f[k] for k in FO.NAMES])


def suite_512(oracle_voxels, slab=32):
    import torch
    from pyradiomics_b200 import _lib, voxel
    from pyradiomics_b200._lib import CLASSES
    n = 512
    nvox = n ** 3
    gb = 1e9
    vol = bench.synth_volume(n, "uniform")
    raw_np = bench.raw_from_levels(vol)
    lev = torch.from_numpy(vol.astype(np.uint8)).cuda()
    raw = torch.from_numpy(raw_np).cuda()
    roi = torch.ones(vol.shape, dtype=torch.uint8, device="cuda")
    s = _lib.make_settings(32, 32)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    outs = {c: torch.empty((_lib.lib().rb_num_features(_lib.CLASS_ID[c]),) + lev.shape, dtype=torch.float32, device="cuda")
            for c in CLASSES}
    fo = torch.empty((voxel.FIRSTORDER_NF,) + lev.shape, dtype=torch.float32, device="cuda")
    alive = voxel.glcm_alive_angles(lev, s)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    a, m, b = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    a.record()
    for c in CLASSES:
        voxel.voxel_features(c, lev, s, out=outs[c], out_z0=0, alive=alive if c == "glcm" else None)
    m.record()
    voxel.firstorder_features(raw, lev, roi, out=fo, out_z0=0)
    b.record()
    b.synchronize()
    wall = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated()
    vox = bench.sample_voxels(n, oracle_voxels, 7)
    got = fo[:, vox[0], vox[1], vox[2]].cpu().numpy().astype(np.float64)
    ref = oracle_windows(raw_np, vol, vox.astype(np.int64))
    err = np.abs(got - ref) / np.maximum(np.abs(ref), 1e-300)
    err = np.where((got == ref) | (np.isnan(got) & np.isnan(ref)), 0.0, err)
    identical = True
    buf = torch.empty((voxel.FIRSTORDER_NF, slab, n, n), dtype=torch.float32, device="cuda")
    for z0 in range(0, n, slab):
        voxel.firstorder_features(raw, lev, roi, z0=z0, z1=z0 + slab, out=buf, out_z0=z0)
        identical &= bool(torch.equal(buf.view(torch.int32), fo[:, z0:z0 + slab].view(torch.int32)))
    return {"volume": "512^3 uniform levels 1..32 (bench.synth_volume), raw int16 (level - 1) * 25 + 3",
            "maps": "75 texture + 18 first-order, float32",
            "device_ms_total": a.elapsed_time(b), "device_ms_texture": a.elapsed_time(m), "device_ms_firstorder": m.elapsed_time(b),
            "wall_s": wall, "peak_max_memory_allocated_gb": peak / gb,
            "oracle_sample": {"voxels": int(vox.shape[1]), "on_faces_edges_corners": int((np.arange(vox.shape[1]) % 4 == 0).sum()),
                              "max_rel_err": float(err.max()), "within_float32_rounding": bool(err.max() <= 2 ** -23)},
            "repeat_bit_identical_slab_by_slab": identical}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--config4-rounds", type=int, default=2)
    ap.add_argument("--oracle-voxels", type=int, default=2048)
    ap.add_argument("--no-512", action="store_true")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_firstorder.py needs a CUDA device")
    line = {"what": "voxel-based first order at kernelRadius 1: generic kernel vs tile kernel, and in the filter suite",
            "gpu": bench.gpu_info(0)}
    for kind in ("uniform", "smooth"):
        line[f"kernel_256_{kind}"] = kernel_times(bench.synth_volume(256, kind), args.reps)
    line["config4_256"] = config4(256, args.config4_rounds)
    line["suite_512_float32_with_firstorder"] = {"skipped": "--no-512"} if args.no_512 else suite_512(args.oracle_voxels)
    line["gpu_after"] = bench.gpu_info(0)
    txt = json.dumps(line)
    print(txt)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
