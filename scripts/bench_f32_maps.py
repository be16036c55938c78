"""Float32 voxel maps written by the texture kernels (rb_voxel_features_dev, out_is_f32 = 1) against float64: one JSON line.

* 256^3 uniform and smooth volumes (bench.py's): per-class CUDA-event time of the fused kernel, float64 and float32
  alternating, median and spread of --reps runs each; bytes the maps take per class; the suite's voxels/s in both modes.
* The plugin end to end (featureclasses, b200_map_dtype="float32", host maps out) with this tree and with another
  checkout given by --baseline-root (its package, and its built library through B200_RADIOMICS_LIB), alternated in fresh
  processes: ms per step.
* The device-resident 512^3 full suite in float32 on one GPU (75 maps, 40.3 GB): voxels/s, peak
  torch.cuda.max_memory_allocated, a sampled oracle comparison (bench.py's: centres a quarter on faces / edges / corners,
  1e-5 relative) and a repeat run compared bit for bit, slab by slab.  Skipped, with the free memory recorded, when the
  card has less free memory than the run needs.

    python scripts/bench_f32_maps.py [--baseline-root DIR] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import bench  # noqa: E402  (the bench volumes, the CPU oracle arm, the parity check, the card's name and power limit)

CLASSES = bench.CLASSES


def class_times(vol, reps):
    """{class: {dtype: [ms per run]}}, float64 and float32 alternating, after one warm-up of each"""
    import torch
    from pyradiomics_b200 import _lib, voxel
    lev = torch.from_numpy(vol.astype(np.uint8)).cuda()
    s = _lib.make_settings(32, 32)
    res = {}
    for c in CLASSES:
        nf = _lib.lib().rb_num_features(_lib.CLASS_ID[c])
        outs = {dt: torch.empty((nf,) + vol.shape, dtype=dt, device="cuda") for dt in (torch.float64, torch.float32)}
        alive = voxel.glcm_alive_angles(lev, s) if c == "glcm" else None
        for dt in outs:
            voxel.voxel_features(c, lev, s, out=outs[dt], out_z0=0, alive=alive)
        ms = {"float64": [], "float32": []}
        for _ in range(reps):
            for dt, name in ((torch.float64, "float64"), (torch.float32, "float32")):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                voxel.voxel_features(c, lev, s, out=outs[dt], out_z0=0, alive=alive)
                b.record()
                b.synchronize()
                ms[name].append(a.elapsed_time(b))
        ref = outs[torch.float64].to(torch.float32)
        nan = torch.isnan(ref)
        same = bool(torch.equal(torch.isnan(outs[torch.float32]), nan) and torch.equal(
            outs[torch.float32].masked_fill(nan, 0).view(torch.int32), ref.masked_fill(nan, 0).view(torch.int32)))
        res[c] = {"ms": ms, "nf": nf, "float32_equals_rounded_float64": same}
        del outs, ref, nan
        torch.cuda.empty_cache()
    return res


def summarise(res, nvox):
    out, tot = {}, {"float64": 0.0, "float32": 0.0}
    for c, r in res.items():
        row = {"maps": r["nf"], "float32_equals_rounded_float64": r["float32_equals_rounded_float64"]}
        for dt, esz in (("float64", 8), ("float32", 4)):
            v = np.array(r["ms"][dt])
            row[dt] = {"median_ms": float(np.median(v)), "min_ms": float(v.min()), "max_ms": float(v.max()),
                       "runs": [round(float(x), 3) for x in v], "bytes_written": r["nf"] * nvox * esz}
            tot[dt] += float(np.median(v))
        row["float32_over_float64"] = row["float32"]["median_ms"] / row["float64"]["median_ms"]
        out[c] = row
    out["suite"] = {dt: {"ms": tot[dt], "voxels_per_s": nvox / (tot[dt] * 1e-3)} for dt in tot}
    return out


def e2e_child(steps):
    """one process: the plugin end to end with float32 maps on the package first on sys.path"""
    import torch
    ctx = bench.Ctx(argparse.Namespace(gpus=1, no_numa_bind=True))
    r = bench.plugin_e2e(ctx, bench.synth_volume(256, "uniform"), steps, "float32")
    torch.cuda.synchronize()
    print(json.dumps({"ms_per_step": r["ms_per_step"], "probe": r["first_value_probe"]}))


def e2e_ab(baseline_root, rounds, steps):
    runs = {"this_build": [], "baseline": []}
    probes = {}
    for _ in range(rounds):
        for name, root in (("this_build", ROOT), ("baseline", os.path.abspath(baseline_root))):
            env = dict(os.environ, B200_RADIOMICS_LIB=os.path.join(root, "pyradiomics_b200", "libb200radiomics.so"))
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--e2e-child", str(steps), "--child-root", root],
                               env=env, capture_output=True, text=True, cwd=root)
            if p.returncode:
                return {"error": f"{name}: exit {p.returncode}: {p.stderr[-800:]}"}
            line = json.loads(p.stdout.strip().splitlines()[-1])
            runs[name].append(line["ms_per_step"])
            probes[name] = line["probe"]
    med = {k: float(np.median(v)) for k, v in runs.items()}
    return {"ms_per_step": {k: [round(x, 1) for x in v] for k, v in runs.items()}, "median_ms_per_step": med,
            "this_over_baseline": med["this_build"] / med["baseline"], "first_value_probe": probes,
            "steps_per_process": steps, "volume": "256^3 uniform, int16 raw, binWidth=25, b200_map_dtype=float32",
            "baseline": "a checkout of the parent commit with its library built"}


def suite_512(oracle, slab=64):
    import torch
    from pyradiomics_b200 import _lib, voxel
    n = 512
    nvox = n ** 3
    need = sum(_lib.lib().rb_num_features(_lib.CLASS_ID[c]) for c in CLASSES) * nvox * 4
    free, total = torch.cuda.mem_get_info()
    gb = 1e9
    # maps + levels + the GLCM queue (1.15 GB) + a repeat slab of the largest class + slack
    want = need + nvox + int(1.2 * gb) + 24 * slab * n * n * 4 + int(0.5 * gb)
    if free < want:
        return {"skipped": f"free memory {free / gb:.1f} GB", "needs_gb": want / gb}
    vol = bench.synth_volume(n, "uniform")
    lev = torch.from_numpy(vol.astype(np.uint8)).cuda()
    del vol
    s = _lib.make_settings(32, 32)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    outs = {c: torch.empty((_lib.lib().rb_num_features(_lib.CLASS_ID[c]),) + lev.shape, dtype=torch.float32, device="cuda")
            for c in CLASSES}
    alive = voxel.glcm_alive_angles(lev, s)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for c in CLASSES:
        voxel.voxel_features(c, lev, s, out=outs[c], out_z0=0, alive=alive if c == "glcm" else None)
    b.record()
    b.synchronize()
    wall = time.perf_counter() - t0
    ms = a.elapsed_time(b)
    peak = torch.cuda.max_memory_allocated()
    # repeat, slab by slab, compared bit for bit with the whole-volume run
    identical = True
    for c in CLASSES:
        buf = torch.empty((outs[c].shape[0], slab, n, n), dtype=torch.float32, device="cuda")
        for z0 in range(0, n, slab):
            voxel.voxel_features(c, lev, s, z0=z0, z1=z0 + slab, out=buf, out_z0=z0, alive=alive if c == "glcm" else None)
            identical &= bool(torch.equal(buf.view(torch.int32), outs[c][:, z0:z0 + slab].view(torch.int32)))
        del buf
    res = {"volume": "512^3 uniform levels 1..32 (bench.synth_volume)", "maps": "75 float32", "map_bytes": need,
           "device_ms": ms, "wall_s": wall, "voxels_per_s": nvox / (ms * 1e-3),
           "peak_max_memory_allocated_gb": peak / gb, "free_before_gb": free / gb, "total_gb": total / gb,
           "repeat_bit_identical_slab_by_slab": identical}
    if oracle is not None:
        res["parity_sample"] = bench.parity_of(outs, 0, oracle[0], oracle[1])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--baseline-root", default=None,
                    help="a checkout with its library built (the parent commit) for the plugin A/B (skipped if absent)")
    ap.add_argument("--e2e-rounds", type=int, default=3)
    ap.add_argument("--e2e-steps", type=int, default=2)
    ap.add_argument("--oracle-voxels", type=int, default=2048)
    ap.add_argument("--no-512", action="store_true")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    ap.add_argument("--e2e-child", type=int, default=None, help=argparse.SUPPRESS)
    ap.add_argument("--child-root", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--e2e-only", action="store_true", help="only the plugin A/B")
    args = ap.parse_args()
    if args.e2e_child is not None:
        sys.path.insert(0, args.child_root)
        return e2e_child(args.e2e_child)

    if args.e2e_only:
        print(json.dumps({"plugin_e2e_float32": e2e_ab(args.baseline_root, args.e2e_rounds, args.e2e_steps)}))
        return
    oracle = None
    if not args.no_512:        # CPU oracle first (fork-safe: CUDA not initialised yet)
        import multiprocessing as mp
        vol = bench.synth_volume(512, "uniform")
        cores = min(os.cpu_count() or 1, 64)
        per_worker = -(-args.oracle_voxels // cores)
        bench.cpu_arm_setup(vol)
        pool = mp.get_context("fork").Pool(cores) if cores > 1 else None
        _, dt, vox, feats = bench.cpu_arm_step(vol, cores, per_worker, 0, pool, keep=True)
        if pool:
            pool.close()
        oracle = (vox, feats)
        del vol
        bench._CPU.clear()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_f32_maps.py needs a CUDA device")
    line = {"what": "float32 voxel maps written by the texture kernels vs float64", "gpu": bench.gpu_info(0)}
    for kind in ("uniform", "smooth"):
        vol = bench.synth_volume(256, kind)
        line[f"classes_256_{kind}"] = summarise(class_times(vol, args.reps), vol.size)
    if args.baseline_root:
        line["plugin_e2e_float32"] = e2e_ab(args.baseline_root, args.e2e_rounds, args.e2e_steps)
    else:
        line["plugin_e2e_float32"] = {"skipped": "no --baseline-root"}
    torch.cuda.empty_cache()
    line["suite_512_float32"] = {"skipped": "--no-512"} if args.no_512 else suite_512(oracle)
    line["gpu_after"] = bench.gpu_info(0)
    txt = json.dumps(line)
    print(txt)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
