"""Voxel maps at kernelRadius 2 to 7: the generic thread-per-centre kernels (windows of <= 343 positions) and the wide
block-per-centre kernels (344 to 3375 positions).  One JSON line.

* bench.py's uniform and smooth volumes (Ng 32) at --size^3: per texture class and first order, CUDA-event time of one
  whole-volume call, at r = 2 and 3 (generic) and r = 4, 5 and 7 (wide); each kernel is warmed up at its first radius.
  The default size is 48: GLCM's entry lists are searched linearly by one thread per angle, on both paths, and one
  128^3 call took 22.9 s at r = 3 (generic) and 110.6 s at r = 4 (wide) on the uniform volume.
* r = 3 through the generic kernels and the wide kernels forced (B200_RADIOMICS_FORCE_WIDE=1), alternated --reps times
  in this process: which side of the 343-position line each path wins on, and whether their maps are the same bits.
* A sampled oracle comparison at every wide radius (the window oracle of tests/helpers.py on --samples centres of the
  smooth volume: worst |got - ref| / max(|ref|, 1) per class), and a repeat run of every wide call compared bit for bit.
* The card's name and power limit.

    python scripts/bench_wide_windows.py [--size 48] [--reps 3] [--samples 6] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import bench  # noqa: E402  (the bench volumes, the card's name and power limit)

CLASSES = bench.CLASSES + ("firstorder",)


def _same_bits(a, b):
    import torch
    na, nb = torch.isnan(a), torch.isnan(b)
    if not torch.equal(na, nb):
        return False
    return torch.equal(torch.where(na, torch.zeros_like(a), a).view(torch.int64),
                       torch.where(nb, torch.zeros_like(b), b).view(torch.int64))


class Volume:
    def __init__(self, vol):
        import torch
        from pyradiomics_b200 import _lib, voxel
        self.vol = vol
        self.lev = torch.from_numpy(vol.astype(np.uint8)).cuda()
        self.img = torch.from_numpy(bench.raw_from_levels(vol)).cuda()
        self.roi = torch.ones(vol.shape, dtype=torch.uint8, device="cuda")
        self.alive = {}
        self._lib, self._voxel = _lib, voxel

    def call(self, cname, r, out):
        """one whole-volume call of class cname at kernelRadius r into out (float64)"""
        if cname == "firstorder":
            return self._voxel.firstorder_features(self.img, self.lev, self.roi, kernelRadius=r, out=out, out_z0=0)
        s = self._lib.make_settings(32, 32, kernelRadius=r)
        if cname == "glcm" and r not in self.alive:
            self.alive[r] = self._voxel.glcm_alive_angles(self.lev, s)
        return self._voxel.voxel_features(cname, self.lev, s, out=out, out_z0=0,
                                          alive=self.alive.get(r) if cname == "glcm" else None)

    def timed(self, cname, r, out):
        import torch
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        self.call(cname, r, out)
        b.record()
        b.synchronize()
        return a.elapsed_time(b)


def nfeat(cname):
    from pyradiomics_b200 import _lib
    return 18 if cname == "firstorder" else _lib.lib().rb_num_features(_lib.CLASS_ID[cname])


def oracle_error(V, cname, r, out, centres):
    """worst |got - ref| / max(|ref|, 1) over the sampled centres (NaN where the oracle has NaN), or a string on a NaN
    mismatch"""
    from helpers import FAST_NAMES, WindowRun, box_features, box_mcc, window_box
    if cname == "firstorder":
        import firstorder_np as FO
        err = 0.0
        raw = bench.raw_from_levels(V.vol).astype(np.float64)
        for c in centres:
            sl = tuple(slice(max(0, c[d] - r), c[d] + r + 1) for d in range(3))
            win = raw[sl].ravel()
            lv = V.vol[sl].ravel()
            _, cnt = np.unique(lv, return_counts=True)
            ref = FO._features(np.sort(win)[None, :], (cnt / cnt.sum())[None, :], 0, 1.0)
            got = out[(slice(None),) + tuple(int(x) for x in c)].cpu().numpy()
            for k, f in enumerate(FO.NAMES):
                rv = float(np.squeeze(ref[f]))
                err = max(err, abs(got[k] - rv) / max(abs(rv), 1.0))
        return err
    run = WindowRun(V.vol.shape, 32, kernelRadius=r)
    err = 0.0
    for c in centres:
        box = window_box(V.vol, c, run.radii)
        f = box_features(box, cname, run)
        if cname == "glcm":
            f["MCC"] = box_mcc(box, run)[0]
        got = out[(slice(None),) + tuple(int(x) for x in c)].cpu().numpy()
        for k, name in enumerate(FAST_NAMES[cname]):
            rv, gv = f[name], got[k]
            if np.isnan(rv) or np.isnan(gv):
                if np.isnan(rv) != np.isnan(gv):
                    return f"NaN mismatch at {tuple(c)} {name}"
                continue
            err = max(err, abs(gv - rv) / max(abs(rv), 1.0))
    return err


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=48)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--samples", type=int, default=6)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_wide_windows: no CUDA device; the timings need an H100")
    n = args.size
    res = {"what": "scripts/bench_wide_windows.py: per-class CUDA-event time of one whole-volume voxel-map call, generic "
                   "kernels at r = 2, 3 and wide kernels at r = 4, 5, 7; generic vs forced wide at r = 3 alternated",
           "size": n, "gpu": bench.gpu_info(0), "volumes": {}}
    rng = np.random.default_rng(7)
    for kind in ("uniform", "smooth"):
        V = Volume(bench.synth_volume(n, kind))
        outs = {c: torch.empty((nfeat(c), n, n, n), dtype=torch.float64, device="cuda") for c in CLASSES}
        per = {}
        for r in (2, 3, 4, 5, 7):
            path = "generic" if (2 * r + 1) ** 3 <= 343 else "wide"
            row = {"path": path, "positions": (2 * r + 1) ** 3}
            centres = rng.integers(0, n, (args.samples, 3))
            for c in CLASSES:
                if r in (2, 4):
                    V.call(c, r, outs[c])                           # warm-up of each kernel path
                ms = V.timed(c, r, outs[c])
                d = {"ms": round(ms, 3), "voxels_per_s": round(n ** 3 / (ms / 1e3), 1)}
                if path == "wide":
                    again = torch.empty_like(outs[c])
                    V.call(c, r, again)
                    d["repeat_same_bits"] = bool(_same_bits(again, outs[c]))
                    del again
                    if kind == "smooth":
                        d["oracle_worst_rel"] = oracle_error(V, c, r, outs[c], centres)
                row[c] = d
                print(kind, r, c, d, file=sys.stderr, flush=True)
            per[f"r{r}"] = row
        # r = 3 both ways, alternated
        ab = {}
        for c in CLASSES:
            other = torch.empty_like(outs[c])
            t = {"generic": [], "wide": []}
            for _ in range(args.reps):
                for name, buf in (("generic", outs[c]), ("wide", other)):
                    if name == "wide":
                        os.environ["B200_RADIOMICS_FORCE_WIDE"] = "1"
                    try:
                        V.call(c, 3, buf)
                        t[name].append(V.timed(c, 3, buf))
                    finally:
                        os.environ.pop("B200_RADIOMICS_FORCE_WIDE", None)
            ab[c] = {k: {"ms_median": round(float(np.median(v)), 3), "ms_min": round(min(v), 3), "ms_max": round(max(v), 3)}
                     for k, v in t.items()}
            ab[c]["same_bits"] = bool(_same_bits(other, outs[c]))
            ab[c]["wide_over_generic"] = round(ab[c]["wide"]["ms_median"] / ab[c]["generic"]["ms_median"], 2)
            print(kind, "r3 A/B", c, ab[c], file=sys.stderr, flush=True)
            del other
        per["r3_generic_vs_wide"] = ab
        res["volumes"][kind] = per
        del outs, V
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
