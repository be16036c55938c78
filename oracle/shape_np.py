"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's shape path.

* ``coefficients(mask, spacing)`` follows radiomics/src/cshape.c:22-242 (calculate_coefficients +
  calculate_meshDiameter): marching cube over every 2x2x2 neighbourhood, surface area and signed
  origin volume per triangle, mesh vertices on the three cube edges that meet at corner (z+1, y+1, x),
  O(V^2) diameters.  The triangle table is the product's generated one (csrc/mc_table.inc, derived from
  geometry and pinned on the reference's single-cube outputs, see csrc/gen_mc_table.py); parity of this
  restatement is pinned by tests/golden/shape_cube_probes.npz, shape_random.npz and shape_expect.json
  (all produced by the compiled reference, tests/golden/make_golden.py --shape-only).
* ``features(mask, spacing)`` follows radiomics/shape.py:54-424.

Pure Python loops: only for small masks.  Only tests/ may import this.
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "pyradiomics_b200", "csrc"))
import gen_mc_table  # noqa: E402

_MID2, _TRI = gen_mc_table.load_table()


def coefficients(mask, spacing):
    m = np.asarray(mask) != 0
    sp = np.asarray(spacing, dtype=np.float64)
    Z, Y, X = m.shape
    area = vol6 = 0.0
    verts = []
    for iz in range(Z - 1):
        for iy in range(Y - 1):
            for ix in range(X - 1):
                cfg = 0
                for c in range(8):
                    if m[iz + (c >> 2 & 1), iy + (c >> 1 & 1), ix + (c & 1)]:
                        cfg |= 1 << c
                own = cfg >> 6 & 1                                   # corner (1,1,0), cshape.c:94-112
                if (cfg >> 7 & 1) != own:
                    verts.append(((iz + 1.0) * sp[0], (iy + 1.0) * sp[1], (ix + 0.5) * sp[2]))
                if (cfg >> 4 & 1) != own:
                    verts.append(((iz + 1.0) * sp[0], (iy + 0.5) * sp[1], (ix + 0.0) * sp[2]))
                if (cfg >> 2 & 1) != own:
                    verts.append(((iz + 0.5) * sp[0], (iy + 1.0) * sp[1], (ix + 0.0) * sp[2]))
                row = _TRI[cfg]
                for k in range(0, 15, 3):
                    if row[k] < 0:
                        break
                    a, b, c3 = ((np.array([iz, iy, ix], dtype=np.float64) + 0.5 * _MID2[row[k + v]]) * sp for v in range(3))
                    vol6 += float(np.dot(np.cross(a, b), c3))                    # cshape.c:143-149
                    area += 0.5 * float(np.linalg.norm(np.cross(a - c3, b - c3)))    # cshape.c:158-178
    dia = [0.0, 0.0, 0.0, 0.0]
    if verts:
        v = np.array(verts)
        for i in range(len(v)):                                       # cshape.c:192-242
            d = v[i] - v[: i + 1]
            d2 = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]
            for q in range(3):
                sel = d2[v[: i + 1, q] == v[i, q]]
                if sel.size:
                    dia[q] = max(dia[q], float(sel.max()))
            dia[3] = max(dia[3], float(d2.max()))
    return area, vol6 / 6.0, tuple(float(np.sqrt(x)) for x in dia)


def features(mask, spacing_zyx):
    """the 14 active + 3 deprecated shape features of a (not yet padded) ROI mask, shape.py:54-424"""
    sp = np.asarray(spacing_zyx, dtype=np.float64)
    m = np.pad(np.asarray(mask) != 0, 1)
    sa, vol, dia = coefficients(m, sp)
    idx = np.array(np.where(m), dtype=np.float64).T
    n = len(idx)
    phys = idx * sp[None, :]
    phys -= phys.mean(0)
    phys /= np.sqrt(n)
    ev = np.linalg.eigvals(phys.T.copy() @ phys)
    ev[(ev < 0) & (ev > -1e-10)] = 0
    ev = np.sort(ev)
    f = {"MeshVolume": vol, "VoxelVolume": n * float(np.prod(sp)), "SurfaceArea": sa, "SurfaceVolumeRatio": sa / vol,
         "Sphericity": (36 * np.pi * vol ** 2) ** (1.0 / 3.0) / sa,
         "Compactness1": vol / (sa ** 1.5 * np.sqrt(np.pi)), "Compactness2": 36.0 * np.pi * vol ** 2 / sa ** 3,
         "SphericalDisproportion": sa / (36 * np.pi * vol ** 2) ** (1.0 / 3.0),
         "Maximum3DDiameter": dia[3], "Maximum2DDiameterSlice": dia[0], "Maximum2DDiameterColumn": dia[1],
         "Maximum2DDiameterRow": dia[2]}
    neg = lambda k: ev[k] < 0
    f["MajorAxisLength"] = np.nan if neg(2) else float(np.sqrt(ev[2]) * 4)
    f["MinorAxisLength"] = np.nan if neg(1) else float(np.sqrt(ev[1]) * 4)
    f["LeastAxisLength"] = np.nan if neg(0) else float(np.sqrt(ev[0]) * 4)
    f["Elongation"] = np.nan if (neg(1) or neg(2)) else float(np.sqrt(ev[1] / ev[2]))
    f["Flatness"] = np.nan if (neg(0) or neg(2)) else float(np.sqrt(ev[0] / ev[2]))
    return f


def coefficients2d(mask, spacing):
    """CPU restatement of calculate_coefficients2D + calculate_meshDiameter2D (radiomics/src/cshape.c:420-595) for an
    already zero-padded 2-D mask: marching squares with edge-midpoint vertices.  Per 2x2 neighbourhood the reference's
    16-entry line table amounts to: 1 or 3 inside corners -> one corner cut (:460-500); two adjacent corners -> one
    straight cut; the two diagonal configurations -> two corner cuts that keep the inside corners apart (probed on the
    compiled reference: [[1,0],[0,1]] has surface 1.0).  The surface is accumulated like the reference does, as half the
    sum of the cross products of the ORIENTED segment end points (:483), and the vertices kept for the diameter are the
    midpoints of the crossed left / bottom square edges (:514-535).  Pinned on the compiled reference (_cshape) by
    tests/golden/shape2d_golden.npz."""
    m = np.asarray(mask) != 0
    sy, sx = float(spacing[0]), float(spacing[1])
    Y, X = m.shape
    per = 0.0
    cross = 0.0
    verts = []
    mid = {0: (0.0, 0.5), 1: (0.5, 1.0), 2: (1.0, 0.5), 3: (0.5, 0.0)}        # edge midpoints: top, right, bottom, left
    corner = [(0, 0), (0, 1), (1, 1), (1, 0)]                                  # p0..p3, clockwise from the origin
    for iy in range(Y - 1):
        for ix in range(X - 1):
            ins = [bool(m[iy + dy, ix + dx]) for dy, dx in corner]
            k = sum(ins)
            if k in (0, 4):
                continue
            # segments: walk the square's edges clockwise (edge e joins corner e and e+1); a segment starts where the
            # boundary goes inside -> outside and ends at the next outside -> inside crossing, so the inside stays on
            # one side of every oriented segment (the diagonal cases pair each inside corner with its own two edges)
            outs = [e for e in range(4) if ins[e] and not ins[(e + 1) % 4]]
            for e in outs:
                f = e
                while True:
                    f = (f + 1) % 4
                    if not ins[f] and ins[(f + 1) % 4]:
                        break
                if k == 2 and ins[0] == ins[2]:          # diagonal: keep the corners apart -> the closing edge is the one BEFORE e
                    f = (e - 1) % 4
                a = ((iy + mid[e][0]) * sy, (ix + mid[e][1]) * sx)
                b = ((iy + mid[f][0]) * sy, (ix + mid[f][1]) * sx)
                cross += a[0] * b[1] - b[0] * a[1]
                per += float(np.sqrt((a[0] - b[0]) ** 2 + (a[1] - b[1]) ** 2))
            if ins[0] != ins[3]:
                verts.append(((iy + 0.5) * sy, ix * sx))
            if ins[3] != ins[2]:
                verts.append(((iy + 1.0) * sy, (ix + 0.5) * sx))
    v = np.array(verts, dtype=np.float64).reshape(-1, 2)
    d2 = 0.0
    for i in range(len(v)):
        if i:
            dy = v[i, 0] - v[:i, 0]
            dx = v[i, 1] - v[:i, 1]
            d2 = max(d2, float((dy * dy + dx * dx).max()))
    return per, abs(cross) / 2.0, float(np.sqrt(d2))


def features2d(mask, spacing_yx):
    """the 9 active + 1 deprecated 2-D shape features of a (not yet padded) 2-D ROI mask, shape2D.py:40-300"""
    sp = np.asarray(spacing_yx, dtype=np.float64)
    m = np.pad(np.asarray(mask) != 0, 1)
    per, sur, dia = coefficients2d(m, sp)
    idx = np.array(np.where(m), dtype=np.float64).T
    n = len(idx)
    phys = idx * sp[None, :]
    phys -= phys.mean(0)
    phys /= np.sqrt(n)
    ev = np.linalg.eigvals(phys.T.copy() @ phys).real
    ev[(ev < 0) & (ev > -1e-10)] = 0
    ev = np.sort(ev)
    sph = (2 * np.sqrt(np.pi * sur)) / per
    return {"MeshSurface": sur, "PixelSurface": n * float(np.prod(sp)), "Perimeter": per, "PerimeterSurfaceRatio": per / sur,
            "Sphericity": sph, "SphericalDisproportion": 1.0 / sph, "MaximumDiameter": dia,
            "MajorAxisLength": np.nan if ev[1] < 0 else float(np.sqrt(ev[1]) * 4),
            "MinorAxisLength": np.nan if ev[0] < 0 else float(np.sqrt(ev[0]) * 4),
            "Elongation": np.nan if (ev[0] < 0 or ev[1] < 0) else float(np.sqrt(ev[0] / ev[1]))}


# ---------------------------------------------------------------------------------------------------------------------
# Vectorised counterparts of coefficients / coefficients2d for large masks (about 200^3 voxels, 10^6 pixels): the same
# table and vertex-ownership rule, no O(V^2) loop.
#
# With spacings of few mantissa bits (0.5, 0.75, 1.25, ...) every coordinate ((index + offset) * spacing), difference,
# product and six-fold tetrahedron volume is an exact double, so the kernels' per-triangle terms are known bit for bit:
# ``mesh`` reports ``exact`` = True, the six-fold volume as a Python int, the area terms, and the four squared
# diameters as exact integers.  For any other spacing it gives the same quantities in the reference's own double
# operations (terms, not sums, are bit-reproducible) plus per-term rounding magnitudes for an error bound.
U = 2.0 ** -53                                   # unit roundoff of float64


def _dyadic(s):
    """(numerator, log2 denominator) of a double"""
    from fractions import Fraction
    f = Fraction(float(s))
    k = f.denominator.bit_length() - 1
    assert f.denominator == 1 << k
    return f.numerator, k


def _hull(p):
    """strict convex hull (monotone chain, integer arithmetic) of lexicographically sorted, distinct 2-D points: the
    positions of its vertices in p"""
    if len(p) <= 2:
        return list(range(len(p)))
    pts = p.tolist()

    def half(order):
        h = []
        for i in order:
            x, y = pts[i]
            while len(h) >= 2:
                (ax, ay), (bx, by) = pts[h[-2]], pts[h[-1]]
                if (bx - ax) * (y - ay) - (by - ay) * (x - ax) > 0:
                    break
                h.pop()
            h.append(i)
        return h

    lo, up = half(range(len(pts))), half(range(len(pts) - 1, -1, -1))
    return lo[:-1] + up[:-1]


def _sq_float(h, sp):
    """coordinates (0.5 * half-index) * spacing, as the reference and the kernels form them"""
    return [(0.5 * h[:, d].astype(np.float64)) * sp[d] for d in range(h.shape[1])]


def _max_d2(hi, hj, sp, scale):
    """max squared distance over all pairs (hi x hj): the float value in the reference's operation order, and the exact
    integer value in units of `scale` (per-axis integer factors) or None"""
    a, b = _sq_float(hi, sp), _sq_float(hj, sp)
    best_f, best_i = 0.0, 0
    step = max(1, (1 << 22) // max(1, len(hj)))
    for r in range(0, len(hi), step):
        s = slice(r, r + step)
        d2 = None
        for d in range(len(sp)):
            t = a[d][s, None] - b[d][None, :]
            t = t * t
            d2 = t if d2 is None else d2 + t
        best_f = max(best_f, float(d2.max()))
        if scale is not None:
            e = sum(((hi[s, d, None] - hj[None, :, d]) ** 2) * scale[d] for d in range(len(sp)))
            best_i = max(best_i, int(e.max()))
    return best_f, (best_i if scale is not None else None)


def _plane_candidates(h, q):
    """per plane h[:, q] = const: the vertices of that plane's 2-D convex hull (indices into h), plane by plane.
    A point that is not extreme in its row of the plane cannot be a hull vertex, so the rows' end points are
    pruned to first (vectorised) and the hull is built on those alone."""
    o1, o2 = [d for d in range(3) if d != q] if h.shape[1] == 3 else (0, 1)
    order = np.lexsort((h[:, o2], h[:, o1], h[:, q])) if h.shape[1] == 3 else np.lexsort((h[:, 1], h[:, 0]))
    hs = h[order]
    key = hs[:, [q, o1]] if h.shape[1] == 3 else hs[:, [0]]
    brk = np.ones(len(hs) + 1, bool)
    brk[1:-1] = (key[1:] != key[:-1]).any(1)
    first, last = np.nonzero(brk[:-1])[0], np.nonzero(brk[1:])[0]
    cand = np.unique(np.concatenate([first, last]))                      # row ends, still in lexicographic order
    plane = hs[cand, q] if h.shape[1] == 3 else np.zeros(len(cand), np.int64)
    cuts = np.nonzero(np.diff(plane))[0] + 1
    out = []
    for grp in np.split(np.arange(len(cand)), cuts):
        idx = cand[grp]
        pts = hs[idx][:, [o1, o2]]
        out.append(order[idx[_hull(pts)]])
    return out


def _diameters(h, sp, exact):
    """diameters of vertex set h (half-index ints, [n, nd]): per-plane maxima for nd = 3 (equal z, equal y, equal x)
    and the overall maximum; floats (squared, reference operation order) and exact integers (or None)"""
    nd = h.shape[1]
    if exact:
        dy = [_dyadic(s) for s in sp]
        kmax = max(k for _, k in dy)
        scale = [n * n * 4 ** (kmax - k) for n, k in dy]            # squared distance in units 4^-(kmax+1)
    else:
        scale = None
    if len(h) == 0:
        return [0.0] * (4 if nd == 3 else 1), ([0] * (4 if nd == 3 else 1) if exact else None)
    hull_sets, dia_f, dia_i = [], [], []
    for q in (range(3) if nd == 3 else [0]):
        planes = _plane_candidates(h, q)
        bf, bi = 0.0, 0
        for ids in planes:
            f, i = _max_d2(h[ids], h[ids], sp, scale)
            bf, bi = max(bf, f), (max(bi, i) if exact else None)
        hull_sets.append(np.concatenate(planes))
        dia_f.append(bf)
        dia_i.append(bi)
    if nd == 3:
        # a vertex of the 3-D hull is a vertex of the hull of each of its three planes
        c = np.intersect1d(np.intersect1d(hull_sets[0], hull_sets[1]), hull_sets[2])
        f, i = _max_d2(h[c], h[c], sp, scale)
        dia_f.append(f)
        dia_i.append(i)
    if exact:
        unit = 4.0 ** -(kmax + 1)
        for f, i in zip(dia_f, dia_i):
            assert i < 2 ** 53 and f == i * unit, (f, i)       # the kernels' double squares and sums are exact too
    return dia_f, (dia_i if exact else None)


def _corner(m, c):
    """corner c (bit 2: z, bit 1: y, bit 0: x) of every 2x2x2 cube of m"""
    Z, Y, X = m.shape
    dz, dy, dx = c >> 2 & 1, c >> 1 & 1, c & 1
    return m[dz:Z - 1 + dz, dy:Y - 1 + dy, dx:X - 1 + dx]


def mesh(mask, spacing):
    """Marching cubes over every 2x2x2 neighbourhood of a 3-D mask, vectorised.  Returns a dict:

    exact        spacing and extent keep every term exact (see above)
    vol6         exact six-fold volume (Python int, in units vol6_unit) when exact, else None
    vol6_unit    2^-(k0 + k1 + k2 + 3) for spacings n_d * 2^-k_d
    vol_terms_abs  sum |six-fold tetra term| (float; exact when exact)
    vol_fsum     correctly rounded sum of the per-triangle six-fold terms (double operations of the reference)
    vol_mag      sum over triangles of the six |monomials| of the triple product: per-term rounding scale
    area_fsum    correctly rounded sum of the per-triangle area terms (bit-equal to the kernels' terms when exact)
    area_terms   (distinct values, counts) of the area terms
    area_mag     sum over triangles of (|a| + |b| + 2|c|) * (|a - c| + |b - c|): per-term rounding scale of the area
    n_tri        number of triangles, n_verts the exact number of mesh vertices, verts their half-index coordinates
    dia2         four squared diameters (equal z, equal y, equal x, all) in the reference's double operations
    dia2_exact   the same as exact integers in units 4^-(kmax + 1) when exact, else None; dia2_unit that unit
    dia          the four diameters sqrt(dia2)"""
    from fractions import Fraction
    m = np.asarray(mask) != 0
    sp = [float(s) for s in spacing]
    Z, Y, X = m.shape
    out = {"n_tri": 0, "n_verts": 0}
    if min(Z, Y, X) < 2:
        return dict(out, verts=np.zeros((0, 3), np.int64), exact=True, vol6=0, vol6_unit=1.0, vol_terms_abs=0.0, vol_fsum=0.0, vol_mag=0.0, area_fsum=0.0,
                    area_terms=(np.zeros(0), np.zeros(0, np.int64)), area_mag=0.0, dia2=[0.0] * 4, dia2_exact=[0] * 4,
                    dia2_unit=1.0, dia=[0.0] * 4)
    cfg = np.zeros((Z - 1, Y - 1, X - 1), np.uint8)
    for c in range(8):
        cfg |= _corner(m, c).astype(np.uint8) << c
    # vertices: the three edges meeting at corner (z+1, y+1, x) = bit 6, to bits 7 (x), 4 (y), 2 (z)
    own = _corner(m, 6)
    vs = []
    for bit, off in ((7, (2, 2, 1)), (4, (2, 1, 0)), (2, (1, 2, 0))):
        iz, iy, ix = np.nonzero(_corner(m, bit) != own)
        vs.append(np.stack([2 * iz + off[0], 2 * iy + off[1], 2 * ix + off[2]], 1).astype(np.int64))
    h = np.concatenate(vs)
    out.update(n_verts=len(h), verts=h)

    dy = [_dyadic(s) for s in sp]
    num = [n for n, _ in dy]
    hmax = [2 * (Z - 1), 2 * (Y - 1), 2 * (X - 1)]
    M = [hmax[d] * abs(num[d]) for d in range(3)]
    exact = 6 * M[0] * M[1] * M[2] < 2 ** 53 and all(M[d] < 2 ** 26 for d in range(3))

    flat = cfg.ravel()
    mixed = np.nonzero((flat != 0) & (flat != 255))[0]
    order = mixed[np.argsort(flat[mixed], kind="stable")]
    cfgs = flat[order]
    cuts = np.nonzero(np.diff(cfgs))[0] + 1
    vol6 = 0
    vol_abs_i = 0
    vol_terms, area_terms, vol_mag, area_mag = [], [], 0.0, 0.0
    for grp in np.split(order, cuts):
        if len(grp) == 0:
            continue
        c = int(flat[grp[0]])
        iz, r = np.divmod(grp, (Y - 1) * (X - 1))
        iy, ix = np.divmod(r, X - 1)
        base = np.stack([2 * iz, 2 * iy, 2 * ix], 1)
        row = _TRI[c]
        for k in range(0, 15, 3):
            if row[k] < 0:
                break
            hv = [base + _MID2[row[k + v]][None, :] for v in range(3)]           # half-index corners a, b, c
            a, b, cc = (_sq_float(x, sp) for x in hv)
            ab = [a[1] * b[2] - b[1] * a[2], a[2] * b[0] - b[2] * a[0], a[0] * b[1] - b[0] * a[1]]
            vol_terms.append(ab[0] * cc[0] + ab[1] * cc[1] + ab[2] * cc[2])
            mono = sum(np.abs(a[i] * b[j] * cc[l]) for i, j, l in ((1, 2, 0), (2, 1, 0), (2, 0, 1), (0, 2, 1),
                                                                      (0, 1, 2), (1, 0, 2)))
            vol_mag += float(mono.sum())
            x = [a[d] - cc[d] for d in range(3)]
            y = [b[d] - cc[d] for d in range(3)]
            cr = [x[1] * y[2] - y[1] * x[2], x[2] * y[0] - y[2] * x[0], x[0] * y[1] - y[0] * x[1]]
            area_terms.append(0.5 * np.sqrt(cr[0] * cr[0] + cr[1] * cr[1] + cr[2] * cr[2]))
            nrm = lambda v: np.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
            area_mag += float(((nrm(a) + nrm(b) + 2 * nrm(cc)) * (nrm(x) + nrm(y))).sum())
            if exact:
                P = [[hv[v][:, d] * num[d] for d in range(3)] for v in range(3)]    # ints, units 2^-(k_d + 1)
                A, B, Cc = P
                t = ((A[1] * B[2] - B[1] * A[2]) * Cc[0] + (A[2] * B[0] - B[2] * A[0]) * Cc[1]
                     + (A[0] * B[1] - B[0] * A[1]) * Cc[2])
                wide = 6 * M[0] * M[1] * M[2] * len(t) >= 2 ** 63         # int64 sums could wrap: sum as ints
                vol6 += int(t.sum(dtype=object if wide else np.int64))
                vol_abs_i += int(np.abs(t).sum(dtype=object if wide else np.int64))
    vt = np.concatenate(vol_terms) if vol_terms else np.zeros(0)
    at = np.concatenate(area_terms) if area_terms else np.zeros(0)
    vals, cnts = np.unique(at, return_counts=True)
    ksum = sum(k for _, k in dy)
    unit = 2.0 ** -(ksum + 3)
    out.update(exact=exact, vol6_unit=unit, vol_mag=vol_mag, area_mag=area_mag, n_tri=len(at),
               area_terms=(vals, cnts), area_fsum=float(sum(Fraction(float(v)) * int(n) for v, n in zip(vals, cnts))),
               vol_fsum=math.fsum(vt))
    if exact:
        out["vol6"] = vol6
        out["vol_terms_abs"] = vol_abs_i * unit
        assert math.fsum(vt) == float(Fraction(vol6) * Fraction(unit))       # the double terms are the exact terms
        assert math.fsum(np.abs(vt)) == float(Fraction(vol_abs_i) * Fraction(unit))
    else:
        out["vol6"] = None
        out["vol_terms_abs"] = float(np.abs(vt).sum())
    d2, d2i = _diameters(h, sp, exact)
    out.update(dia2=d2, dia2_exact=d2i, dia=[float(np.sqrt(v)) for v in d2],
               dia2_unit=4.0 ** -(max(k for _, k in dy) + 1))
    return out


def mesh2d(mask, spacing):
    """Marching squares over every 2x2 neighbourhood of an already padded 2-D mask, vectorised.  Returns a dict:

    eighths      exact count of inside eighths of a pixel (surface = eighths / 8 * sy * sx)
    n_diag, n_x, n_y  segment counts: corner cuts (length diag = sqrt(0.25 sy^2 + 0.25 sx^2)), cuts along x (length
                 sx) and along y (length sy); per_fsum their correctly rounded total length, n_sq the squares cut
    n_verts      exact number of mesh vertices (crossed left and bottom square edges), verts their half-index coordinates
    dia2         squared diameter in the reference's double operations; dia2_exact the exact integer in units
                 4^-(kmax + 1) when every square and sum is exact, else None; dia = sqrt(dia2)
    cross2       twice the reference's signed surface: sum of the oriented segment cross products (per_fsum-style
                 correctly rounded), and cross_mag the sum of their |products| (its cancellation scale)"""
    from fractions import Fraction
    m = np.asarray(mask) != 0
    sy, sx = float(spacing[0]), float(spacing[1])
    Y, X = m.shape
    if Y < 2 or X < 2:
        return {"verts": np.zeros((0, 2), np.int64), "eighths": 0, "n_diag": 0, "n_x": 0, "n_y": 0, "n_sq": 0, "per_fsum": 0.0, "n_verts": 0, "dia2": 0.0,
                "dia2_exact": 0, "dia": 0.0, "cross2": 0.0, "cross_mag": 0.0}
    p0, p1, p2, p3 = m[:-1, :-1], m[:-1, 1:], m[1:, 1:], m[1:, :-1]
    cnt = p0.astype(np.int64) + p1 + p2 + p3
    diag_pair = (cnt == 2) & (p0 == p2)
    adj = (cnt == 2) & (p0 != p2)
    along_x = adj & (p0 == p1)
    one_three = (cnt == 1) | (cnt == 3)
    eighths = int(8 * (cnt == 4).sum() + (cnt == 1).sum() + 7 * (cnt == 3).sum() + 2 * diag_pair.sum() + 4 * adj.sum())
    n_diag = int(one_three.sum() + 2 * diag_pair.sum())
    n_x, n_y = int(along_x.sum()), int((adj & ~along_x).sum())
    diag = float(np.sqrt(0.25 * sy * sy + 0.25 * sx * sx))
    per = float(n_diag * Fraction(diag) + n_x * Fraction(sx) + n_y * Fraction(sy))
    # vertices: crossed left edge (p0 | p3) at (2y+1, 2x), crossed bottom edge (p3 - p2) at (2y+2, 2x+1)
    ly, lx = np.nonzero(p0 != p3)
    by, bx = np.nonzero(p3 != p2)
    h = np.concatenate([np.stack([2 * ly + 1, 2 * lx], 1), np.stack([2 * by + 2, 2 * bx + 1], 1)]).astype(np.int64)
    dy = [_dyadic(s) for s in (sy, sx)]
    exact = all(2 * max(Y, X) * abs(n) < 2 ** 26 for n, _ in dy)
    d2, d2i = _diameters(h, [sy, sx], exact)
    cr, mag = _signed_cross2d(m, sy, sx)
    return {"eighths": eighths, "n_diag": n_diag, "n_x": n_x, "n_y": n_y, "n_sq": int((one_three | (cnt == 2)).sum()),
            "per_fsum": per, "n_verts": len(h), "verts": h, "dia2": d2[0], "dia2_exact": d2i[0] if exact else None,
            "dia": float(np.sqrt(d2[0])), "cross2": cr, "cross_mag": mag}


def _signed_cross2d(m, sy, sx):
    """the reference's surface sum, vectorised: for every cut segment a -> b (oriented as in coefficients2d) the cross
    product a_y * b_x - b_y * a_x; returns their correctly rounded sum and the sum of |a_y * b_x| + |b_y * a_x|"""
    mid = np.array([(0.0, 0.5), (0.5, 1.0), (1.0, 0.5), (0.5, 0.0)])
    corner = [(0, 0), (0, 1), (1, 1), (1, 0)]
    Y, X = m.shape
    ins = [m[dy:Y - 1 + dy, dx:X - 1 + dx] for dy, dx in corner]
    code = sum(ins[e].astype(np.int64) << e for e in range(4))
    terms, mag = [], 0.0
    for c in range(1, 15):
        iy, ix = np.nonzero(code == c)
        if len(iy) == 0:
            continue
        inside = [bool(c >> e & 1) for e in range(4)]
        k = sum(inside)
        for e in [e for e in range(4) if inside[e] and not inside[(e + 1) % 4]]:
            f = e
            while True:
                f = (f + 1) % 4
                if not inside[f] and inside[(f + 1) % 4]:
                    break
            if k == 2 and inside[0] == inside[2]:
                f = (e - 1) % 4
            ay, ax = (iy + mid[e][0]) * sy, (ix + mid[e][1]) * sx
            by, bx = (iy + mid[f][0]) * sy, (ix + mid[f][1]) * sx
            terms.append(ay * bx - by * ax)
            mag += float((np.abs(ay * bx) + np.abs(by * ax)).sum())
    return (math.fsum(np.concatenate(terms)) if terms else 0.0), mag


def sum_bound(depth, abs_sum, mag=0.0, per_term=0):
    """error bound of a double sum of terms: recursive summation with chains of at most `depth` additions errs by at
    most depth * u * sum|terms|; terms that are themselves rounded add per_term * u * mag (mag: their rounding scale,
    `vol_mag` / `area_mag` of mesh; 0 when the terms are exact)"""
    return depth * U * abs_sum + per_term * U * mag
