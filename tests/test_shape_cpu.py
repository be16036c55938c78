"""Shape path on the CPU box: the generated marching-cubes table and the oracle restatement against the
reference's outputs (tests/golden/shape_*.{npz,json}, produced by the compiled reference `_cshape` and
the reference RadiomicsShape class, tests/golden/make_golden.py --shape-only)."""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "oracle"))
import shape_np  # noqa: E402

G = os.path.join(HERE, "golden")


def test_table_reproduces_every_single_cube_probe():
    pr = np.load(os.path.join(G, "shape_cube_probes.npz"))
    for cfg in range(256):
        m = np.zeros((2, 2, 2), dtype=bool)
        for i in range(8):
            if cfg >> i & 1:
                m[i >> 2 & 1, i >> 1 & 1, i & 1] = True
        for k, sp in enumerate(pr["spacings"]):
            sa, vol, _ = shape_np.coefficients(m, sp)
            assert sa == pytest.approx(pr["probes"][cfg, k, 0], rel=1e-12, abs=1e-13), (cfg, k)
            assert vol == pytest.approx(pr["probes"][cfg, k, 1], rel=1e-12, abs=1e-13), (cfg, k)


def test_table_is_well_formed():
    mids, tri = shape_np._MID2, shape_np._TRI
    assert mids.shape == (12, 3) and tri.shape == (256, 16)
    assert (tri[0] == -1).all() and (tri[255] == -1).all()
    for cfg in range(256):
        row = tri[cfg]
        n = int((row >= 0).sum())
        assert n % 3 == 0 and (row[n:] == -1).all()
        for e in row[:n]:                       # a triangle corner sits on an edge whose ends differ in the mask
            a = [int(v) for v in (mids[e] // 2)]
            b = [int(v) for v in ((mids[e] + 1) // 2)]
            ia, ib = a[0] << 2 | a[1] << 1 | a[2], b[0] << 2 | b[1] << 1 | b[2]
            assert (cfg >> ia & 1) != (cfg >> ib & 1), (cfg, e)


@pytest.mark.parametrize("name", ["blob", "noise", "sparse", "touching_border", "single", "plane"])
def test_oracle_coefficients_match_reference(name):
    d = np.load(os.path.join(G, "shape_random.npz"))
    sa, vol, dia = shape_np.coefficients(d[f"{name}_mask"], d[f"{name}_spacing"])
    ref = d[f"{name}_coeff"]
    assert sa == pytest.approx(ref[0], rel=1e-11, abs=1e-12)
    assert vol == pytest.approx(ref[1], rel=1e-11, abs=1e-9)
    assert list(dia) == [pytest.approx(v, rel=1e-15, abs=0) for v in ref[2:6]]


@pytest.mark.parametrize("case", ["brain2", "breast1", "lung1"])
def test_oracle_features_match_reference_class(case):
    exp = json.load(open(os.path.join(G, "shape_expect.json")))[case]
    seg = np.load(os.path.join(G, "segment_cases.npz"))
    got = shape_np.features(seg[f"{case}_mask"], seg[f"{case}_spacing"][::-1])
    for f, v in exp["features"].items():
        assert got[f] == pytest.approx(v, rel=1e-9), f
    for f, v in exp["baseline"].items():          # the stored CSV, at the reference's own 3 % (tests/testUtils.py:266-275)
        assert got[f] == pytest.approx(v, rel=0.03), f


def test_committed_table_is_what_the_generator_derives():
    """csrc/mc_table.inc is the output of gen_mc_table.build() on the committed probes (geometry + black-box selection),
    not a hand-edited or transcribed table."""
    import gen_mc_table as g
    table = g.build()
    mids, tri = g.load_table()
    assert [tuple(m) for m in mids] == list(g.EDGE_MID2)
    for cfg, tris in enumerate(table):
        flat = [e for t in tris for e in t]
        assert list(tri[cfg][:len(flat)]) == flat and (tri[cfg][len(flat):] == -1).all(), cfg


SHAPE2D = ["disc", "noise", "sparse", "touching_border", "single", "checker", "ring"]


@pytest.mark.parametrize("name", SHAPE2D)
def test_shape2d_restatement_matches_compiled_reference_goldens(name):
    """oracle/shape_np.coefficients2d against the reference's calculate_coefficients2D (tests/golden/shape2d_golden.npz,
    written by make_golden.py --shape2d-only from the compiled _cshape)"""
    import shape_np as S
    d = np.load(os.path.join(G, "shape2d_golden.npz"))
    per, sur, dia = S.coefficients2d(np.pad(d[name + "_mask"], 1), d[name + "_spacing"])
    ref = d[name + "_coeff"]
    assert per == pytest.approx(ref[0], rel=1e-13) and sur == pytest.approx(ref[1], rel=1e-12, abs=1e-14)
    assert dia == ref[2]


# ---------------------------------------------------------------------------------------------------------------------
# The vectorised oracle (shape_np.mesh / mesh2d) that the large-mask GPU tests use, pinned on three references: the loop
# oracle and the goldens above, exact O(V^2) diameters, and the compiled reference _cshape on non-dyadic spacings.
DYADIC = [(0.75, 1.25, 0.5), (1.0, 1.0, 1.0), (0.5, 2.0, 1.5)]


def _brute_d2(h, sp):
    """exact squared diameters over every vertex pair, as Fractions: 3-D (equal z, equal y, equal x, all), 2-D (all)"""
    from fractions import Fraction
    P = [[Fraction(int(v)) * Fraction(float(s)) / 2 for v, s in zip(row, sp)] for row in h]
    nd = len(sp)
    best = [Fraction(0)] * (4 if nd == 3 else 1)
    for i in range(len(P)):
        for j in range(i):
            d = sum((P[i][k] - P[j][k]) ** 2 for k in range(nd))
            best[-1] = max(best[-1], d)
            if nd == 3:
                for q in range(3):
                    if h[i][q] == h[j][q]:
                        best[q] = max(best[q], d)
    return best


def test_mesh_oracle_matches_loop_oracle_on_goldens_and_probes():
    """mesh() gives the loop oracle's diameters bit for bit and its area / volume within both sums' bounds on every
    golden mask, and every single-cube probe's area and volume"""
    d = np.load(os.path.join(G, "shape_random.npz"))
    for name in ["blob", "noise", "sparse", "touching_border", "single", "plane"]:
        m, sp = d[f"{name}_mask"], d[f"{name}_spacing"]
        o, ref = shape_np.mesh(m, sp), d[f"{name}_coeff"]
        assert o["dia"] == list(ref[2:6]), name
        loop = shape_np.coefficients(m, sp)
        assert o["dia"] == list(loop[2]), name
        n = o["n_tri"]
        tol_a = 2 * shape_np.sum_bound(n, o["area_fsum"], o["area_mag"], 4)
        tol_v = 2 * shape_np.sum_bound(n, o["vol_terms_abs"], o["vol_mag"], 8) / 6
        assert abs(o["area_fsum"] - ref[0]) <= tol_a and abs(o["area_fsum"] - loop[0]) <= tol_a, name
        assert abs(o["vol_fsum"] / 6 - ref[1]) <= tol_v and abs(o["vol_fsum"] / 6 - loop[1]) <= tol_v, name
    pr = np.load(os.path.join(G, "shape_cube_probes.npz"))
    for cfg in range(256):
        m = np.zeros((2, 2, 2), dtype=bool)
        for i in range(8):
            m[i >> 2 & 1, i >> 1 & 1, i & 1] = bool(cfg >> i & 1)
        for k, sp in enumerate(pr["spacings"]):
            o = shape_np.mesh(m, sp)
            assert o["area_fsum"] == pytest.approx(pr["probes"][cfg, k, 0], rel=1e-14, abs=1e-15), (cfg, k)
            assert o["vol_fsum"] / 6 == pytest.approx(pr["probes"][cfg, k, 1], rel=1e-14, abs=1e-15), (cfg, k)


@pytest.mark.parametrize("sp", DYADIC)
def test_mesh_oracle_exact_terms_on_dyadic_spacings(sp):
    """with dyadic spacings the oracle's double terms are the exact terms: its fsum is the exact six-fold volume
    rounded once, and the loop oracle (plain sequential double sums) lands within that sum's bound"""
    rng = np.random.default_rng(3)
    m = rng.random((9, 10, 11)) < 0.45
    o = shape_np.mesh(m, sp)
    assert o["exact"]
    from fractions import Fraction
    assert o["vol_fsum"] == float(Fraction(o["vol6"]) * Fraction(o["vol6_unit"]))
    loop = shape_np.coefficients(m, sp)
    assert abs(loop[0] - o["area_fsum"]) <= shape_np.sum_bound(o["n_tri"], o["area_fsum"]) + shape_np.U * o["area_fsum"]
    assert abs(loop[1] - o["vol_fsum"] / 6) <= shape_np.sum_bound(o["n_tri"], o["vol_terms_abs"]) / 6 + 2 * shape_np.U * abs(loop[1])
    assert o["dia"] == list(loop[2])
    assert [v * o["dia2_unit"] for v in o["dia2_exact"]] == o["dia2"]


def test_mesh_diameter_pruning_matches_brute_force():
    """the hull-pruned diameters equal exact all-pairs maxima on 300 random small masks (3-D and 2-D), of every density
    from a few voxels to almost full, with flat (extent 2) axes among them"""
    rng = np.random.default_rng(17)
    from fractions import Fraction
    for t in range(300):
        nd = 3 if t % 3 else 2
        shape = tuple(int(v) for v in rng.integers(2, 8 if nd == 3 else 14, nd))
        m = rng.random(shape) < rng.uniform(0.05, 0.95)
        sp = tuple(float(v) for v in rng.choice([0.5, 0.75, 1.0, 1.25, 2.0, 3.0], nd))
        o = shape_np.mesh(m, sp) if nd == 3 else shape_np.mesh2d(m, sp)
        exact = o["dia2_exact"] if nd == 3 else [o["dia2_exact"]]
        brute = _brute_d2(o["verts"].tolist(), sp)
        unit = Fraction(o["dia2_unit"]) if nd == 3 else Fraction(1, 4 ** (max(shape_np._dyadic(s)[1] for s in sp) + 1))
        assert [Fraction(v) * unit for v in exact] == brute, (t, shape, sp)


def test_mesh2d_matches_loop_oracle_and_goldens():
    d = np.load(os.path.join(G, "shape2d_golden.npz"))
    for name in SHAPE2D:
        m, sp = np.pad(d[name + "_mask"], 1), d[name + "_spacing"]
        o, ref = shape_np.mesh2d(m, sp), d[name + "_coeff"]
        per, sur, dia = shape_np.coefficients2d(m, sp)
        assert o["dia"] == ref[2] == dia, name
        nseg = o["n_diag"] + o["n_x"] + o["n_y"]
        pmax = float(np.hypot(m.shape[0] * sp[0], m.shape[1] * sp[1]))
        assert abs(o["per_fsum"] - ref[0]) <= shape_np.sum_bound(nseg, o["per_fsum"]) + 6 * shape_np.U * pmax * nseg, name
        exact_sur = o["eighths"] * 0.125 * sp[0] * sp[1]
        assert abs(sur - ref[1]) <= 1e-15 * abs(ref[1])
        assert abs(exact_sur - ref[1]) <= shape_np.sum_bound(nseg + 5, o["cross_mag"]) / 2 + 3 * shape_np.U * exact_sur, name


def _cshape():
    import build_ref
    try:
        return build_ref.load("_cshape")
    except ImportError as e:
        pytest.fail(f"the compiled reference _cshape is missing ({e}); build() compiles it into oracle/_ref/")


@pytest.mark.parametrize("seed", range(4))
def test_mesh_oracle_matches_compiled_reference_on_non_dyadic_spacings(seed):
    """random moderate masks (up to ~10^4 vertices) and spacings like (2.1, 0.7, 1.3): the compiled reference's
    diameters bit for bit (the oracle forms them with the same double operations), area and volume within the sum of
    the reference's sequential-sum bound and both sides' per-term rounding"""
    ref = _cshape()
    rng = np.random.default_rng(100 + seed)
    shape = tuple(int(v) for v in rng.integers(12, 30, 3))
    z, y, x = np.meshgrid(*[np.linspace(-1, 1, s) for s in shape], indexing="ij")
    m = (z * z + y * y * 1.3 + x * x * 0.8 < 0.8) & (rng.random(shape) > 0.1) if seed % 2 else rng.random(shape) < 0.3
    sp = [(2.1, 0.7, 1.3), (0.83, 1.17, 2.9), (1.1, 1.1, 3.3), (0.3, 0.45, 0.6)][seed]
    o = shape_np.mesh(m, sp)
    assert not o["exact"]
    sa, vol, dia = ref.calculate_coefficients(m.astype(np.int8), np.array(sp))
    assert o["dia"] == list(dia)
    n = o["n_tri"]
    assert abs(sa - o["area_fsum"]) <= shape_np.sum_bound(n, o["area_fsum"], 2 * o["area_mag"], 4)
    assert abs(vol - o["vol_fsum"] / 6) <= shape_np.sum_bound(n, o["vol_terms_abs"], 2 * o["vol_mag"], 8) / 6


@pytest.mark.parametrize("seed", range(3))
def test_mesh2d_matches_compiled_reference_on_non_dyadic_spacings(seed):
    ref = _cshape()
    rng = np.random.default_rng(200 + seed)
    Y, X = (int(v) for v in rng.integers(40, 120, 2))
    yy, xx = np.meshgrid(np.linspace(-1, 1, Y), np.linspace(-1, 1, X), indexing="ij")
    m = np.pad((yy * yy + xx * xx < 0.7 + 0.2 * rng.random((Y, X))) if seed != 1 else rng.random((Y, X)) < 0.5, 1)
    sp = [(2.1, 0.7), (0.83, 1.17), (0.3, 0.45)][seed]
    o = shape_np.mesh2d(m, sp)
    per, sur, dia = ref.calculate_coefficients2D(m.astype(np.int8), np.array(sp))
    assert dia == o["dia"]
    nseg = o["n_diag"] + o["n_x"] + o["n_y"]
    pmax = float(np.hypot((Y + 2) * sp[0], (X + 2) * sp[1]))
    assert abs(per - o["per_fsum"]) <= shape_np.sum_bound(nseg, per) + 6 * shape_np.U * pmax * nseg
    exact_sur = o["eighths"] * 0.125 * sp[0] * sp[1]
    assert abs(sur - exact_sur) <= shape_np.sum_bound(nseg + 5, o["cross_mag"]) / 2 + 3 * shape_np.U * exact_sur
