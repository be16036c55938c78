"""CPU checks of the two third-party pre-filter restatements (oracle/filters_np.py; PARITY UNPINNED: PyWavelets / SimpleITK
are not dependencies of the project): the documented phase / alignment of
the stationary wavelet transform, perfect reconstruction with the matching synthesis bank, Parseval, and the level loop of
the reference's _swt3."""
import numpy as np
import pytest

import filters_np as FN

LO = np.array([-0.01565572813546454, -0.0727326195128539, 0.38486484686420286, 0.8525720202122554, 0.3378976624578092,
               -0.0727326195128539])
HI = np.array([(-1) ** (k + 1) * LO[5 - k] for k in range(6)])


def test_swt_axis_impulse_phase():
    """out[n] = sum_j h[j] x[(n + F/2 - j) mod N]: tap j lands at p - F/2 + j"""
    N, p = 16, 5
    x = np.zeros(N)
    x[p] = 1
    for h in (LO, HI):
        out = FN.swt_axis(x, h, 0)
        for j in range(6):
            assert out[(p - 3 + j) % N] == h[j]
        assert np.count_nonzero(out) == 6


def test_swt_level1_perfect_reconstruction_and_parseval():
    """undecimated two-channel bank: x = 1/2 (R_lo a + R_hi d) with the time-reversed filters at the mirrored phase"""
    rng = np.random.default_rng(0)
    x = rng.normal(size=64)
    a, d = FN.swt_axis(x, LO, 0), FN.swt_axis(x, HI, 0)
    rec = np.zeros_like(x)
    for j in range(6):
        # adjoint of out[n] = sum_j h[j] x[n + 3 - j]:  x~[m] += h[j] out[m - 3 + j]
        rec += LO[j] * np.roll(a, 3 - j) + HI[j] * np.roll(d, 3 - j)
    assert np.allclose(rec / 2, x, atol=1e-12)
    assert abs((a ** 2).sum() + (d ** 2).sum() - 2 * (x ** 2).sum()) < 1e-10


@pytest.mark.parametrize("shape", [(6, 8, 10), (5, 7, 9)])
def test_swt3_levels_structure(shape):
    rng = np.random.default_rng(1)
    x = rng.normal(size=shape)
    approx1, lev1 = FN.swt3_levels(x, LO, HI, (2, 1, 0), level=1)
    one = FN.swtn_level1(x, LO, HI, (2, 1, 0))
    assert np.allclose(approx1, one["aaa"]) and all(np.allclose(lev1[0][k], one[k]) for k in lev1[0])
    approx2, lev2 = FN.swt3_levels(x, LO, HI, (2, 1, 0), level=2)
    assert len(lev2) == 2 and all(np.allclose(lev2[0][k], lev1[0][k]) for k in lev1[0])
    if all(s % 2 == 0 for s in shape):
        again = FN.swtn_level1(approx1, LO, HI, (2, 1, 0))          # even sizes: level 2 == level 1 of the (unpadded) approximation
        assert np.allclose(approx2, again["aaa"])
    else:
        again = FN.swtn_level1(approx1, LO, HI, (2, 1, 0))          # odd sizes: the padded sample is carried, NOT re-wrapped
        assert not np.allclose(approx2, again["aaa"])
    a_s, lev_s = FN.swt3_levels(x, LO, HI, (2, 1, 0), level=1, start_level=1)
    assert np.allclose(a_s, approx2) and all(np.allclose(lev_s[0][k], lev2[1][k]) for k in lev_s[0])
