"""Host-side feature formulas for SEGMENT-based extraction: one (small) texture matrix per ROI has
already been built on the GPU; turning it into the 24/16/16/14/5 scalar features is O(Ng^2) host
work, exactly the layer the reference keeps in Python (radiomics/glcm.py:208-887, glrlm.py:174-523,
glszm.py:108-434, gldm.py:103-430, ngtdm.py:116-287).  Voxel-based extraction does NOT come through
here -- there the features are fused into the CUDA kernels (csrc/vox_features.cuh, glcm_fast.cuh).

Each *_features function takes the processed matrix of ONE ROI (no voxel axis) and returns {feature: float}; the
<CLASS>_NAMES tables name the features (GLCM / GLRLM / NGTDM in the order of the voxel kernels' maps,
_lib.feature_names; GLSZM / GLDM map the shared size-matrix formulas to the class's names).
"""
from __future__ import annotations

import numpy as np

EPS = np.spacing(1)


def _mean_ignoring_nan(v):
    v = np.asarray(v, float)
    ok = ~np.isnan(v)
    return float(v[ok].mean()) if ok.any() else float("nan")


def _entropy(p):
    return -float(np.sum(p * np.log2(p + EPS)))


# ---------------------------------------------------------------------------------- GLCM
GLCM_NAMES = ("Autocorrelation", "ClusterProminence", "ClusterShade", "ClusterTendency", "Contrast", "Correlation",
              "DifferenceAverage", "DifferenceEntropy", "DifferenceVariance", "Id", "Idm", "Idmn", "Idn", "Imc1", "Imc2",
              "InverseVariance", "JointAverage", "JointEnergy", "JointEntropy", "MCC", "MaximumProbability", "SumAverage",
              "SumEntropy", "SumSquares")


def glcm_process(P, levels, symmetrical=True, weights=None):
    """raw counts [B,Ng,Ng,Na] of a batch of B matrices -> normalised [B,n,n,A] restricted to the present levels, with
    the reference's symmetrisation / weighting / removal of the angles that are empty for EVERY matrix of the batch
    (glcm.py:149-205): one common angle axis, so the batch stacks."""
    idx = np.asarray(levels, int) - 1
    P = P[:, idx][:, :, idx].astype(float)
    if symmetrical:
        P = P + P.transpose(0, 2, 1, 3)
    if weights is not None:
        P = (P * weights[None, None, None, :]).sum(3, keepdims=True)
    tot = P.sum((1, 2))
    if P.shape[3] > 1:
        keep = tot.sum(0) != 0
        P, tot = P[..., keep], tot[:, keep]
    tot = np.where(tot == 0, np.nan, tot)
    return P / tot[:, None, None, :]


def glcm_features(p, levels, Ng):
    lv = np.asarray(levels, float)
    n, A = lv.size, p.shape[2]
    per_angle = {k: np.full(A, np.nan) for k in GLCM_NAMES if k != "JointAverage"}
    ux_all = np.full(A, np.nan)
    li = lv.astype(int)
    kd = np.abs(li[:, None] - li[None, :])
    ks = li[:, None] + li[None, :]
    I, J = lv[:, None], lv[None, :]
    kD = np.arange(Ng, dtype=float)
    for a in range(A):
        q = p[:, :, a]
        if np.isnan(q).any():
            continue
        px, py = q.sum(1), q.sum(0)
        ux, uy = float((q * I).sum()), float((q * J).sum())
        ux_all[a] = ux
        r = per_angle
        r["Autocorrelation"][a] = (q * I * J).sum()
        dev = I + J - ux - uy
        r["ClusterTendency"][a] = (q * dev ** 2).sum()
        r["ClusterShade"][a] = (q * dev ** 3).sum()
        r["ClusterProminence"][a] = (q * dev ** 4).sum()
        r["Contrast"][a] = (q * (I - J) ** 2).sum()
        sx, sy = np.sqrt((q * (I - ux) ** 2).sum()), np.sqrt((q * (J - uy) ** 2).sum())
        r["Correlation"][a] = 1.0 if sx * sy == 0 else (q * (I - ux) * (J - uy)).sum() / (sx * sy + EPS)
        pd = np.bincount(kd.ravel(), weights=q.ravel(), minlength=Ng)[:Ng]
        ps = np.bincount(ks.ravel(), weights=q.ravel(), minlength=2 * Ng + 1)
        da = float((kD * pd).sum())
        r["DifferenceAverage"][a] = da
        r["DifferenceEntropy"][a] = _entropy(pd)
        r["DifferenceVariance"][a] = (pd * (kD - da) ** 2).sum()
        r["JointEnergy"][a] = (q ** 2).sum()
        hxy = _entropy(q)
        r["JointEntropy"][a] = hxy
        hx, hy = _entropy(px), _entropy(py)
        pxy = px[:, None] * py[None, :]
        hxy1 = -float((q * np.log2(pxy + EPS)).sum())
        hxy2 = -float((pxy * np.log2(pxy + EPS)).sum())
        div = max(hx, hy)
        r["Imc1"][a] = (hxy - hxy1) / div if div != 0 else 0.0
        with np.errstate(invalid="ignore"):
            r["Imc2"][a] = 0.0 if hxy2 == hxy else np.sqrt(1 - np.exp(-2 * (hxy2 - hxy)))
        r["Idm"][a] = (pd / (1 + kD ** 2)).sum()
        r["Idmn"][a] = (pd / (1 + kD ** 2 / Ng ** 2)).sum()
        r["Id"][a] = (pd / (1 + kD)).sum()
        r["Idn"][a] = (pd / (1 + kD / Ng)).sum()
        r["InverseVariance"][a] = (pd[1:] / kD[1:] ** 2).sum()
        r["MaximumProbability"][a] = q.max()
        r["SumAverage"][a] = (np.arange(2 * Ng + 1, dtype=float) * ps).sum()
        r["SumEntropy"][a] = _entropy(ps)
        r["SumSquares"][a] = (q * (I - ux) ** 2).sum()
        if n >= 2:
            Q = (q / (px[:, None] * py[None, :] + EPS)) @ q.T
            ev = np.sort(np.linalg.eigvals(Q).real)
            r["MCC"][a] = np.sqrt(max(ev[-2], 0.0))
    out = {k: _mean_ignoring_nan(v) for k, v in per_angle.items()}
    if n < 2:
        out["MCC"] = 1.0
    out["JointAverage"] = float(ux_all.mean()) if A else float("nan")   # plain mean (glcm.py:292)
    return out


# ---------------------------------------------------------------------------------- GLRLM
GLRLM_NAMES = ("GrayLevelNonUniformity", "GrayLevelNonUniformityNormalized", "GrayLevelVariance", "HighGrayLevelRunEmphasis",
               "LongRunEmphasis", "LongRunHighGrayLevelEmphasis", "LongRunLowGrayLevelEmphasis", "LowGrayLevelRunEmphasis",
               "RunEntropy", "RunLengthNonUniformity", "RunLengthNonUniformityNormalized", "RunPercentage", "RunVariance",
               "ShortRunEmphasis", "ShortRunHighGrayLevelEmphasis", "ShortRunLowGrayLevelEmphasis")


def glrlm_process(P, levels, weights=None):
    """raw [Ng,Nr,Na] -> [n,R,A] with absent levels, empty angles and empty run lengths removed
    (glrlm.py:120-127,153-170,184-188).  Returns (P, run_lengths, runs_per_angle)."""
    P = P[np.asarray(levels, int) - 1].astype(float)
    if weights is not None:
        P = (P * weights[None, None, :]).sum(2, keepdims=True)
    Nr = P.sum((0, 1))
    if P.shape[2] > 1:
        keep = Nr != 0
        P, Nr = P[:, :, keep], Nr[keep]
    Nr = np.where(Nr == 0, np.nan, Nr)
    used = P.sum((0, 2)) != 0
    j = np.arange(1, P.shape[1] + 1, dtype=float)[used]
    return P[:, used], j, Nr


def glrlm_features(P, j, Nr, levels):
    i = np.asarray(levels, float)
    A = P.shape[2]
    r = {k: np.full(A, np.nan) for k in GLRLM_NAMES}
    i2, j2 = i[:, None] ** 2, j[None, :] ** 2
    for a in range(A):
        if np.isnan(Nr[a]):
            continue
        M, N = P[:, :, a], Nr[a]
        pr, pg = M.sum(0), M.sum(1)
        r["ShortRunEmphasis"][a] = (pr / j ** 2).sum() / N
        r["LongRunEmphasis"][a] = (pr * j ** 2).sum() / N
        r["GrayLevelNonUniformity"][a] = (pg ** 2).sum() / N
        r["GrayLevelNonUniformityNormalized"][a] = (pg ** 2).sum() / N ** 2
        r["RunLengthNonUniformity"][a] = (pr ** 2).sum() / N
        r["RunLengthNonUniformityNormalized"][a] = (pr ** 2).sum() / N ** 2
        r["RunPercentage"][a] = N / (pr * j).sum()
        qg, qr = pg / N, pr / N
        r["GrayLevelVariance"][a] = (qg * (i - (qg * i).sum()) ** 2).sum()
        r["RunVariance"][a] = (qr * (j - (qr * j).sum()) ** 2).sum()
        r["RunEntropy"][a] = _entropy(M / N)
        r["LowGrayLevelRunEmphasis"][a] = (pg / i ** 2).sum() / N
        r["HighGrayLevelRunEmphasis"][a] = (pg * i ** 2).sum() / N
        r["ShortRunLowGrayLevelEmphasis"][a] = (M / (i2 * j2)).sum() / N
        r["ShortRunHighGrayLevelEmphasis"][a] = (M * i2 / j2).sum() / N
        r["LongRunLowGrayLevelEmphasis"][a] = (M * j2 / i2).sum() / N
        r["LongRunHighGrayLevelEmphasis"][a] = (M * i2 * j2).sum() / N
    return {k: _mean_ignoring_nan(v) for k, v in r.items()}


# ------------------------------------------------------------------------- GLSZM / GLDM
def size_matrix_features(M, levels, j):
    """M [n, J] counts, j = the size / dependence value of each kept column."""
    i = np.asarray(levels, float)
    N = M.sum()
    N = 1.0 if N == 0 else N
    pj, pg = M.sum(0), M.sum(1)
    i2, j2 = i[:, None] ** 2, j[None, :] ** 2
    Np = (pj * j).sum()
    qg, qj = pg / N, pj / N
    return {
        "SmallEmphasis": (pj / j ** 2).sum() / N, "LargeEmphasis": (pj * j ** 2).sum() / N,
        "GrayLevelNonUniformity": (pg ** 2).sum() / N, "GrayLevelNonUniformityNormalized": (pg ** 2).sum() / N ** 2,
        "SizeNonUniformity": (pj ** 2).sum() / N, "SizeNonUniformityNormalized": (pj ** 2).sum() / N ** 2,
        "Percentage": N / (1.0 if Np == 0 else Np),
        "GrayLevelVariance": (qg * (i - (qg * i).sum()) ** 2).sum(),
        "SizeVariance": (qj * (j - (qj * j).sum()) ** 2).sum(),
        "Entropy": _entropy(M / N),
        "LowGrayLevelEmphasis": (pg / i ** 2).sum() / N, "HighGrayLevelEmphasis": (pg * i ** 2).sum() / N,
        "SmallLowGrayLevelEmphasis": (M / (i2 * j2)).sum() / N, "SmallHighGrayLevelEmphasis": (M * i2 / j2).sum() / N,
        "LargeLowGrayLevelEmphasis": (M * j2 / i2).sum() / N, "LargeHighGrayLevelEmphasis": (M * i2 * j2).sum() / N,
    }


GLSZM_NAMES = {
    "SmallEmphasis": "SmallAreaEmphasis", "LargeEmphasis": "LargeAreaEmphasis",
    "GrayLevelNonUniformity": "GrayLevelNonUniformity",
    "GrayLevelNonUniformityNormalized": "GrayLevelNonUniformityNormalized",
    "SizeNonUniformity": "SizeZoneNonUniformity", "SizeNonUniformityNormalized": "SizeZoneNonUniformityNormalized",
    "Percentage": "ZonePercentage", "GrayLevelVariance": "GrayLevelVariance", "SizeVariance": "ZoneVariance",
    "Entropy": "ZoneEntropy", "LowGrayLevelEmphasis": "LowGrayLevelZoneEmphasis",
    "HighGrayLevelEmphasis": "HighGrayLevelZoneEmphasis", "SmallLowGrayLevelEmphasis": "SmallAreaLowGrayLevelEmphasis",
    "SmallHighGrayLevelEmphasis": "SmallAreaHighGrayLevelEmphasis",
    "LargeLowGrayLevelEmphasis": "LargeAreaLowGrayLevelEmphasis",
    "LargeHighGrayLevelEmphasis": "LargeAreaHighGrayLevelEmphasis",
}
GLDM_NAMES = {
    "SmallEmphasis": "SmallDependenceEmphasis", "LargeEmphasis": "LargeDependenceEmphasis",
    "GrayLevelNonUniformity": "GrayLevelNonUniformity", "SizeNonUniformity": "DependenceNonUniformity",
    "SizeNonUniformityNormalized": "DependenceNonUniformityNormalized", "GrayLevelVariance": "GrayLevelVariance",
    "SizeVariance": "DependenceVariance", "Entropy": "DependenceEntropy",
    "LowGrayLevelEmphasis": "LowGrayLevelEmphasis", "HighGrayLevelEmphasis": "HighGrayLevelEmphasis",
    "SmallLowGrayLevelEmphasis": "SmallDependenceLowGrayLevelEmphasis",
    "SmallHighGrayLevelEmphasis": "SmallDependenceHighGrayLevelEmphasis",
    "LargeLowGrayLevelEmphasis": "LargeDependenceLowGrayLevelEmphasis",
    "LargeHighGrayLevelEmphasis": "LargeDependenceHighGrayLevelEmphasis",
}


def size_matrix_process(P, levels):
    """raw [Ng, J] -> present levels, empty columns dropped; returns (M, j values)."""
    M = P[np.asarray(levels, int) - 1].astype(float)
    used = M.sum(0) != 0
    return M[:, used], np.arange(1, M.shape[1] + 1, dtype=float)[used]


# ---------------------------------------------------------------------------------- NGTDM
NGTDM_NAMES = ("Busyness", "Coarseness", "Complexity", "Contrast", "Strength")


def ngtdm_features(P):
    """P [n,3] = (n_i, s_i, i) for the levels with n_i > 0."""
    n, s, i = P[:, 0].astype(float), P[:, 1].astype(float), P[:, 2].astype(float)
    Nvp = n.sum()
    p = n / Nvp
    Ngp = int((n > 0).sum())
    ps = float((p * s).sum())
    di = i[:, None] - i[None, :]
    out = {"Coarseness": 1.0 / ps if ps != 0 else 1e6}
    div = Ngp * (Ngp - 1)
    out["Contrast"] = float((p[:, None] * p[None, :] * di ** 2).sum() * s.sum() / Nvp / div) if div else 0.0
    ad = float(np.abs((i * p)[:, None] - (i * p)[None, :]).sum())
    out["Busyness"] = ps / ad if ad != 0 else 0.0
    pis = p * s
    out["Complexity"] = float((np.abs(di) * (pis[:, None] + pis[None, :]) / (p[:, None] + p[None, :])).sum() / Nvp)
    ss = float(s.sum())
    out["Strength"] = float(((p[:, None] + p[None, :]) * di ** 2).sum() / ss) if ss != 0 else 0.0
    return out
