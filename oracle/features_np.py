"""TEST INFRASTRUCTURE ONLY -- numpy restatement ("port") of the reference's texture feature
formulas, evaluated on the dense matrices returned by the cMatrices-style functions
(oracle port or the compiled reference).  Checker for the fused CUDA feature kernels and the
feature half of bench.py's cpu_baseline; never imported by the product path.

Follows (per-voxel axis 0 everywhere, so segment mode is just Nvox = 1):
  GLCM   reference radiomics/glcm.py:123-205 (matrix post-processing), :208-258 (coefficients),
         :260-887 (24 features)
  GLRLM  reference radiomics/glrlm.py:97-172, :174-194, :196-523 (16 features)
  GLSZM  reference radiomics/glszm.py:75-106, :108-138, :140-434 (16 features)
  GLDM   reference radiomics/gldm.py:84-136, :138-430 (14 features)
  NGTDM  reference radiomics/ngtdm.py:98-131, :133-287 (5 features)
Pinned against the reference's own golden CSV values and voxel-mode runs (tests/golden/).

One documented deviation: MCC is evaluated per (voxel, angle) and empty angles are dropped by
the nanmean, instead of letting one NaN abort the whole batch (reference defect, SURVEY.md
Appendix A #6; this equals the reference run with voxelBatch=1).
"""
from __future__ import annotations

import numpy as np

EPS = np.spacing(1)


def angle_weights(angles, spacing_zyx, norm, kind):
    """kind 'glcm' -> exp(-d^2) weights (glcm.py:160-181); 'glrlm' -> d (glrlm.py:130-150)."""
    if norm is None:
        return None
    a = np.abs(np.asarray(angles, float)) * np.asarray(spacing_zyx, float)[-angles.shape[1]:]
    if norm == "infinity":
        d = a.max(1)
    elif norm == "euclidean":
        d = np.sqrt((a ** 2).sum(1))
    elif norm == "manhattan":
        d = a.sum(1)
    else:  # 'no_weighting' and unknown names
        return np.ones(len(angles))
    return np.exp(-d ** 2) if kind == "glcm" else d


def _nanmean(x, axis):
    with np.errstate(invalid="ignore", divide="ignore"):
        cnt = np.sum(~np.isnan(x), axis)
        tot = np.nansum(x, axis)
        return np.where(cnt > 0, tot / np.maximum(cnt, 1), np.nan)


def _xlog2(p):
    return p * np.log2(p + EPS)


# --------------------------------------------------------------------------- GLCM
def glcm_matrix(P, gray_levels, symmetrical=True, weights=None):
    idx = np.asarray(gray_levels, int) - 1
    P = P[:, idx][:, :, idx].astype(float)
    if symmetrical:
        P = P + np.swapaxes(P, 1, 2)
    if weights is not None:
        P = (P * weights).sum(3, keepdims=True)
    S = P.sum((1, 2))
    if P.shape[3] > 1:
        keep = S.sum(0) != 0
        P, S = P[..., keep], S[:, keep]
    S = np.where(S == 0, np.nan, S)
    return P / S[:, None, None, :]


def glcm_features(p, gray_levels, Ng, n_roi_levels=None):
    """p: normalised [V,n,n,A] (NaN where an angle is empty for that voxel)."""
    lv = np.asarray(gray_levels, float)
    n = lv.size
    I = lv[None, :, None, None]
    J = lv[None, None, :, None]
    with np.errstate(invalid="ignore", divide="ignore"):
        px = p.sum(2)          # [V,n,A]
        py = p.sum(1)          # [V,n,A]
        ux = (p * I).sum((1, 2))     # [V,A]
        uy = (p * J).sum((1, 2))
        f = {}
        f["Autocorrelation"] = _nanmean((p * I * J).sum((1, 2)), 1)
        f["JointAverage"] = ux.mean(1)
        dev = (I + J) - ux[:, None, None, :] - uy[:, None, None, :]
        f["ClusterProminence"] = _nanmean((p * dev ** 4).sum((1, 2)), 1)
        f["ClusterShade"] = _nanmean((p * dev ** 3).sum((1, 2)), 1)
        f["ClusterTendency"] = _nanmean((p * dev ** 2).sum((1, 2)), 1)
        f["Contrast"] = _nanmean((p * (I - J) ** 2).sum((1, 2)), 1)
        dx = I - ux[:, None, None, :]
        dy = J - uy[:, None, None, :]
        sx = np.sqrt((p * dx ** 2).sum((1, 2)))
        sy = np.sqrt((p * dy ** 2).sum((1, 2)))
        cor = (p * dx * dy).sum((1, 2)) / (sx * sy + EPS)
        cor = np.where(sx * sy == 0, 1.0, cor)
        f["Correlation"] = _nanmean(cor, 1)
        # difference / sum histograms
        li = lv.astype(int)
        kd = np.abs(li[:, None] - li[None, :])
        ks = li[:, None] + li[None, :]
        V, A = p.shape[0], p.shape[3]
        pd = np.zeros((V, Ng, A))
        ps = np.zeros((V, 2 * Ng + 1, A))
        # unbuffered adds in (a, b) order: every bin sums its entries in the order of a double loop over (a, b)
        pf = p.reshape(V, n * n, A)
        np.add.at(pd, (slice(None), kd.reshape(-1)), pf)
        np.add.at(ps, (slice(None), ks.reshape(-1)), pf)
        kD = np.arange(Ng, dtype=float)[None, :, None]
        kS = np.arange(2 * Ng + 1, dtype=float)[None, :, None]
        da = (kD * pd).sum(1)
        f["DifferenceAverage"] = _nanmean(da, 1)
        f["DifferenceEntropy"] = _nanmean(-_xlog2(pd).sum(1), 1)
        f["DifferenceVariance"] = _nanmean((pd * (kD - da[:, None, :]) ** 2).sum(1), 1)
        f["JointEnergy"] = _nanmean((p ** 2).sum((1, 2)), 1)
        HXY = -_xlog2(p).sum((1, 2))
        f["JointEntropy"] = _nanmean(HXY, 1)
        HX = -_xlog2(px).sum(1)
        HY = -_xlog2(py).sum(1)
        pxpy = px[:, :, None, :] * py[:, None, :, :]
        HXY1 = -(p * np.log2(pxpy + EPS)).sum((1, 2))
        HXY2 = -(pxpy * np.log2(pxpy + EPS)).sum((1, 2))
        div = np.fmax(HX, HY)
        imc1 = np.where(div != 0, (HXY - HXY1) / np.where(div != 0, div, 1), 0.0)
        imc1 = np.where(np.isnan(HXY), np.nan, imc1)
        f["Imc1"] = _nanmean(imc1, 1)
        imc2 = np.sqrt(1 - np.exp(-2 * (HXY2 - HXY)))
        imc2 = np.where(HXY2 == HXY, 0.0, imc2)
        f["Imc2"] = _nanmean(imc2, 1)
        f["Idm"] = _nanmean((pd / (1 + kD ** 2)).sum(1), 1)
        f["Idmn"] = _nanmean((pd / (1 + kD ** 2 / Ng ** 2)).sum(1), 1)
        f["Id"] = _nanmean((pd / (1 + kD)).sum(1), 1)
        f["Idn"] = _nanmean((pd / (1 + kD / Ng)).sum(1), 1)
        f["InverseVariance"] = _nanmean((pd[:, 1:, :] / kD[:, 1:, :] ** 2).sum(1), 1)
        f["MaximumProbability"] = _nanmean(p.max((1, 2)), 1)
        f["SumAverage"] = _nanmean((kS * ps).sum(1), 1)
        f["SumEntropy"] = _nanmean(-_xlog2(ps).sum(1), 1)
        f["SumSquares"] = _nanmean((p * dx ** 2).sum((1, 2)), 1)
        # MCC: Q(i,j) = sum_k p(i,k) p(j,k) / (px(i) py(k) + eps)   (glcm.py:679-707)
        if n < 2:
            f["MCC"] = np.ones(V)
        else:
            mcc = np.full((V, A), np.nan)
            for v in range(V):
                for a in range(A):
                    pa = p[v, :, :, a]
                    if np.isnan(pa).any():
                        continue
                    den = px[v, :, a][:, None] * py[v, :, a][None, :] + EPS     # [i,k]
                    Q = (pa / den) @ pa.T
                    ev = np.sort(np.linalg.eigvals(Q).real)
                    mcc[v, a] = np.sqrt(max(ev[-2], 0.0))
            f["MCC"] = _nanmean(mcc, 1)
    return f


# --------------------------------------------------------------------------- GLRLM
def glrlm_features(P, gray_levels, weights=None):
    """P raw [V,Ng,Nr,A] from calculate_glrlm."""
    idx = np.asarray(gray_levels, int) - 1
    P = P[:, idx].astype(float)
    if weights is not None:
        P = (P * weights).sum(3, keepdims=True)
    Nr = P.sum((1, 2))
    if P.shape[3] > 1:
        keep = Nr.sum(0) != 0
        P, Nr = P[..., keep], Nr[:, keep]
    Nr = np.where(Nr == 0, np.nan, Nr)
    iv = np.asarray(gray_levels, float)[None, :, None]
    jv = np.arange(1, P.shape[2] + 1, dtype=float)[None, :, None]
    I2 = iv[:, :, None, :] ** 2
    J2 = jv[:, None, :, :] ** 2
    with np.errstate(invalid="ignore", divide="ignore"):
        pr = P.sum(1)
        pg = P.sum(2)
        f = {}
        f["ShortRunEmphasis"] = _nanmean((pr / jv ** 2).sum(1) / Nr, 1)
        f["LongRunEmphasis"] = _nanmean((pr * jv ** 2).sum(1) / Nr, 1)
        f["GrayLevelNonUniformity"] = _nanmean((pg ** 2).sum(1) / Nr, 1)
        f["GrayLevelNonUniformityNormalized"] = _nanmean((pg ** 2).sum(1) / Nr ** 2, 1)
        f["RunLengthNonUniformity"] = _nanmean((pr ** 2).sum(1) / Nr, 1)
        f["RunLengthNonUniformityNormalized"] = _nanmean((pr ** 2).sum(1) / Nr ** 2, 1)
        f["RunPercentage"] = _nanmean(Nr / (pr * jv).sum(1), 1)
        qg = pg / Nr[:, None, :]
        ug = (qg * iv).sum(1, keepdims=True)
        f["GrayLevelVariance"] = _nanmean((qg * (iv - ug) ** 2).sum(1), 1)
        qr = pr / Nr[:, None, :]
        ur = (qr * jv).sum(1, keepdims=True)
        f["RunVariance"] = _nanmean((qr * (jv - ur) ** 2).sum(1), 1)
        q = P / Nr[:, None, None, :]
        f["RunEntropy"] = _nanmean(-_xlog2(q).sum((1, 2)), 1)
        f["LowGrayLevelRunEmphasis"] = _nanmean((pg / iv ** 2).sum(1) / Nr, 1)
        f["HighGrayLevelRunEmphasis"] = _nanmean((pg * iv ** 2).sum(1) / Nr, 1)
        f["ShortRunLowGrayLevelEmphasis"] = _nanmean((P / (I2 * J2)).sum((1, 2)) / Nr, 1)
        f["ShortRunHighGrayLevelEmphasis"] = _nanmean((P * I2 / J2).sum((1, 2)) / Nr, 1)
        f["LongRunLowGrayLevelEmphasis"] = _nanmean((P * J2 / I2).sum((1, 2)) / Nr, 1)
        f["LongRunHighGrayLevelEmphasis"] = _nanmean((P * I2 * J2).sum((1, 2)) / Nr, 1)
    return f


# ------------------------------------------------------------ GLSZM / GLDM share a shape
def _size_matrix_features(P, gray_levels, names):
    """P [V,n,J] counts (level x size/dependence, j = column+1); names maps generic -> class
    feature names.  Nz (0 -> 1) normalises everything."""
    iv = np.asarray(gray_levels, float)[None, :]
    jv = np.arange(1, P.shape[2] + 1, dtype=float)[None, :]
    pj = P.sum(1)
    pg = P.sum(2)
    Nz = P.sum((1, 2))
    Nz = np.where(Nz == 0, 1.0, Nz)
    I2 = iv[:, :, None] ** 2
    J2 = jv[:, None, :] ** 2
    g = {}
    g["SmallEmphasis"] = (pj / jv ** 2).sum(1) / Nz
    g["LargeEmphasis"] = (pj * jv ** 2).sum(1) / Nz
    g["GrayLevelNonUniformity"] = (pg ** 2).sum(1) / Nz
    g["GrayLevelNonUniformityNormalized"] = (pg ** 2).sum(1) / Nz ** 2
    g["SizeNonUniformity"] = (pj ** 2).sum(1) / Nz
    g["SizeNonUniformityNormalized"] = (pj ** 2).sum(1) / Nz ** 2
    Np = (pj * jv).sum(1)
    g["Percentage"] = Nz / np.where(Np == 0, 1.0, Np)
    qg = pg / Nz[:, None]
    ug = (qg * iv).sum(1, keepdims=True)
    g["GrayLevelVariance"] = (qg * (iv - ug) ** 2).sum(1)
    qj = pj / Nz[:, None]
    uj = (qj * jv).sum(1, keepdims=True)
    g["SizeVariance"] = (qj * (jv - uj) ** 2).sum(1)
    q = P / Nz[:, None, None]
    g["Entropy"] = -_xlog2(q).sum((1, 2))
    g["LowGrayLevelEmphasis"] = (pg / iv ** 2).sum(1) / Nz
    g["HighGrayLevelEmphasis"] = (pg * iv ** 2).sum(1) / Nz
    g["SmallLowGrayLevelEmphasis"] = (P / (I2 * J2)).sum((1, 2)) / Nz
    g["SmallHighGrayLevelEmphasis"] = (P * I2 / J2).sum((1, 2)) / Nz
    g["LargeLowGrayLevelEmphasis"] = (P * J2 / I2).sum((1, 2)) / Nz
    g["LargeHighGrayLevelEmphasis"] = (P * I2 * J2).sum((1, 2)) / Nz
    return {names[k]: v for k, v in g.items() if k in names}


GLSZM_NAMES = {
    "SmallEmphasis": "SmallAreaEmphasis", "LargeEmphasis": "LargeAreaEmphasis",
    "GrayLevelNonUniformity": "GrayLevelNonUniformity",
    "GrayLevelNonUniformityNormalized": "GrayLevelNonUniformityNormalized",
    "SizeNonUniformity": "SizeZoneNonUniformity",
    "SizeNonUniformityNormalized": "SizeZoneNonUniformityNormalized",
    "Percentage": "ZonePercentage", "GrayLevelVariance": "GrayLevelVariance",
    "SizeVariance": "ZoneVariance", "Entropy": "ZoneEntropy",
    "LowGrayLevelEmphasis": "LowGrayLevelZoneEmphasis", "HighGrayLevelEmphasis": "HighGrayLevelZoneEmphasis",
    "SmallLowGrayLevelEmphasis": "SmallAreaLowGrayLevelEmphasis",
    "SmallHighGrayLevelEmphasis": "SmallAreaHighGrayLevelEmphasis",
    "LargeLowGrayLevelEmphasis": "LargeAreaLowGrayLevelEmphasis",
    "LargeHighGrayLevelEmphasis": "LargeAreaHighGrayLevelEmphasis",
}
GLDM_NAMES = {
    "SmallEmphasis": "SmallDependenceEmphasis", "LargeEmphasis": "LargeDependenceEmphasis",
    "GrayLevelNonUniformity": "GrayLevelNonUniformity",
    "SizeNonUniformity": "DependenceNonUniformity",
    "SizeNonUniformityNormalized": "DependenceNonUniformityNormalized",
    "GrayLevelVariance": "GrayLevelVariance", "SizeVariance": "DependenceVariance",
    "Entropy": "DependenceEntropy",
    "LowGrayLevelEmphasis": "LowGrayLevelEmphasis", "HighGrayLevelEmphasis": "HighGrayLevelEmphasis",
    "SmallLowGrayLevelEmphasis": "SmallDependenceLowGrayLevelEmphasis",
    "SmallHighGrayLevelEmphasis": "SmallDependenceHighGrayLevelEmphasis",
    "LargeLowGrayLevelEmphasis": "LargeDependenceLowGrayLevelEmphasis",
    "LargeHighGrayLevelEmphasis": "LargeDependenceHighGrayLevelEmphasis",
}


def glszm_features(P, gray_levels):
    return _size_matrix_features(P[:, np.asarray(gray_levels, int) - 1].astype(float), gray_levels, GLSZM_NAMES)


def gldm_features(P, gray_levels):
    return _size_matrix_features(P[:, np.asarray(gray_levels, int) - 1].astype(float), gray_levels, GLDM_NAMES)


# --------------------------------------------------------------------------- NGTDM
def ngtdm_features(P):
    """P raw [V,Ng,3] = (n_i, s_i, i)."""
    keep = P[:, :, 0].sum(0) != 0
    P = P[:, keep].astype(float)
    n, s, i = P[:, :, 0], P[:, :, 1], P[:, :, 2]
    Nvp = n.sum(1)
    with np.errstate(invalid="ignore", divide="ignore"):
        p = n / Nvp[:, None]
        Ngp = (n > 0).sum(1)
        nz = p != 0
        both = nz[:, :, None] & nz[:, None, :]
        f = {}
        ps = (p * s).sum(1)
        f["Coarseness"] = np.where(ps != 0, 1.0 / np.where(ps != 0, ps, 1), 1e6)
        di = i[:, :, None] - i[:, None, :]
        con = (p[:, :, None] * p[:, None, :] * di ** 2).sum((1, 2)) * s.sum(1) / Nvp
        div = Ngp * (Ngp - 1)
        f["Contrast"] = np.where(div != 0, con / np.where(div != 0, div, 1), 0.0)
        ip = i * p
        ad = np.where(both, np.abs(ip[:, :, None] - ip[:, None, :]), 0.0).sum((1, 2))
        f["Busyness"] = np.where(ad != 0, ps / np.where(ad != 0, ad, 1), 0.0)
        pis = p * s
        num = np.where(both, pis[:, :, None] + pis[:, None, :], 0.0)
        den = p[:, :, None] + p[:, None, :]
        den = np.where(den == 0, 1.0, den)
        f["Complexity"] = (np.abs(di) * num / den).sum((1, 2)) / Nvp
        st = np.where(both, (p[:, :, None] + p[:, None, :]) * di ** 2, 0.0).sum((1, 2))
        ss = s.sum(1)
        f["Strength"] = np.where(ss != 0, st / np.where(ss != 0, ss, 1), 0.0)
    return f
