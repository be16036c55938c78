// First-order statistics of one kernel window (SURVEY.md section 8f rank 2; reference
// radiomics/firstorder.py:40-474): 18 features from the raw intensities of the masked window
// voxels (NaN-aware in the reference = only masked, in-volume voxels count) and, for Entropy /
// Uniformity, the histogram of their discretised levels.  __host__ __device__ like the texture math.
#pragma once
#include "vox_features.cuh"

namespace rb {

enum FirstOrderF { F_P10, F_P90, F_Energy, F_Entropy, F_IQR, F_Kurtosis, F_Maximum, F_MAD, F_Mean, F_Median, F_Minimum,
                   F_Range, F_RMAD, F_RMS, F_Skewness, F_TotalEnergy, F_Uniformity, F_Variance, FIRSTORDER_NF };

// numpy's default ("linear") percentile of sorted x[0..n-1], including its lerp form
RB_HD double fo_percentile(const double* x, int n, double q) {
  const double pos = (double)(n - 1) * q / 100.0;
  int lo = (int)pos;
  if (lo > n - 1) lo = n - 1;
  const int hi = lo + 1 < n ? lo + 1 : n - 1;
  const double t = pos - (double)lo, a = x[lo], b = x[hi], d = b - a;
  return t >= 0.5 ? b - d * (1.0 - t) : a + d * t;
}

// x: the n window intensities (unsorted, destroyed: sorted in place); w: the window's levels (0 = not
// in the kernel), wn entries
template <int WCAP>
RB_HD void firstorder_voxel(double* x, int n, const uint16_t* w, int wn, double shift, double voxel_volume, double* out) {
  for (int i = 1; i < n; i++) {              // insertion sort (n <= 343, typically 27)
    const double v = x[i];
    int j = i - 1;
    while (j >= 0 && x[j] > v) { x[j + 1] = x[j]; j--; }
    x[j + 1] = v;
  }
  double sum = 0, en = 0;
  for (int i = 0; i < n; i++) { sum += x[i]; const double s = x[i] + shift; en += s * s; }
  // means divide by n as np.mean does: sum * (1 / n) misses a constant window's value by an ulp for some n, and then
  // Variance / Skewness / Kurtosis of a flat window come out as ~1e-30 / +-1 / 1 instead of 0
  const double mean = sum / n;
  double mad = 0, m2 = 0, m3 = 0, m4 = 0;
  for (int i = 0; i < n; i++) {
    const double d = x[i] - mean, d2 = d * d;
    mad += fabs(d); m2 += d2; m3 += d2 * d; m4 += d2 * d2;
  }
  m2 /= n; m3 /= n; m4 /= n;
  const double p10 = fo_percentile(x, n, 10.0), p90 = fo_percentile(x, n, 90.0);
  double ks = 0; int kn = 0;
  for (int i = 0; i < n; i++) if (!(x[i] < p10) && !(x[i] > p90)) { ks += x[i]; kn++; }
  const double kmean = ks / kn;
  double rmad = 0;
  for (int i = 0; i < n; i++) if (!(x[i] < p10) && !(x[i] > p90)) rmad += fabs(x[i] - kmean);
  // level histogram of the window
  int val[WCAP]; uint16_t lidx[WCAP]; int cnt[WCAP];
  const int nl = compact_levels<WCAP>(w, wn, val, lidx);
  for (int k = 0; k < nl; k++) cnt[k] = 0;
  int N = 0;
  for (int p = 0; p < wn; p++) if (lidx[p] != NOLEV) { cnt[lidx[p]]++; N++; }
  const double invN = 1.0 / (N ? N : 1);
  double ent = 0, uni = 0;
  for (int k = 0; k < nl; k++) { const double p = cnt[k] * invN; ent -= p * log2(p + EPS); uni += p * p; }
  const double m2s = m2 == 0 ? 1.0 : m2;
  out[F_P10] = p10; out[F_P90] = p90; out[F_Energy] = en; out[F_Entropy] = ent;
  out[F_IQR] = fo_percentile(x, n, 75.0) - fo_percentile(x, n, 25.0);
  out[F_Kurtosis] = m4 / (m2s * m2s);
  out[F_Maximum] = x[n - 1]; out[F_MAD] = mad / n; out[F_Mean] = mean; out[F_Median] = fo_percentile(x, n, 50.0);
  out[F_Minimum] = x[0]; out[F_Range] = x[n - 1] - x[0]; out[F_RMAD] = rmad / kn; out[F_RMS] = sqrt(en / n);
  out[F_Skewness] = m3 / (m2s * sqrt(m2s)); out[F_TotalEnergy] = en * voxel_volume; out[F_Uniformity] = uni;
  out[F_Variance] = m2;
}

}  // namespace rb
