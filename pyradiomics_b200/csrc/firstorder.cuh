// First-order statistics of one kernel window (SURVEY.md section 8f rank 2; reference
// radiomics/firstorder.py:40-474): 18 features from the raw intensities of the masked window
// voxels (NaN-aware in the reference = only masked, in-volume voxels count) and, for Entropy /
// Uniformity, the histogram of their discretised levels.  __host__ __device__ like the texture math.
//
// Two bodies share the stage after the sort (firstorder_sorted), so their results are the same bits:
//   firstorder_voxel<WCAP>  any window: insertion sort in place, level classes by first-occurrence compaction
//   firstorder_full_body    a full 3x3x3 window (27 values, no NaN, 27 non-zero levels): stable ranks from the 351 pair
//                           compares, a scatter into per-thread scratch, level classes from the equality masks
#pragma once
#include "straightline.inc"
#include "vox_features.cuh"

namespace rb {

enum FirstOrderF { F_P10, F_P90, F_Energy, F_Entropy, F_IQR, F_Kurtosis, F_Maximum, F_MAD, F_Mean, F_Median, F_Minimum,
                   F_Range, F_RMAD, F_RMS, F_Skewness, F_TotalEnergy, F_Uniformity, F_Variance, FIRSTORDER_NF };

// numpy's default ("linear") percentile of sorted x[0..n-1], including its lerp form
template <typename XS>
RB_HD double fo_percentile(const XS& x, int n, double q) {
  const double pos = (double)(n - 1) * q / 100.0;
  int lo = (int)pos;
  if (lo > n - 1) lo = n - 1;
  const int hi = lo + 1 < n ? lo + 1 : n - 1;
  const double t = pos - (double)lo, a = x[lo], b = x[hi], d = b - a;
  return t >= 0.5 ? b - d * (1.0 - t) : a + d * t;
}

// a level class of c of the window's voxels (invN = 1 / their number): its Entropy and Uniformity terms
RB_HD void fo_level_class(int c, double invN, double& ent, double& uni) {
  const double p = c * invN;
  ent -= p * log2(p + EPS);
  uni += p * p;
}

// The 18 features from the n window intensities in ascending order, x[i] (a pointer or an accessor with operator[]),
// and the level classes' Entropy / Uniformity.  Every sum runs over x in order.
template <typename XS>
RB_HD void firstorder_sorted(const XS& x, int n, double ent, double uni, double shift, double voxel_volume, double* out) {
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
  const double m2s = m2 == 0 ? 1.0 : m2;
  const double xmin = x[0], xmax = x[n - 1];
  out[F_P10] = p10; out[F_P90] = p90; out[F_Energy] = en; out[F_Entropy] = ent;
  out[F_IQR] = fo_percentile(x, n, 75.0) - fo_percentile(x, n, 25.0);
  out[F_Kurtosis] = m4 / (m2s * m2s);
  out[F_Maximum] = xmax; out[F_MAD] = mad / n; out[F_Mean] = mean; out[F_Median] = fo_percentile(x, n, 50.0);
  out[F_Minimum] = xmin; out[F_Range] = xmax - xmin; out[F_RMAD] = rmad / kn; out[F_RMS] = sqrt(en / n);
  out[F_Skewness] = m3 / (m2s * sqrt(m2s)); out[F_TotalEnergy] = en * voxel_volume; out[F_Uniformity] = uni;
  out[F_Variance] = m2;
}

// insertion sort of x[0..n-1] in place: stable, and with NaN the order every body of the window must reproduce
RB_HD void fo_insertion_sort(double* x, int n) {
  for (int i = 1; i < n; i++) {
    const double v = x[i];
    int j = i - 1;
    while (j >= 0 && x[j] > v) { x[j + 1] = x[j]; j--; }
    x[j + 1] = v;
  }
}

// Entropy / Uniformity of the nl level classes cnt[] (N window voxels with a level), in class order
RB_HD void fo_level_classes(const int* cnt, int nl, int N, double& ent, double& uni) {
  const double invN = 1.0 / (N ? N : 1);
  ent = 0; uni = 0;
  for (int k = 0; k < nl; k++) fo_level_class(cnt[k], invN, ent, uni);
}

// x: the n window intensities (unsorted, destroyed: sorted in place); w: the window's levels (0 = not
// in the kernel), wn entries
template <int WCAP>
RB_HD void firstorder_voxel(double* x, int n, const uint16_t* w, int wn, double shift, double voxel_volume, double* out) {
  fo_insertion_sort(x, n);                   // n <= 343, typically 27
  // level histogram of the window, classes in order of first occurrence
  int val[WCAP]; uint16_t lidx[WCAP]; int cnt[WCAP];
  const int nl = compact_levels<WCAP>(w, wn, val, lidx);
  for (int k = 0; k < nl; k++) cnt[k] = 0;
  int N = 0;
  for (int p = 0; p < wn; p++) if (lidx[p] != NOLEV) { cnt[lidx[p]]++; N++; }
  double ent, uni;
  fo_level_classes(cnt, nl, N, ent, uni);
  firstorder_sorted(x, n, ent, uni, shift, voxel_volume, out);
}

// element i of a per-thread column of scratch with element stride st (device: shared memory laid out [entry][thread])
struct FoColumn {
  const double* p;
  int st;
  RB_HD double operator[](int i) const { return p[i * st]; }
};

// A full window: xv = its 27 intensities in window (z, y, x) order, none NaN; wl = its 27 levels, all non-zero.  scr:
// per-thread scratch of 27 doubles, element stride st.  Bit-identical to firstorder_voxel<27> on the same window:
//   * the insertion sort is stable, so x_i precedes x_j (i < j) exactly when x_i <= x_j -- with no NaN that is a total
//     order, and rank_j = #{i < j : x_i <= x_j} + #{i > j : x_j < x_i} is x_j's position in the sorted array, -0.0 and
//     +0.0 included; the values are scattered to scr[rank] and read back in order;
//   * a level class is a position that is the lowest set bit of its own equality mask, taken in increasing position:
//     the classes of compact_levels, in its order, with popcount members, and N = 27.
template <typename W>
RB_HD void firstorder_full_body(const double* xv, const W* wl, double shift, double voxel_volume, double* scr, int st,
                                double* out) {
  int rank[27];
#pragma unroll
  for (int i = 0; i < 27; i++) rank[i] = 0;
#pragma unroll
  for (int j = 1; j < 27; j++)
#pragma unroll
    for (int i = 0; i < j; i++) {
      const int le = xv[i] <= xv[j];
      rank[j] += le;
      rank[i] += 1 - le;
    }
#pragma unroll
  for (int i = 0; i < 27; i++) scr[rank[i] * st] = xv[i];
  int key[27];
#pragma unroll
  for (int v = 0; v < 27; v++) key[v] = (int)wl[v];
  uint32_t e[27];
  RB_EQMASKS_27_KEY(key, e);
  const double invN = 1.0 / 27;
  double ent = 0, uni = 0;
#pragma unroll
  for (int v = 0; v < 27; v++)
    if ((e[v] & ((1u << v) - 1)) == 0) fo_level_class(RB_POPC(e[v]), invN, ent, uni);
  firstorder_sorted(FoColumn{scr, st}, 27, ent, uni, shift, voxel_volume, out);
}

}  // namespace rb
