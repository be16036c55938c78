// Per-voxel arithmetic of the 3-D local binary pattern (reference radiomics/imageoperations.py:1169-1314, getLBP3DImage),
// __host__ __device__ so that tests/host_emul/lbp3d_emul.cpp runs the same code on the CPU.  For one ROI voxel p:
//   f_v  = cubic B-spline sample at p + vertex v (scipy.ndimage.map_coordinates(order=3, mode='constant'): mirrored
//          neighbourhood inside [0, n-1] on every axis, 0 as soon as one coordinate leaves it), cast to the image's dtype
//          (integers: round half away from zero, clamp to the type's range; float32: round to float32);
//   k    = Fisher kurtosis of the Nv samples (scipy.stats.kurtosis, biased, two-pass; NaN when m2 <= (eps * mean)^2);
//   s_v  = f_v >= img[p];  c_nm = sum_v s_v Y_nm(v);  E_n = sum_v (sum_m c_nm Y_nm(v))^2 (complex square);
//   map n+1 = Re(sqrt(E_n)).
#pragma once
#include <math.h>
#include <stdint.h>

#include "pixel.cuh"                              // RB_HD, rb_dtype, load_f64

namespace rb {

constexpr int LBP_MAX_NV = 162;                 // icosphere subdivision 2
constexpr int LBP_MAX_LEVELS = 4;
constexpr int LBP_MAX_KPOS = LBP_MAX_LEVELS * (LBP_MAX_LEVELS + 1) / 2;    // harmonics with m >= 0

// Sphere vertices and harmonics table; passed by value to the kernel (__grid_constant__, < 32 KB of parameters).
// y_re / y_im [v][n (n + 1) / 2 + m] = Y_n^m(vertex v) for m >= 0; Y_n^-m = (-1)^m conj(Y_n^m).
struct Lbp3dTables {
  int nv, levels, sample_dt, pad_;
  double vert[LBP_MAX_NV][3];                   // (z, y, x) offsets in voxels
  double y_re[LBP_MAX_NV][LBP_MAX_KPOS];
  double y_im[LBP_MAX_NV][LBP_MAX_KPOS];
};

// SciPy's cast of an interpolated value to an integer output: +-0.5 towards the sign, clamp, truncate
RB_HD double lbp_round_clamp(double v, double lo, double hi) {
  v = v > 0 ? v + 0.5 : v - 0.5;
  v = v > hi ? hi : v;
  v = v < lo ? lo : v;
  return (double)(long long)v;
}

RB_HD double lbp_cast(double v, int dt) {
  switch (dt) {
    case RB_DT_FLOAT64: return v;
    case RB_DT_FLOAT32: return (double)(float)v;
    case RB_DT_INT16: return lbp_round_clamp(v, -32768.0, 32767.0);
    case RB_DT_INT32: return lbp_round_clamp(v, -2147483648.0, 2147483647.0);
    case RB_DT_UINT8: return lbp_round_clamp(v, 0.0, 255.0);
    case RB_DT_UINT16: return lbp_round_clamp(v, 0.0, 65535.0);
    default: return lbp_round_clamp(v, -9223372036854775808.0, 9223372036854774784.0);
  }
}

RB_HD int lbp_mirror(int i, int n) {
  if (n == 1) return 0;
  const int period = 2 * n - 2;
  i = i < 0 ? -i : i;
  i %= period;
  return i >= n ? period - i : i;
}

// cubic B-spline interpolation of coefficient volume `c` (Z, Y, X) at continuous index (cz, cy, cx)
RB_HD double lbp_spline_sample(const double* __restrict__ c, int Z, int Y, int X, double cz, double cy, double cx) {
  const double cc[3] = {cz, cy, cx};
  const int nn[3] = {Z, Y, X};
  double W[3][4];
  int I[3][4];
#pragma unroll
  for (int d = 0; d < 3; d++) {
    if (!(cc[d] >= 0.0 && cc[d] <= (double)(nn[d] - 1))) return 0.0;
    const double f = floor(cc[d]);
    const double y = cc[d] - f, z = 1.0 - y;
    W[d][1] = (y * y * (y - 2.0) * 3.0 + 4.0) / 6.0;
    W[d][2] = (z * z * (z - 2.0) * 3.0 + 4.0) / 6.0;
    W[d][0] = z * z * z / 6.0;
    W[d][3] = 1.0 - W[d][0] - W[d][1] - W[d][2];
#pragma unroll
    for (int k = 0; k < 4; k++) I[d][k] = lbp_mirror((int)f - 1 + k, nn[d]);
  }
  const long long plane = (long long)Y * X;
  double v = 0.0;
#pragma unroll
  for (int a = 0; a < 4; a++)
#pragma unroll
    for (int b = 0; b < 4; b++) {
      const double wab = W[0][a] * W[1][b];
      const double* row = c + (long long)I[0][a] * plane + (long long)I[1][b] * X;
#pragma unroll
      for (int k = 0; k < 4; k++) v += wab * W[2][k] * row[I[2][k]];
    }
  return v;
}

// Re(sqrt(re + i im)), principal branch (what numpy's complex sqrt returns)
RB_HD double lbp_re_csqrt(double re, double im) {
  const double d = hypot(re, im);
  if (re >= 0.0) return sqrt(0.5 * (d + re));
  const double t = sqrt(0.5 * (d - re));
  return t == 0.0 ? 0.0 : fabs(im) / (2.0 * t);
}

// All outputs of voxel (z, y, x): out[l * ostride] for l < levels are the level maps, out[levels * ostride] the kurtosis.
// `coef`: the B-spline coefficients of the image, `img`: the image itself (centre value; dtype code img_dt).
RB_HD void lbp3d_voxel(const double* __restrict__ coef, const void* __restrict__ img, int img_dt, int Z, int Y, int X, int z,
                       int y, int x, const Lbp3dTables& T, double* __restrict__ out, long long ostride) {
  const int nv = T.nv, L = T.levels;
  const double centre = load_f64(img, img_dt, ((long long)z * Y + y) * X + x);
  double f[LBP_MAX_NV];
  double sum = 0.0;
  for (int v = 0; v < nv; v++) {
    const double s = lbp_cast(lbp_spline_sample(coef, Z, Y, X, (double)z + T.vert[v][0], (double)y + T.vert[v][1],
                                                (double)x + T.vert[v][2]), T.sample_dt);
    f[v] = s;
    sum += s;
  }
  const double mean = sum / nv;
  double m2 = 0.0, m4 = 0.0;
  uint64_t bits[(LBP_MAX_NV + 63) / 64] = {0, 0, 0};
  for (int v = 0; v < nv; v++) {
    const double d = f[v] - mean, d2 = d * d;
    m2 += d2;
    m4 += d2 * d2;
    if (f[v] >= centre) bits[v >> 6] |= 1ull << (v & 63);
  }
  m2 /= nv;
  m4 /= nv;
  const double eps = T.sample_dt == RB_DT_FLOAT32 ? 1.1920928955078125e-07 : 2.220446049250313e-16;
  const double zero = eps * mean;
  out[(long long)L * ostride] = m2 <= zero * zero ? (double)NAN : m4 / (m2 * m2) - 3.0;

  // c_nm for m >= 0 (c_n,-m = (-1)^m conj(c_nm), exactly, because the table obeys the same symmetry)
  const int kp = L * (L + 1) / 2;
  double cr[LBP_MAX_KPOS], ci[LBP_MAX_KPOS];
  for (int k = 0; k < kp; k++) cr[k] = ci[k] = 0.0;
  for (int v = 0; v < nv; v++)
    if (bits[v >> 6] >> (v & 63) & 1)
      for (int k = 0; k < kp; k++) { cr[k] += T.y_re[v][k]; ci[k] += T.y_im[v][k]; }
  double er[LBP_MAX_LEVELS], ei[LBP_MAX_LEVELS];
  for (int n = 0; n < L; n++) er[n] = ei[n] = 0.0;
  for (int v = 0; v < nv; v++) {
    for (int n = 0; n < L; n++) {
      const int k0 = n * (n + 1) / 2;
      double gr = 0.0, gi = 0.0;
      for (int m = -n; m <= n; m++) {
        const int k = k0 + (m < 0 ? -m : m);
        double a = cr[k], b = ci[k], p = T.y_re[v][k], q = T.y_im[v][k];
        if (m < 0) {                                  // (-1)^m conj(.) on both factors: the signs cancel
          b = -b;
          q = -q;
        }
        gr += a * p - b * q;
        gi += a * q + b * p;
      }
      er[n] += gr * gr - gi * gi;
      ei[n] += 2.0 * gr * gi;
    }
  }
  for (int n = 0; n < L; n++) out[(long long)n * ostride] = lbp_re_csqrt(er[n], ei[n]);
}

}  // namespace rb
