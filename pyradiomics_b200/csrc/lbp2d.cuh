// Per-pixel arithmetic of the 2-D local binary pattern (reference radiomics/imageoperations.py:1094-1166, getLBP2DImage ->
// skimage.feature.local_binary_pattern), __host__ __device__ so that tests/host_emul/lbp2d_emul.cpp runs the same code on
// the CPU.  For pixel (r, c) of one slice, k = 0..P-1:
//   t_k = bilinear sample at (r' = r + rp[k], c' = c + cp[k]): minr = floor, maxr = ceil, dr = r' - minr (cols alike),
//         top = (1 - dc) tl + dc tr, bottom = (1 - dc) bl + dc br, t = (1 - dr) top + dr bottom; a corner outside the
//         slice reads 0;
//   s_k = (t_k - centre >= 0);
// then the code of `method` (default, ror, uniform, nri_uniform, var).  Every product, sum, difference and quotient is
// rounded on its own: the device spells them as __d*_rn (no FMA contraction), the host build needs -ffp-contract=off.
#pragma once
#include <math.h>
#include <stdint.h>

#include "lbp3d.cuh"                             // RB_HD, load_f64

namespace rb {

constexpr int LBP2D_MAX_P = 31;                  // the library's int32 weights 2**arange(P) overflow beyond
enum { LBP2D_DEFAULT = 0, LBP2D_ROR = 1, LBP2D_UNIFORM = 2, LBP2D_NRI_UNIFORM = 3, LBP2D_VAR = 4 };

// sample offsets, rp = round(-R sin(2 pi k / P), 5), cp = round(R cos(2 pi k / P), 5), computed by the host
struct Lbp2dOffsets {
  int P, pad_;
  double rp[LBP2D_MAX_P];
  double cp[LBP2D_MAX_P];
};

#ifdef __CUDA_ARCH__
RB_HD double l2_add(double a, double b) { return __dadd_rn(a, b); }
RB_HD double l2_sub(double a, double b) { return __dsub_rn(a, b); }
RB_HD double l2_mul(double a, double b) { return __dmul_rn(a, b); }
RB_HD double l2_div(double a, double b) { return __ddiv_rn(a, b); }
RB_HD int l2_popc(uint32_t v) { return __popc(v); }
#else
RB_HD double l2_add(double a, double b) { return a + b; }
RB_HD double l2_sub(double a, double b) { return a - b; }
RB_HD double l2_mul(double a, double b) { return a * b; }
RB_HD double l2_div(double a, double b) { return a / b; }
RB_HD int l2_popc(uint32_t v) { return __builtin_popcount(v); }
#endif

// One slice seen through an index mapping: pixel (r, c) is at base + r * rs + c * cs of the volume.
struct Lbp2dSlice {
  const void* img;
  int dt, rows, cols;
  long long base, rs, cs;
};

RB_HD double lbp2d_pixel_value(const Lbp2dSlice& s, long long r, long long c) {
  if (r < 0 || r >= s.rows || c < 0 || c >= s.cols) return 0.0;
  return load_f64(s.img, s.dt, s.base + r * s.rs + c * s.cs);
}

RB_HD double lbp2d_sample(const Lbp2dSlice& s, double r, double c) {
  const double fr = floor(r), fc = floor(c);
  const long long minr = (long long)fr, minc = (long long)fc, maxr = (long long)ceil(r), maxc = (long long)ceil(c);
  const double dr = l2_sub(r, (double)minr), dc = l2_sub(c, (double)minc);
  const double tl = lbp2d_pixel_value(s, minr, minc), tr = lbp2d_pixel_value(s, minr, maxc);
  const double bl = lbp2d_pixel_value(s, maxr, minc), br = lbp2d_pixel_value(s, maxr, maxc);
  const double wc = l2_sub(1.0, dc), wr = l2_sub(1.0, dr);
  const double top = l2_add(l2_mul(wc, tl), l2_mul(dc, tr));
  const double bottom = l2_add(l2_mul(wc, bl), l2_mul(dc, br));
  return l2_add(l2_mul(wr, top), l2_mul(dr, bottom));
}

// the code of one sign-bit pattern (bit k = s_k), P <= 31
RB_HD double lbp2d_code(int method, uint32_t bits, int P) {
  if (method == LBP2D_DEFAULT) return (double)bits;
  if (method == LBP2D_ROR) {
    uint32_t v = bits, best = bits;
    for (int i = 1; i < P; i++) {
      v = (v >> 1) | ((v & 1u) << (P - 1));
      best = v < best ? v : best;
    }
    return (double)best;
  }
  const int changes = l2_popc((bits ^ (bits >> 1)) & ((1u << (P - 1)) - 1u));   // k = 0..P-2, not circular
  const int n_ones = l2_popc(bits);
  if (method == LBP2D_UNIFORM) return changes <= 2 ? (double)n_ones : (double)(P + 1);
  // LBP2D_NRI_UNIFORM
  if (changes > 2) return (double)(P * (P - 1) + 2);
  if (n_ones == 0) return 0.0;
  if (n_ones == P) return (double)(P * (P - 1) + 1);
  int first_one = 0, first_zero = 0;
  while (!(bits >> first_one & 1u)) first_one++;
  while (bits >> first_zero & 1u) first_zero++;
  const int rot_index = first_one == 0 ? n_ones - first_zero : P - first_one;
  return (double)(1 + (n_ones - 1) * P + rot_index);
}

// LBP of pixel (r, c) of slice `s` (METHOD one of the LBP2D_* codes)
template <int METHOD>
RB_HD double lbp2d_pixel(const Lbp2dSlice& s, int r, int c, const Lbp2dOffsets& O) {
  const int P = O.P;
  const double centre = lbp2d_pixel_value(s, r, c);
  uint32_t bits = 0;
  double sum = 0.0, sq = 0.0;
  for (int k = 0; k < P; k++) {
    const double t = lbp2d_sample(s, l2_add((double)r, O.rp[k]), l2_add((double)c, O.cp[k]));
    if (METHOD == LBP2D_VAR) {
      sum = l2_add(sum, t);
      sq = l2_add(sq, l2_mul(t, t));
    } else if (l2_sub(t, centre) >= 0.0) {
      bits |= 1u << k;
    }
  }
  if (METHOD == LBP2D_VAR) {
    const double v = l2_div(l2_sub(sq, l2_div(l2_mul(sum, sum), (double)P)), (double)P);
    return v != 0.0 ? v : (double)NAN;
  }
  return lbp2d_code(METHOD, bits, P);
}

// What NumPy stores when a float64 value is assigned into an array of type T (the reference's im_arr[idx, ...] = slice,
// an unsafe cast), written out because neither machine's conversion gives it: the GPU's cvt.rzi saturates, and C leaves
// out-of-range conversions undefined.  The rule is NumPy's on x86-64, where its cast loops use the truncating
// cvttsd2si / cvttpd2dq family, whose out-of-range and NaN result is the "integer indefinite" (the type's minimum):
//   float64: the value;  float32: rounded to nearest, +-inf beyond the float32 range, NaN stays NaN;
//   int32: trunc(v) when -2^31 <= trunc(v) < 2^31, else INT32_MIN (NaN and +-inf included);
//   int16, uint16, uint8: the low 16 / 8 bits of that int32 (NumPy converts through a 32-bit integer): 70000.5 -> 4464,
//         2^31 - 1 -> -1 / 65535 / 255, 2^31 -> 0;
//   int64: trunc(v) when -2^63 <= trunc(v) < 2^63, else INT64_MIN.
// Measured with NumPy 2.3 for every dtype on arrays of 1 to 257 elements at four offsets (the vector loops and the scalar
// tail) with and without NumPy's AVX / AVX2 / AVX-512 dispatch: one result per value every time.  AArch64's fcvtzs
// saturates instead, so NumPy there differs for values outside int32 / int64; that platform is not matched.
RB_HD int32_t numpy_cast_i32(double v) { return v > -2147483649.0 && v < 2147483648.0 ? (int32_t)v : INT32_MIN; }
template <typename T> RB_HD T numpy_cast(double v);
template <> RB_HD double numpy_cast<double>(double v) { return v; }
template <> RB_HD float numpy_cast<float>(double v) { return (float)v; }
template <> RB_HD int32_t numpy_cast<int32_t>(double v) { return numpy_cast_i32(v); }
template <> RB_HD int16_t numpy_cast<int16_t>(double v) { return (int16_t)(uint16_t)(uint32_t)numpy_cast_i32(v); }
template <> RB_HD uint16_t numpy_cast<uint16_t>(double v) { return (uint16_t)(uint32_t)numpy_cast_i32(v); }
template <> RB_HD uint8_t numpy_cast<uint8_t>(double v) { return (uint8_t)(uint32_t)numpy_cast_i32(v); }
template <> RB_HD int64_t numpy_cast<int64_t>(double v) {
  return v >= -9223372036854775808.0 && v < 9223372036854775808.0 ? (int64_t)v : INT64_MIN;
}

// slice geometry of voxel (z, y, x) of a (Z, Y, X) volume cut along `axis` (the reference's swapaxes(0, axis)):
// axis 0: rows y, cols x;  axis 1: rows z, cols x;  axis 2: rows y, cols z.
RB_HD void lbp2d_slice_of(const void* img, int dt, int Z, int Y, int X, int axis, int z, int y, int x, Lbp2dSlice& s, int& r,
                          int& c) {
  const long long plane = (long long)Y * X;
  s.img = img;
  s.dt = dt;
  if (axis == 0) {
    s.rows = Y; s.cols = X; s.rs = X; s.cs = 1; r = y; c = x;
  } else if (axis == 1) {
    s.rows = Z; s.cols = X; s.rs = plane; s.cs = 1; r = z; c = x;
  } else {
    s.rows = Y; s.cols = Z; s.rs = X; s.cs = plane; r = y; c = z;
  }
  s.base = ((long long)z * Y + y) * X + x - (long long)r * s.rs - (long long)c * s.cs;
}

}  // namespace rb
