// GLRLM fast path: kernelRadius 1, full 3-D (13 distance-1 angles), unweighted, 8-bit levels.
// Same semantics as glrlm_voxel<> (vox_features.cuh), restructured around bitmasks: the 27 window
// levels are compared once into per-position equality masks; for each angle every masked window
// voxel that ENDS a run (its successor along the angle is outside the window / unmasked / another
// level) contributes one run whose length (1..3) comes from two more bit tests.  Sums that are
// linear in the runs are exact integers; sum_i pg(i)^2 and the run entropy come from popcounts of
// (equality mask & run-end masks) and a log2 table -- no merged run list, no transcendental calls.
// __host__ __device__ (tests/host_emul checks it on the CPU; test-only).
#pragma once
#include "glcm_fast.cuh"

namespace rb {

struct GlrlmFastTables {
  uint32_t VA[GF_NA], VA2[GF_NA];   // positions whose successor / second successor is inside the window
  uint8_t delta[GF_NA];       // index offset of the angle (dz*9 + dy*3 + dx > 0 for the 13 angles)
  double log2t[32];
  double clog2[32];           // c * log2(c)
  double inv2[256];           // 1 / level^2
};

inline void glrlm_fast_build_tables(GlrlmFastTables& T) {
  int ang[13][3], k = 0;
  for (int z = 1; z >= -1; z--) for (int y = 1; y >= -1; y--) for (int x = 1; x >= -1; x--)
    if (k < 13) { ang[k][0] = z; ang[k][1] = y; ang[k][2] = x; k++; }
  for (int a = 0; a < 13; a++) {
    T.VA[a] = T.VA2[a] = 0;
    T.delta[a] = (uint8_t)(ang[a][0] * 9 + ang[a][1] * 3 + ang[a][2]);
    for (int z = 0; z < 3; z++) for (int y = 0; y < 3; y++) for (int x = 0; x < 3; x++) {
      const int v = z * 9 + y * 3 + x;
      auto pos = [&](int m) {
        const int z2 = z + m * ang[a][0], y2 = y + m * ang[a][1], x2 = x + m * ang[a][2];
        return (z2 < 0 || z2 > 2 || y2 < 0 || y2 > 2 || x2 < 0 || x2 > 2) ? 31 : z2 * 9 + y2 * 3 + x2;
      };
      const int nx = pos(1), nx2 = pos(2);
      if (nx != 31) T.VA[a] |= 1u << v;
      if (nx2 != 31) T.VA2[a] |= 1u << v;
    }
  }
  T.log2t[0] = 0;
  T.clog2[0] = 0;
  for (int c = 1; c < 32; c++) { T.log2t[c] = log2((double)c); T.clog2[c] = c * log2((double)c); }
  T.inv2[0] = 0;
  for (int g = 1; g < 256; g++) T.inv2[g] = 1.0 / ((double)g * g);
}

// wl: the 27 window levels (registers), out: 16 features in GlrlmF order.
//
// Bit-parallel formulation: with E = equality mask of one level class and d = the angle's index
// offset, the voxels whose successor along the angle is in the window AND of the same class are
// NS = OR_classes( E & (E >> d) & VA ).  Then run ends = M & ~NS, "previous voxel is the same class"
// PS = NS << d, "previous two" PS2 = PS & (PS << d), and the run-length-1/2/3 end masks follow with
// three more logic ops -- for all 27 voxels at once.  Everything else is popcounts per class.
// (Round 2 tried a class-free formulation -- every quantity as a sum over the 27 run-end positions, no dynamically
// indexed arrays: 511 instead of 645 warp instructions per voxel, but 4 fp64 accumulations per position and angle and
// more shared-memory table lookups; it was slower than this one and was dropped.)
RB_HD void glrlm_fast_voxel(const int* wl, const GlrlmFastTables& T, double* out) {
  uint32_t e[27];
  RB_EQMASKS_27(wl, e);
  uint32_t M = 0;
  // compact the level classes (data-dependent count): mask + level of each distinct level that occurs at least TWICE.
  // A level that occurs once is a run of length 1 along every angle: its share of every sum below is the same for the
  // 13 angles and is added once (S_*).  27 i.i.d. levels out of 32 have ~12 such singletons and ~7 repeated levels, so
  // the per-angle class loops run ~7 instead of ~18 times (those loops are most of the kernel's instructions).
  uint32_t cls[13];                                       // at most 13 levels can occur twice among 27 voxels
  int clg[13];
  int nl = 0;
  int S_n = 0, S_g = 0, S_g2 = 0;
  double S_ig = 0;
#pragma unroll
  for (int v = 0; v < 27; v++) {
    if (wl[v]) M |= 1u << v;
    if (e[v] && (e[v] & ((1u << v) - 1)) == 0) {
      if (e[v] == (1u << v)) { S_n++; S_g += wl[v]; S_g2 += wl[v] * wl[v]; S_ig += T.inv2[wl[v]]; }
      else { cls[nl] = e[v]; clg[nl] = wl[v]; nl++; }
    }
  }
  const int Np = RB_POPC(M);
  double sum[GLRLM_NF];
#pragma unroll
  for (int k = 0; k < GLRLM_NF; k++) sum[k] = 0;
  int nang = 0;
  for (int a = 0; a < GF_NA; a++) {
    const int d = T.delta[a];
    const uint32_t VA = T.VA[a];
    // cmatrices.c:524-534: an angle none of whose lines holds two masked voxels is dropped
    if (!(((M & VA) & (M >> d)) | ((M & T.VA2[a]) & (M >> (2 * d))))) continue;
    uint32_t NS = 0;
    for (int k = 0; k < nl; k++) NS |= cls[k] & (cls[k] >> d);
    NS &= VA;
    const uint32_t ENDS = M & ~NS, PS = NS << d, PS2 = PS & (PS << d);
    const uint32_t L1 = ENDS & ~PS, L2 = ENDS & PS & ~PS2, L3 = ENDS & PS2;
    const int n1 = RB_POPC(L1), n2 = RB_POPC(L2), n3 = RB_POPC(L3);
    int B1 = S_g2, B2 = 0, B3 = 0, C = S_g, sg = S_n;
    double A1 = S_ig, A2 = 0, A3 = 0, lg = 0;
    for (int k = 0; k < nl; k++) {
      const uint32_t E = cls[k];
      const int c1 = RB_POPC(E & L1), c2 = RB_POPC(E & L2), c3 = RB_POPC(E & L3), ce = c1 + c2 + c3;
      const int g = clg[k], g2 = g * g;
      const double ig = T.inv2[g];
      sg += ce * ce; C += ce * g;
      B1 += c1 * g2; B2 += c2 * g2; B3 += c3 * g2;
      A1 += c1 * ig; A2 += c2 * ig; A3 += c3 * ig;
      lg += T.clog2[c1] + T.clog2[c2] + T.clog2[c3];
    }
    const int Nr = n1 + n2 + n3;
    const double invNr = 1.0 / Nr, invNr2 = invNr * invNr;
    const int lre_n = n1 + 4 * n2 + 9 * n3, B = B1 + B2 + B3;
    sum[R_ShortRunEmphasis] += (n1 + n2 * 0.25 + n3 * (1.0 / 9.0)) * invNr;
    sum[R_LongRunEmphasis] += lre_n * invNr;
    sum[R_GrayLevelNonUniformity] += sg * invNr;
    sum[R_GrayLevelNonUniformityNormalized] += sg * invNr2;
    const int rl = n1 * n1 + n2 * n2 + n3 * n3;
    sum[R_RunLengthNonUniformity] += rl * invNr;
    sum[R_RunLengthNonUniformityNormalized] += rl * invNr2;
    sum[R_RunPercentage] += (double)Nr / Np;
    sum[R_GrayLevelVariance] += (double)(Nr * B - C * C) * invNr2;
    sum[R_RunVariance] += (double)(Nr * lre_n - Np * Np) * invNr2;
    sum[R_RunEntropy] += T.log2t[Nr] - lg * invNr;
    sum[R_LowGrayLevelRunEmphasis] += (A1 + A2 + A3) * invNr;
    sum[R_HighGrayLevelRunEmphasis] += B * invNr;
    sum[R_ShortRunLowGrayLevelEmphasis] += (A1 + A2 * 0.25 + A3 * (1.0 / 9.0)) * invNr;
    sum[R_ShortRunHighGrayLevelEmphasis] += (B1 + B2 * 0.25 + B3 * (1.0 / 9.0)) * invNr;
    sum[R_LongRunLowGrayLevelEmphasis] += (A1 + 4.0 * A2 + 9.0 * A3) * invNr;
    sum[R_LongRunHighGrayLevelEmphasis] += (double)(B1 + 4 * B2 + 9 * B3) * invNr;
    nang++;
  }
  const double inv = nang ? 1.0 / nang : NAN;
#pragma unroll
  for (int k = 0; k < GLRLM_NF; k++) out[k] = nang ? sum[k] * inv : NAN;
}

}  // namespace rb
