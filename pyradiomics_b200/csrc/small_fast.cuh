// Fast paths of GLSZM, GLDM and NGTDM for the headline configuration (kernelRadius 1, full 3-D,
// distance-1 26-neighbourhood, 8-bit levels).  Same semantics as glszm_voxel / gldm_voxel /
// ngtdm_voxel (vox_features.cuh, the generic fallback and cross-check), built on the 27 x 27-bit
// equality masks of the window like the GLCM / GLRLM fast paths:
//   GLDM  dependence of a voxel = popcount(close-level mask & static neighbour mask); merged
//         (level, dependence) counts = popcount(equal-(level, dependence) mask)
//   NGTDM a full-window body in exact integers and a general one; Busyness from one sort, Contrast and
//         Strength in closed forms of integer moments, only Complexity keeps a pairwise level loop
//   GLSZM zones of one level = flood fill of its equality mask by separable bitmask dilation
// __host__ __device__ (tests/host_emul checks them on the CPU; test-only).
#pragma once
#include "glcm_fast.cuh"

namespace rb {

struct SmallFastTables {
  double log2t[32];     // log2(c), c = 0..31
  double inv2[256];     // 1 / g^2
  double invsq[32];     // 1 / j^2, j = 1..28
  double rcp[64];       // 1 / c
  double dclog2[32];    // (c + 1) log2(c + 1) - c log2(c): what one more zone adds to a (level, size) group of c
};

inline void small_fast_build_tables(SmallFastTables& T) {
  T.log2t[0] = 0; T.invsq[0] = 0; T.inv2[0] = 0; T.rcp[0] = 0;
  for (int c = 1; c < 32; c++) { T.log2t[c] = log2((double)c); T.invsq[c] = 1.0 / ((double)c * c); }
  for (int g = 1; g < 256; g++) T.inv2[g] = 1.0 / ((double)g * g);
  for (int c = 1; c < 64; c++) T.rcp[c] = 1.0 / (double)c;
  for (int c = 0; c < 32; c++) T.dclog2[c] = (c + 1) * log2((double)(c + 1)) - (c ? c * log2((double)c) : 0.0);
}

// 26-neighbourhood of window position v inside the 3x3x3 window (compile-time constant per v)
RB_HD constexpr uint32_t nb26(int v) {
  uint32_t m = 0;
  const int z = v / 9, y = (v / 3) % 3, x = v % 3;
  for (int dz = -1; dz <= 1; dz++) for (int dy = -1; dy <= 1; dy++) for (int dx = -1; dx <= 1; dx++) {
    if (!dz && !dy && !dx) continue;
    const int z2 = z + dz, y2 = y + dy, x2 = x + dx;
    if (z2 < 0 || z2 > 2 || y2 < 0 || y2 > 2 || x2 < 0 || x2 > 2) continue;
    m |= 1u << (z2 * 9 + y2 * 3 + x2);
  }
  return m;
}
template <int V> struct NB26 { static constexpr uint32_t value = nb26(V); };

// compile-time unrolled loop over the 27 window positions: F::template run<V>(args...)
template <int V, int END> struct ForPos {
  template <typename F> static RB_HD void go(F& f) { f.template at<V>(); ForPos<V + 1, END>::go(f); }
};
template <int END> struct ForPos<END, END> { template <typename F> static RB_HD void go(F&) {} };

// ---------------------------------------------------------------------------------------- GLDM
// Two bodies, chosen by the window alone: FULL (all 27 levels non-zero) has no unmasked positions, so Nz = 27 and the
// reciprocals are constants.  The dependence counts n_j come from a packed histogram (DependenceNonUniformity =
// sum_j n_j^2), the merged (level, dependence) counts from the equality masks of the keys g << 5 | dependence; once
// those keys are formed the levels and the level masks are dead, which keeps the kernel within 128 registers.
struct GldmPass1 {
  const uint32_t* cl; int* dep;
  template <int V> RB_HD void at() { dep[V] = (int)RB_POPC(cl[V] & NB26<V>::value); }
};

template <bool FULL>
RB_HD void gldm_fast_body(const int* wl, int alpha, const SmallFastTables& T, double* out) {
  uint32_t eq[27];
  if (FULL) RB_EQMASKS_27_KEY(wl, eq);
  else RB_EQMASKS_27(wl, eq);
  int gl = 0;
#pragma unroll
  for (int v = 0; v < 27; v++) gl += RB_POPC(eq[v]);
  uint32_t cl[27];
  if (alpha == 0) {
#pragma unroll
    for (int v = 0; v < 27; v++) cl[v] = eq[v];
  } else {
    // "dependent" relation |g_u - g_v| <= alpha between masked voxels
#pragma unroll
    for (int v = 0; v < 27; v++) cl[v] = 0;
#pragma unroll
    for (int p = 0; p < 27; p++)
#pragma unroll
      for (int q = p + 1; q < 27; q++) {
        const int d = wl[p] - wl[q];
        if ((FULL || (wl[p] && wl[q])) && d <= alpha && -d <= alpha) { cl[p] |= 1u << q; cl[q] |= 1u << p; }
      }
  }
  int dep[27];
  GldmPass1 p1{cl, dep};
  ForPos<0, 27>::go(p1);
  int Nz = 0, Sj = 0, Sj2 = 0, B = 0, C = 0, X4 = 0;
  double Sinv = 0, A = 0, X1 = 0, X2 = 0, X3 = 0, lg = 0;
  unsigned long long h0 = 0, h1 = 0, h2 = 0;   // dependence histogram, 5-bit fields: 0..11 | 12..23 | 24..26
  int key[27];                         // g << 5 | dependence; unmasked positions: distinct negative sentinels
#pragma unroll
  for (int v = 0; v < 27; v++) {
    const bool in = FULL || wl[v];
    const int g = wl[v], g2 = g * g, j = dep[v] + 1, j2 = j * j;
    key[v] = in ? g << 5 | dep[v] : -1 - v;
    if (in) {
      const double ig = T.inv2[g], ij = T.invsq[j];
      Nz++; Sj += j; Sj2 += j2; B += g2; C += g; X4 += g2 * j2;
      Sinv += ij; A += ig; X1 += ig * ij; X2 += g2 * ij; X3 += j2 * ig;
      if (dep[v] < 12) h0 += 1ull << (5 * dep[v]);
      else if (dep[v] < 24) h1 += 1ull << (5 * (dep[v] - 12));
      else h2 += 1ull << (5 * (dep[v] - 24));
    }
  }
  int dn = 0;                          // sum_j n_j^2
#pragma unroll
  for (int k = 0; k < 12; k++) { const int c = (int)(h0 >> (5 * k)) & 31; dn += c * c; }
#pragma unroll
  for (int k = 0; k < 12; k++) { const int c = (int)(h1 >> (5 * k)) & 31; dn += c * c; }
#pragma unroll
  for (int k = 0; k < 3; k++) { const int c = (int)(h2 >> (5 * k)) & 31; dn += c * c; }
  uint32_t kq[27];
  RB_EQMASKS_27_KEY(key, kq);
#pragma unroll
  for (int v = 0; v < 27; v++)
    if (FULL || key[v] >= 0) lg += T.log2t[RB_POPC(kq[v])];
  const double inv = FULL ? 1.0 / 27 : 1.0 / Nz, inv2 = inv * inv;
  out[0] = T.log2t[Nz] - lg * inv;                 // DependenceEntropy
  out[1] = dn * inv;                               // DependenceNonUniformity
  out[2] = dn * inv2;                              // DependenceNonUniformityNormalized
  out[3] = (double)(Nz * Sj2 - Sj * Sj) * inv2;    // DependenceVariance
  out[4] = gl * inv;                               // GrayLevelNonUniformity
  out[5] = (double)(Nz * B - C * C) * inv2;        // GrayLevelVariance
  out[6] = B * inv;                                // HighGrayLevelEmphasis
  out[7] = Sj2 * inv;                              // LargeDependenceEmphasis
  out[8] = X4 * inv;                               // LargeDependenceHighGrayLevelEmphasis
  out[9] = X3 * inv;                               // LargeDependenceLowGrayLevelEmphasis
  out[10] = A * inv;                               // LowGrayLevelEmphasis
  out[11] = Sinv * inv;                            // SmallDependenceEmphasis
  out[12] = X2 * inv;                              // SmallDependenceHighGrayLevelEmphasis
  out[13] = X1 * inv;                              // SmallDependenceLowGrayLevelEmphasis
}

// ---------------------------------------------------------------------------------------- NGTDM
// Two bodies, chosen by the window alone (so slab and whole-volume maps agree bit for bit):
//   full window (a centre whose 27 levels are all non-zero: 97.7 % of a 256^3 volume, all but the faces) -- every
//     position v has the constant neighbour count cnt_v in {7, 11, 17, 26} and Nvp = 27.  The neighbour sums are
//     separable 3x3x3 box sums, and diff_v * L = |cnt_v g_v - sum_v| * (L / cnt_v), L = lcm(7, 11, 17, 26) = 34034, is
//     an integer <= 254 L (8.6 M): class sums and sum_i s_i are exact int32, sum_i n_i s_i is an exact double, and every
//     feature is rounded only in its last few operations, independently of the summation order.
//   general window (volume faces, ROI borders, holes) -- zeros are unmasked, counts come from the mask, and
//     diff_v = |cnt_v g_v - sum_v| * (1 / cnt_v) from the rcp table.
// Both bodies add each position's diff to its class's lowest position (the representative) in per-thread shared
// scratch -- 27 fixed steps, no branch per class -- and then compact the classes in place (entry k <= position v, which
// is already read).  The Busyness denominator sum_{a<b} |i_a n_a - i_b n_b| is an integer: sorting the 27 values
// x_v = g_v n_v on the representatives (0 elsewhere) gives it as sum_k (2k - 53 + nl) x_(k), the zeros adding nothing.
// Only Complexity, with its 1 / (n_a + n_b) per pair of classes, keeps a pair loop.
constexpr int NGTDM_L = 34034;

// neighbour count of window position (z, y, x) in a full 3x3x3 window: 7 at a corner, 11 on an edge, 17 on a face, 26
RB_HD constexpr int ngtdm_full_cnt(int v) {
  return (v % 3 == 1 ? 3 : 2) * ((v / 3) % 3 == 1 ? 3 : 2) * (v / 9 == 1 ? 3 : 2) - 1;
}

// d as a double, exactly, for 0 <= d < 2^32 (on the device: one fp64 add instead of the slower int -> fp64 conversion)
RB_HD double ngtdm_i2d(int d) {
#ifdef __CUDA_ARCH__
  return __hiloint2double(0x43300000, d) - 4503599627370496.0;
#else
  return (double)d;
#endif
}

// sum_{a<b} |i_a - i_b| (n_a s_a + n_b s_b) / (n_a + n_b) over the nl compacted classes (pk = n << 8 | i, ns = n s)
RB_HD double ngtdm_complexity_pairs(const int* pk, const double* ns, int st, int nl, const SmallFastTables& T) {
  double c0 = 0, c1 = 0;
  for (int a = 0; a + 1 < nl; a++) {
    const int pa = pk[a * st], na = pa >> 8, ia = pa & 255;
    const double sa = ns[a * st];
    int b = a + 1;
    for (; b + 1 < nl; b += 2) {                // two independent chains
      const int p0 = pk[b * st], p1 = pk[(b + 1) * st];
      const int x0 = ia - (p0 & 255), x1 = ia - (p1 & 255);
      c0 += ngtdm_i2d(x0 < 0 ? -x0 : x0) * ((sa + ns[b * st]) * T.rcp[na + (p0 >> 8)]);
      c1 += ngtdm_i2d(x1 < 0 ? -x1 : x1) * ((sa + ns[(b + 1) * st]) * T.rcp[na + (p1 >> 8)]);
    }
    if (b < nl) {
      const int p0 = pk[b * st], x0 = ia - (p0 & 255);
      c0 += ngtdm_i2d(x0 < 0 ? -x0 : x0) * ((sa + ns[b * st]) * T.rcp[na + (p0 >> 8)]);
    }
  }
  return c0 + c1;
}

// general body: diff_v = |cnt_v g_v - sum_v| / cnt_v (static neighbour lists, unmasked voxels carry level 0) added to
// the class representative's entry of scr_ns
struct NgtdmGeneralDiff {
  const int* wl; const uint32_t* eq; uint32_t M; const SmallFastTables* T; double* scr_ns; int st; double ssum;
  template <int V> RB_HD void at() {
    if (!wl[V]) return;
    constexpr uint32_t nb = NB26<V>::value;
    int sum = 0;
#pragma unroll
    for (int u = 0; u < 27; u++) if (nb >> u & 1u) sum += wl[u];
    const int cnt = RB_POPC(M & nb), x = cnt * wl[V] - sum;
    const double d = ngtdm_i2d(x < 0 ? -x : x) * T->rcp[cnt];     // (cnt = 0: x = 0)
    ssum += d;
    const int r = RB_CTZ(eq[V]);
    const double prev = r == V ? 0.0 : scr_ns[r * st];
    scr_ns[r * st] = prev + d;
  }
};

// scr_pk / scr_ns: per-thread scratch of 27 entries each, element stride st (device: shared memory laid out
// [entry][thread]).  FULL: wl must be a full window (all 27 levels non-zero).
template <bool FULL>
RB_HD void ngtdm_fast_body(const int* wl, const SmallFastTables& T, double* out, int* scr_pk, double* scr_ns, int st) {
  int B = 0, C = 0;
#pragma unroll
  for (int v = 0; v < 27; v++) { B += wl[v] * wl[v]; C += wl[v]; }
  uint32_t eq[27];
  RB_EQMASKS_27(wl, eq);
  int Nvp = 27, SE = 0;                          // FULL: sum_v diff_v * L
  double ssum = 0;                               // general: sum_v diff_v
  if (FULL) {
    // box sums over the window, separably (x, then y, then z); sum_v = box_v - g_v
    int bx[27], by[27], bz[27];
#pragma unroll
    for (int r = 0; r < 27; r += 3) {
      bx[r] = wl[r] + wl[r + 1]; bx[r + 1] = bx[r] + wl[r + 2]; bx[r + 2] = wl[r + 1] + wl[r + 2];
    }
#pragma unroll
    for (int r = 0; r < 27; r += 9)
#pragma unroll
      for (int x = 0; x < 3; x++) {
        const int* b = bx + r + x;
        by[r + x] = b[0] + b[3]; by[r + 3 + x] = by[r + x] + b[6]; by[r + 6 + x] = b[3] + b[6];
      }
#pragma unroll
    for (int yx = 0; yx < 9; yx++) {
      bz[yx] = by[yx] + by[9 + yx]; bz[9 + yx] = bz[yx] + by[18 + yx]; bz[18 + yx] = by[9 + yx] + by[18 + yx];
    }
    // each position's integer diff to its class representative (rep <= v, so the representative's entry is set first)
#pragma unroll
    for (int v = 0; v < 27; v++) {
      const int cnt = ngtdm_full_cnt(v);
      const int x = (cnt + 1) * wl[v] - bz[v];
      const int e = (x < 0 ? -x : x) * (NGTDM_L / cnt);
      SE += e;
      const int r = RB_CTZ(eq[v]);
      const int prev = r == v ? 0 : scr_pk[r * st];
      scr_pk[r * st] = prev + e;
    }
  } else {
    uint32_t M = 0;
#pragma unroll
    for (int v = 0; v < 27; v++) if (wl[v]) M |= 1u << v;
    Nvp = RB_POPC(M);
    NgtdmGeneralDiff p1{wl, eq, M, &T, scr_ns, st, 0.0};
    ForPos<0, 27>::go(p1);
    ssum = p1.ssum;
  }
  // compact the classes: entry nl <= v is already read.  Non-representatives write a dead entry at nl (overwritten by
  // the next representative, or past the end).
  int nl = 0, SL = 0, SL2 = 0;
  double pw = 0;                                 // sum_i n_i s_i (FULL: times L)
  int X[27];
#pragma unroll
  for (int v = 0; v < 27; v++) {
    const bool rep = eq[v] && (eq[v] & ((1u << v) - 1)) == 0;
    const int n = RB_POPC(eq[v]), g = wl[v];
    const double ns = FULL ? ngtdm_i2d(n) * ngtdm_i2d(scr_pk[v * st]) : ngtdm_i2d(n) * scr_ns[v * st];
    scr_pk[nl * st] = n << 8 | g;
    scr_ns[nl * st] = ns;
    X[v] = rep ? g * n : 0;
    if (rep) { nl++; SL += g; SL2 += g * g; pw += ns; }
  }
  RB_NGTDM_SORT27(X);
  int bd = 0;                                    // sum_{a<b} |i_a n_a - i_b n_b|
#pragma unroll
  for (int k = 0; k < 27; k++) bd += (2 * k - 53 + nl) * X[k];
  const double cpx = ngtdm_complexity_pairs(scr_pk, scr_ns, st, nl, T);
  // u = the unit of the diffs (FULL: L); p_i = n_i / Nvp
  const double u = FULL ? (double)NGTDM_L : 1.0, N = (double)Nvp;
  const double sdiff = FULL ? (double)SE : ssum;
  out[N_Coarseness] = pw != 0 ? N * u / pw : 1e6;                         // 1 / sum_i p_i s_i
  const double div = (double)nl * (nl - 1);
  // Contrast = sum_ij p_i p_j (i-j)^2 * sum s / Nvp / (nl (nl-1)), sum_ij p_i p_j (i-j)^2 = 2 (Nvp B - C^2) / Nvp^2
  out[N_Contrast] = div != 0 ? 2.0 * (double)(Nvp * B - C * C) * sdiff / (N * N * N * u * div) : 0.0;
  out[N_Busyness] = bd != 0 ? pw / (2.0 * u * (double)bd) : 0.0;       // sum_i p_i s_i / sum_ij |i p_i - j p_j|
  out[N_Complexity] = 2.0 * cpx / (N * u);      // sum_{i != j} |i-j| (p_i s_i + p_j s_j) / (p_i + p_j) / Nvp
  // Strength = sum_ij (p_i + p_j)(i-j)^2 / sum s = (2/Nvp) (nl B - 2 C SL + Nvp SL2) / sum s
  out[N_Strength] = sdiff != 0 ? 2.0 * u * (double)(nl * B - 2 * C * SL + Nvp * SL2) / (N * sdiff) : 0.0;
}

// a window is full when all 27 levels are non-zero
RB_HD bool window27_full(const int* wl) {
  bool full = true;
#pragma unroll
  for (int v = 0; v < 27; v++) full &= wl[v] != 0;
  return full;
}

// convenience: private scratch, body chosen by the window (host emulation)
RB_HD void ngtdm_fast_voxel(const int* wl, const SmallFastTables& T, double* out) {
  int pk[27] = {0};
  double ns[27] = {0};
  if (window27_full(wl)) ngtdm_fast_body<true>(wl, T, out, pk, ns, 1);
  else ngtdm_fast_body<false>(wl, T, out, pk, ns, 1);
}

// ---------------------------------------------------------------------------------------- GLSZM
RB_HD uint32_t dilate26(uint32_t m) {
  constexpr uint32_t X0 = 0x1249249u, X2 = 0x4924924u;       // positions with x == 0 / x == 2
  constexpr uint32_t Y0 = 0x01C0E07u, Y2 = 0x70381C0u;       // y == 0 / y == 2
  m |= ((m & ~X2) << 1) | ((m & ~X0) >> 1);
  m |= ((m & ~Y2) << 3) | ((m & ~Y0) >> 3);
  m |= (m << 9) | (m >> 9);
  return m & 0x7FFFFFFu;
}

struct GlszmAcc {
  int Nz, Sg, Sg2, Ss2, X4, gln;
  double A, Sinv, X1, X2, X3, lg;
  unsigned long long h0, h1, h2;      // zone-size histogram, 5-bit fields: sizes 1..12 | 13..24 | 25..27
};

// Equality masks of the window as the other fast paths.  A level that occurs ONCE is one zone of size 1: its share of
// every sum is added in the static loop below (27 i.i.d. levels out of 32: ~12 such levels); only the levels that
// occur at least twice (<= 13 of them, ~7) go through the flood fill.  Their masks and levels live in per-thread
// scratch scr (mask | g << 32, 13 entries, element stride st; device: shared memory laid out [entry][thread]).  The
// merged (level, size) counts come from the histogram's growth inside the level: a zone that joins c earlier zones of
// its level and size adds (c+1) log2(c+1) - c log2(c) to sum_groups c log2(c).  FULL: wl must be a full window.
template <bool FULL>
RB_HD void glszm_fast_body(const int* wl, const SmallFastTables& T, double* out, unsigned long long* scr, int st) {
  uint32_t eq[27];
  if (FULL) RB_EQMASKS_27_KEY(wl, eq);
  else RB_EQMASKS_27(wl, eq);
  uint32_t M = 0;
  int nl = 0, S_n = 0, S_g = 0, S_g2 = 0;
  double S_ig = 0;
#pragma unroll
  for (int v = 0; v < 27; v++) {
    if (!FULL && wl[v]) M |= 1u << v;
    if (eq[v] && (eq[v] & ((1u << v) - 1)) == 0) {
      if (eq[v] == (1u << v)) { S_n++; S_g += wl[v]; S_g2 += wl[v] * wl[v]; S_ig += T.inv2[wl[v]]; }
      else { scr[nl * st] = eq[v] | (unsigned long long)wl[v] << 32; nl++; }
    }
  }
  GlszmAcc a;
  a.Nz = S_n; a.Sg = S_g; a.Sg2 = S_g2; a.Ss2 = S_n; a.X4 = S_g2; a.gln = S_n;
  a.A = S_ig; a.Sinv = (double)S_n; a.X1 = S_ig; a.X2 = (double)S_g2; a.X3 = S_ig; a.lg = 0;
  a.h0 = (unsigned long long)S_n; a.h1 = a.h2 = 0;
  for (int k = 0; k < nl; k++) {
    const unsigned long long e = scr[k * st];
    uint32_t m = (uint32_t)e;
    const int g = (int)(e >> 32), g2 = g * g;
    const double ig = T.inv2[g];
    const unsigned long long l0 = a.h0, l1 = a.h1, l2 = a.h2;    // the histogram before this level
    int zc = 0;                                        // <= 8 mutually non-adjacent zones fit a 3x3x3 window
    while (m) {
      uint32_t comp = m & (0u - m);
      for (;;) {
        const uint32_t nx = dilate26(comp) & m;
        if (nx == comp) break;
        comp = nx;
      }
      m &= ~comp;
      const int sz = RB_POPC(comp), s2 = sz * sz;
      zc++;
      const double is = T.invsq[sz];
      a.Nz++; a.Sg += g; a.Sg2 += g2; a.Ss2 += s2; a.X4 += g2 * s2;
      a.A += ig; a.Sinv += is; a.X1 += ig * is; a.X2 += g2 * is; a.X3 += s2 * ig;
      int c;                                           // earlier zones of this level and size
      if (sz <= 12) { c = (int)((a.h0 - l0) >> (5 * (sz - 1))) & 31; a.h0 += 1ull << (5 * (sz - 1)); }
      else if (sz <= 24) { c = (int)((a.h1 - l1) >> (5 * (sz - 13))) & 31; a.h1 += 1ull << (5 * (sz - 13)); }
      else { c = (int)((a.h2 - l2) >> (5 * (sz - 25))) & 31; a.h2 += 1ull << (5 * (sz - 25)); }
      a.lg += T.dclog2[c];
    }
    a.gln += zc * zc;
  }
  int szn = 0;
#pragma unroll
  for (int k = 0; k < 12; k++) {
    const int c0 = (int)(a.h0 >> (5 * k)) & 31, c1 = (int)(a.h1 >> (5 * k)) & 31;
    szn += c0 * c0 + c1 * c1;
  }
#pragma unroll
  for (int k = 0; k < 3; k++) { const int c2 = (int)(a.h2 >> (5 * k)) & 31; szn += c2 * c2; }
  const int Np = FULL ? 27 : RB_POPC(M), Nz = a.Nz;
  const double inv = FULL ? T.rcp[Nz] : 1.0 / Nz, inv2 = inv * inv;
  out[S_GLN] = a.gln * inv; out[S_GLNN] = a.gln * inv2;
  out[S_GLV] = (double)(Nz * a.Sg2 - a.Sg * a.Sg) * inv2;
  out[S_HGLE] = a.Sg2 * inv; out[S_LargeE] = a.Ss2 * inv; out[S_LargeHGLE] = a.X4 * inv; out[S_LargeLGLE] = a.X3 * inv;
  out[S_LGLE] = a.A * inv; out[S_SizeNU] = szn * inv; out[S_SizeNUN] = szn * inv2; out[S_SmallE] = a.Sinv * inv;
  out[S_SmallHGLE] = a.X2 * inv; out[S_SmallLGLE] = a.X1 * inv;
  out[S_Entropy] = T.log2t[Nz] - a.lg * inv;
  out[S_Percentage] = FULL ? Nz * (1.0 / 27) : (double)Nz / Np;
  out[S_SizeVar] = (double)(Nz * a.Ss2 - Np * Np) * inv2;
}

// convenience: private scratch, body chosen by the window (host emulation)
RB_HD void glszm_fast_voxel(const int* wl, const SmallFastTables& T, double* out) {
  unsigned long long scr[13];
  if (window27_full(wl)) glszm_fast_body<true>(wl, T, out, scr, 1);
  else glszm_fast_body<false>(wl, T, out, scr, 1);
}
RB_HD void gldm_fast_voxel(const int* wl, int alpha, const SmallFastTables& T, double* out) {
  if (window27_full(wl)) gldm_fast_body<true>(wl, alpha, T, out);
  else gldm_fast_body<false>(wl, alpha, T, out);
}

}  // namespace rb
