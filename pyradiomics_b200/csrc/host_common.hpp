// Host-side helpers shared by the C-ABI (capi.cu) and the test-only host emulation:
// neighbour-offset ("angle") enumeration, the per-launch parameter block and the rule that picks each voxel kernel.
#pragma once
#include <math.h>
#include <string.h>

#include <vector>

#include "../../include/b200radiomics.h"
#include "vox_features.cuh"

namespace rb {

// Enumerate neighbour offsets exactly in the reference's order (reference
// radiomics/src/cmatrices.c:756-892, get_angle_count + build_angles): components run from
// +maxdist down to -maxdist, dimension 0 slowest; an offset is kept when its Chebyshev norm is a
// requested distance, |component| < size in every dimension and it does not leave the force2D
// plane.  The list is point-symmetric, so "unidirectional" is its first half.
// Returns the offsets as (dz,dy,dx) rows for nd == 3 and (dy,dx) rows for nd == 2.
inline int generate_angles(const int* size, int nd, const int* distances, int ndist, bool bidirectional,
                           int force2Ddim /* -1 = off */, std::vector<int>& out) {
  out.clear();
  if (nd < 1 || nd > 3) return -1;
  int D = 0;
  for (int i = 0; i < ndist; i++) { if (distances[i] < 1) return 0; if (distances[i] > D) D = distances[i]; }
  std::vector<int> all;
  int off[3] = {0, 0, 0};
  long long total = 1;
  for (int d = 0; d < nd; d++) total *= (2 * D + 1);
  for (long long c = 0; c < total; c++) {
    long long r = c;
    for (int d = nd - 1; d >= 0; d--) { off[d] = D - (int)(r % (2 * D + 1)); r /= (2 * D + 1); }
    int norm = 0; bool ok = true;
    for (int d = 0; d < nd; d++) {
      int a = off[d] < 0 ? -off[d] : off[d];
      if (a >= size[d] || (d == force2Ddim && a != 0)) ok = false;
      if (a > norm) norm = a;
    }
    if (!ok || norm == 0) continue;
    bool wanted = false;
    for (int i = 0; i < ndist; i++) if (distances[i] == norm) wanted = true;
    if (!wanted) continue;
    for (int d = 0; d < nd; d++) all.push_back(off[d]);
  }
  int na = (int)(all.size() / nd);
  if (!bidirectional) na /= 2;
  out.assign(all.begin(), all.begin() + (size_t)na * nd);
  return na;
}

// Up to NA_MAX (dz, dy, dx) offsets, passed to the matrix kernels by value
struct AngleSet {
  int na;
  int8_t a[NA_MAX][3];
};

// The front end every segment-mode builder starts from (segment_geometry, segment_kernels.cu): the volume as Z x Y x X
// (a 2-D image is one plane) and its offsets as (dz, dy, dx) rows.
struct SegmentGeometry {
  int Z, Y, X;
  long long n;   // Z * Y * X, 1..2^31-1
  AngleSet A;
  int H;         // largest |offset component|
};
// Checks Ng (1..65535), the voxel count and the offset count (at most na_max; "more than NA_MAX angles" counts both
// directions); angles_out (may be NULL) receives the offsets as the reference returns them, Na x nd.
int segment_geometry(const int* size, int nd, const int* distances, int ndist, bool bidirectional, int force2D,
                     int force2Ddimension, int Ng, int na_max, int* angles_out, SegmentGeometry& G);

enum Weighting { W_NONE = 0, W_INFINITY = 1, W_EUCLIDEAN = 2, W_MANHATTAN = 3, W_NO_WEIGHTING = 4 };
enum TexClass { C_GLCM = 0, C_GLRLM = 1, C_GLSZM = 2, C_GLDM = 3, C_NGTDM = 4 };
static const int kNumFeatures[5] = {GLCM_NF, GLRLM_NF, GLSZM_NF, GLDM_NF, NGTDM_NF};

// per-angle weight (reference radiomics/glcm.py:160-181 -> exp(-d^2); glrlm.py:130-150 -> d)
inline double angle_weight(const int* a3, const double* spacing_zyx, int weighting, bool glcm) {
  double v[3];
  for (int d = 0; d < 3; d++) v[d] = fabs((double)a3[d]) * spacing_zyx[d];
  double dist;
  switch (weighting) {
    case W_INFINITY: dist = fmax(v[0], fmax(v[1], v[2])); break;
    case W_EUCLIDEAN: dist = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); break;
    case W_MANHATTAN: dist = v[0] + v[1] + v[2]; break;
    default: return 1.0;
  }
  return glcm ? exp(-dist * dist) : dist;
}

using VoxSettings = rb_voxel_settings;

// Build the launch parameter block of one class for a (Z,Y,X) volume.  Returns 0 or a negative
// error (-3 bad argument / unsupported size).
inline int fill_vox_params(int cls, int Z, int Y, int X, const VoxSettings& s, VoxParams& P) {
  memset(&P, 0, sizeof(P));
  P.Z = Z; P.Y = Y; P.X = X; P.sy = X; P.sz = (long long)X * Y;
  int f2 = s.force2D ? s.force2Ddimension : -1;
  int r = s.kernelRadius;
  if (r < 1) return -3;
  P.rz = f2 == 0 ? 0 : r; P.ry = f2 == 1 ? 0 : r; P.rx = f2 == 2 ? 0 : r;
  int size[3] = {Z, Y, X};
  int one[1] = {1};
  const int* dist = s.distances; int nd = s.ndist; bool bidir = true;
  if (cls == C_GLCM) bidir = false;
  if (cls == C_GLRLM) { bidir = false; dist = one; nd = 1; }
  if (cls == C_GLSZM) { dist = one; nd = 1; }
  std::vector<int> ang;
  int na = generate_angles(size, 3, dist, nd, bidir, f2, ang);
  if (na <= 0 || na > NA_MAX || (!bidir && na > NW_MAX)) return -3;
  P.na = na;
  for (int a = 0; a < na; a++) for (int d = 0; d < 3; d++) P.ang[a][d] = (int8_t)ang[a * 3 + d];
  P.symmetric = s.symmetricalGLCM; P.alpha = s.gldm_a; P.Ng = s.Ng; P.n_roi_levels = s.n_roi_levels;
  P.init_value = s.initValue;
  P.weighted = (s.weighting != W_NONE && (cls == C_GLCM || cls == C_GLRLM)) ? 1 : 0;
  if (P.weighted)
    for (int a = 0; a < na; a++) P.wgt[a] = angle_weight(&ang[a * 3], s.spacing_zyx, s.weighting, cls == C_GLCM);
  for (int a = 0; a < na && a < NW_MAX; a++) P.alive[a >> 5] |= 1u << (a & 31);
  return 0;
}

inline int window_capacity(const VoxParams& P) { return (2 * P.rz + 1) * (2 * P.ry + 1) * (2 * P.rx + 1); }

// The generic kernels' window classes: a window of `positions` runs in the 27-, 125- or 343-position instantiation
// (kernelRadius 1, 2, 3 in 3-D), and its entry lists are sized by that class; the wide kernels size theirs for
// WIDE_WCAP_MAX above 343 positions.
constexpr int GENERIC_WCAP_MAX = 343, WIDE_WCAP_MAX = 3375;
constexpr int window_class(int positions) {
  return positions <= 27 ? 27 : positions <= 125 ? 125 : positions <= GENERIC_WCAP_MAX ? GENERIC_WCAP_MAX : WIDE_WCAP_MAX;
}

// Which kernel a voxel-map launch runs on, texture and first order alike: the r = 1 fast kernel when it fits
// (fast_fits: voxel_fast_path / firstorder_fast_path below), else the thread-per-centre generic kernels up to 7^3 = 343
// positions, the block-per-centre wide kernels (voxel_wide.cu, firstorder.cu) up to 15^3 = 3375 (kernelRadius 4 to 7 in
// 3-D; larger force2D / 2-D windows), nothing beyond.  Two overrides, for tests: force_wide
// (B200_RADIOMICS_FORCE_WIDE=1) sends every window, fast and generic ones included, to the wide kernels; force_generic
// (B200_RADIOMICS_FORCE_GENERIC=1) declines the fast kernel.  The host emulation (tests/host_emul) returns the values
// as they are, and runs the generic path, so it stops at WP_WIDE.
enum WindowPath { WP_GENERIC, WP_WIDE, WP_UNSUPPORTED, WP_FAST };
inline WindowPath window_path(int positions, bool force_wide, bool fast_fits = false, bool force_generic = false) {
  if (fast_fits && !force_generic && !force_wide) return WP_FAST;
  if (positions > WIDE_WCAP_MAX) return WP_UNSUPPORTED;
  return positions > GENERIC_WCAP_MAX || force_wide ? WP_WIDE : WP_GENERIC;
}

// Whether texture class cls runs its kernelRadius-1 fast kernel (voxel_fast_launch) rather than the generic one: 8-bit
// levels and a 3x3x3 window, plus the angle set and weighting the class's fast body is written for.  The host
// emulation takes the same decision.
inline bool voxel_fast_path(int cls, int level_bytes, const VoxParams& P) {
  if (level_bytes != 1 || P.rz != 1 || P.ry != 1 || P.rx != 1 || P.Ng > 255) return false;
  switch (cls) {
    case C_GLCM: return P.na == 13 && P.symmetric && !P.weighted;
    case C_GLRLM: return P.na == 13 && !P.weighted;
    case C_GLSZM: case C_GLDM: case C_NGTDM: return P.na == 26;
    default: return false;
  }
}

// the same for the first-order maps (firstorder_fast_launch): 8-bit levels and a 3x3x3 window
inline bool firstorder_fast_path(int level_bytes, int rz, int ry, int rx) {
  return level_bytes == 1 && rz == 1 && ry == 1 && rx == 1;
}

}  // namespace rb
