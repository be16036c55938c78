// TEST-ONLY: compiles the __host__ __device__ per-voxel feature math of
// pyradiomics_b200/csrc/vox_features.cuh with g++ so the arithmetic can be checked against the
// oracle on machines without a GPU.  Not part of the product (which has no CPU path).
#include <stdint.h>
#include <stdlib.h>

#include "../../pyradiomics_b200/csrc/host_common.hpp"
#include "../../pyradiomics_b200/csrc/glcm_fast.cuh"

using namespace rb;

template <int WCAP>
static void run(int cls, const uint16_t* lev, const uint8_t* centers, const VoxParams& P, double* out, int* status) {
  const int nf = kNumFeatures[cls];
  const long long nvox = (long long)P.Z * P.Y * P.X;
  for (int z = 0; z < P.Z; z++) for (int y = 0; y < P.Y; y++) for (int x = 0; x < P.X; x++) {
    long long i = ((long long)z * P.Y + y) * P.X + x;
    bool c = centers ? centers[i] != 0 : lev[i] != 0;
    if (!c) { for (int k = 0; k < nf; k++) out[k * nvox + i] = P.init_value; continue; }
    uint16_t w[WCAP]; double f[32];
    load_window<uint16_t>(lev, P, z, y, x, w);
    switch (cls) {
      case C_GLCM: if (P.weighted) glcm_voxel<WCAP, true>(w, P, f, status); else glcm_voxel<WCAP, false>(w, P, f, status); break;
      case C_GLRLM: if (P.weighted) glrlm_voxel<WCAP, true>(w, P, f); else glrlm_voxel<WCAP, false>(w, P, f); break;
      case C_GLSZM: glszm_voxel<WCAP>(w, P, f); break;
      case C_GLDM: gldm_voxel<WCAP>(w, P, f); break;
      case C_NGTDM: ngtdm_voxel<WCAP>(w, P, f); break;
    }
    for (int k = 0; k < nf; k++) out[k * nvox + i] = f[k];
  }
}

extern "C" int emul_voxel_features(int cls, const uint16_t* lev, const uint8_t* centers, int Z, int Y, int X,
                                   const VoxSettings* s, const uint32_t* alive, double* out) {
  VoxParams P;
  int rc = fill_vox_params(cls, Z, Y, X, *s, P);
  if (rc) return rc;
  if (alive) for (int k = 0; k < (NW_MAX + 31) / 32; k++) P.alive[k] = alive[k];
  int status = 0;
  int cap = window_capacity(P);
  if (cap <= 27) run<27>(cls, lev, centers, P, out, &status);
  else if (cap <= 125) run<125>(cls, lev, centers, P, out, &status);
  else if (cap <= 343) run<343>(cls, lev, centers, P, out, &status);
  else return -5;
  return status;
}

#include "../../pyradiomics_b200/csrc/glrlm_fast.cuh"
// MCC eigen-task of one 27-voxel window and angle slot through the dispatcher (dense register solve up to 12 levels,
// register Lanczos above); cls < 0: derive it
extern "C" double emul_glcm_solve_window_cls(const uint8_t* w, int slot, int Ng, int cls) {
  GlcmFastTables* T = new GlcmFastTables;
  glcm_fast_build_tables(*T, Ng);
  GlcmSolveTables ST;
  glcm_solve_tables_from(*T, ST);
  if (cls < 0) {
    bool seen[256] = {false}; int n = 0;
    for (int t = 0; t < ST.np[slot]; t++) {
      const uint8_t a = w[ST.pA[slot][t]], b = w[ST.pB[slot][t]];
      if (!a || !b) continue;
      if (!seen[a]) { seen[a] = true; n++; }
      if (!seen[b]) { seen[b] = true; n++; }
    }
    cls = glcm_task_class(n);
  }
  double r = glcm_fast_solve(w, 1, ST, slot, cls);
  delete T;
  return r;
}

#include "../../pyradiomics_b200/csrc/small_fast.cuh"
// The kernelRadius-1 fast path of class cls on the host: -5 when voxel_fast_path sends these settings to the generic
// kernels, else every centre (non-zero level) through the class's per-voxel fast math.  alive: GLCM's alive angles
// (NULL: all).
extern "C" int emul_fast(int cls, const uint16_t* lev, int Z, int Y, int X, const VoxSettings* s, const uint32_t* alive,
                         double* out) {
  VoxParams P;
  int rc = fill_vox_params(cls, Z, Y, X, *s, P);
  if (rc) return rc;
  if (alive) for (int k = 0; k < (NW_MAX + 31) / 32; k++) P.alive[k] = alive[k];
  if (!voxel_fast_path(cls, s->Ng <= 255 ? 1 : 2, P)) return -5;     // the level width rb_level_bytes picks
  GlcmFastTables* TC = cls == C_GLCM ? new GlcmFastTables : nullptr;
  GlrlmFastTables* TR = cls == C_GLRLM ? new GlrlmFastTables : nullptr;
  SmallFastTables* TS = cls >= C_GLSZM ? new SmallFastTables : nullptr;
  if (TC) glcm_fast_build_tables(*TC, s->Ng);
  if (TR) glrlm_fast_build_tables(*TR);
  if (TS) small_fast_build_tables(*TS);
  const int nf = kNumFeatures[cls];
  const long long nvox = (long long)Z * Y * X;
  for (int z = 0; z < Z; z++) for (int y = 0; y < Y; y++) for (int x = 0; x < X; x++) {
    long long i = ((long long)z * Y + y) * X + x;
    if (!lev[i]) { for (int k = 0; k < nf; k++) out[k * nvox + i] = P.init_value; continue; }
    uint16_t w16[27]; uint8_t w8[27]; uint32_t eq[27]; int wl[27]; double f[32];
    load_window<uint16_t>(lev, P, z, y, x, w16);
    for (int k = 0; k < 27; k++) { w8[k] = (uint8_t)w16[k]; wl[k] = w16[k]; }
    switch (cls) {
      case C_GLCM: glcm_fast_voxel(w8, 1, eq, 1, *TC, P, f); break;
      case C_GLRLM: glrlm_fast_voxel(wl, *TR, f); break;
      case C_GLSZM: glszm_fast_voxel(wl, *TS, f); break;
      case C_GLDM: gldm_fast_voxel(wl, P.alpha, *TS, f); break;
      case C_NGTDM: ngtdm_fast_voxel(wl, *TS, f); break;
    }
    for (int k = 0; k < nf; k++) out[k * nvox + i] = f[k];
  }
  delete TC; delete TR; delete TS;
  return 0;
}

#include "../../pyradiomics_b200/csrc/firstorder.cuh"
// first-order window statistics on the host: img (double), mask (window membership), lev (levels)
extern "C" int emul_firstorder(const double* img, const uint8_t* mask, const uint16_t* lev, int Z, int Y, int X, int rz,
                               int ry, int rx, double shift, double vv, double* out) {
  const long long nvox = (long long)Z * Y * X;
  for (int z = 0; z < Z; z++) for (int y = 0; y < Y; y++) for (int x = 0; x < X; x++) {
    long long i = ((long long)z * Y + y) * X + x;
    if (!mask[i]) { for (int k = 0; k < FIRSTORDER_NF; k++) out[k * nvox + i] = 0; continue; }
    double xs[343]; uint16_t w[343]; int n = 0, wn = 0; double f[FIRSTORDER_NF];
    for (int dz = -rz; dz <= rz; dz++) for (int dy = -ry; dy <= ry; dy++) for (int dx = -rx; dx <= rx; dx++, wn++) {
      int zz = z + dz, yy = y + dy, xx = x + dx;
      w[wn] = 0;
      if (zz < 0 || zz >= Z || yy < 0 || yy >= Y || xx < 0 || xx >= X) continue;
      long long j = ((long long)zz * Y + yy) * X + xx;
      if (!mask[j]) continue;
      xs[n++] = img[j]; w[wn] = lev[j];
    }
    firstorder_voxel<343>(xs, n, w, wn, shift, vv, f);
    for (int k = 0; k < FIRSTORDER_NF; k++) out[k * nvox + i] = f[k];
  }
  return 0;
}

#include "../../pyradiomics_b200/csrc/glcm_lanczos.cuh"
// register Lanczos solver of the large axis-angle eigen-tasks: w27 = window levels with the angle axis fastest;
// scratch laid out like the device's shared memory ([node][thread], stride st, this thread = lane)
extern "C" double emul_glcm_lanczos_axis(const uint8_t* w27, int N, int st, int lane, int* n_out) {
  GlcmFastTables* T = new GlcmFastTables;
  glcm_fast_build_tables(*T, 32);
  GlcmSolveTables ST;
  glcm_solve_tables_from(*T, ST);
  int wl[27];
  for (int i = 0; i < 27; i++) wl[i] = w27[i];
  double* sm = new double[(size_t)LZ_NARR * 18 * st];
  for (int i = 0; i < LZ_NARR * 18 * st; i++) sm[i] = 1e300;      // poison: a wrong stride shows
  double r = NAN;
  if (N == 14) r = glcm_lanczos_axis<14>(wl, ST, sm + lane, st, n_out);
  else if (N == 16) r = glcm_lanczos_axis<16>(wl, ST, sm + lane, st, n_out);
  else if (N == 18) r = glcm_lanczos_axis<18>(wl, ST, sm + lane, st, n_out);
  delete[] sm;
  delete T;
  return r;
}
// connectivity + bipartite sweep of phase A in position space; returns 2*connected + bipartite (eq masks from the straight-line compare block)
extern "C" int emul_glcm_graph_scan(const uint8_t* w27, int dsh, uint32_t lo_mask, int selfpair) {
  int wl[27]; uint32_t e[27];
  for (int i = 0; i < 27; i++) wl[i] = w27[i];
  RB_EQMASKS_27(wl, e);
  uint32_t NZ = 0;
  for (int i = 0; i < 27; i++) if (wl[i]) NZ |= 1u << i;
  const uint32_t EA = NZ & (NZ >> dsh) & lo_mask;
  if (!EA) return -1;
  bool connected = false, bipartite = false;
  glcm_graph_scan(e, 1, EA, dsh, EA | (EA << dsh), selfpair != 0, &connected, &bipartite);
  return (connected ? 2 : 0) | (bipartite ? 1 : 0);
}

// MCC of ONE GLCM given as a dense n x n matrix of counts or weights (rows / columns = levels 1..n) through
// glcm_angle_features, the generic kernel's per-angle math (entry list of 2048, 343 levels, the 32-row dense solve);
// *status receives its status bits (bit 0: over the dense solve's capacity)
extern "C" double emul_glcm_matrix_mcc(const double* M, int n, int symmetric, int* status) {
  if (n < 1 || n > 343) return NAN;
  Entries<2048, double>* E = new Entries<2048, double>;
  E->clear();
  for (int i = 0; i < n; i++)
    for (int j = 0; j < n; j++)
      if (M[i * n + j] != 0) E->add(((uint32_t)i << 16) | (uint32_t)j, M[i * n + j]);
  VoxParams* P = new VoxParams;
  memset(P, 0, sizeof(*P));
  P->Ng = n; P->n_roi_levels = n < 2 ? 2 : n; P->symmetric = symmetric;
  int val[343];
  for (int k = 0; k < n; k++) val[k] = k + 1;
  double f[GLCM_NF];
  int st = 0;
  const bool ok = glcm_angle_features<2048, 343, 32, double>(*E, n, val, *P, f, &st);
  if (status) *status = st;
  delete E;
  delete P;
  return ok ? f[G_MCC] : NAN;
}
