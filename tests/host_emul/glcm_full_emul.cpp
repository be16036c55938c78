// TEST-ONLY: GLCM phase A's full-window body and its general body compiled with g++, so that
// tests/test_glcm_full_window_emul.py can run both on the same window and compare them without a GPU.
#include <stdint.h>
#include <string.h>

#include "../../pyradiomics_b200/csrc/host_common.hpp"
#include "../../pyradiomics_b200/csrc/glcm_fast.cuh"

using namespace rb;

static int params(const VoxSettings* s, VoxParams& P) {
  if (fill_vox_params(C_GLCM, 3, 3, 3, *s, P)) return -1;
  if (P.na != 13 || P.rz != 1 || P.ry != 1 || P.rx != 1 || !P.symmetric || P.weighted || s->Ng > 255) return -5;
  return 0;
}

// one angle slot of one window through glcm_fast_angle<NP, FULL>: sums[24] (that angle's feature values), the task bit and
// task size class.  Returns the task bitmask, or < 0 on bad arguments.
extern "C" long long emul_glcm_angle(const uint8_t* w27, int slot, int full, const VoxSettings* s, double* sums,
                                     unsigned long long* tcls) {
  VoxParams P;
  if (params(s, P) || slot < 0 || slot >= GF_NA) return -1;
  GlcmFastTables* T = new GlcmFastTables;
  glcm_fast_build_tables(*T, s->Ng);
  int wl[27];
  uint32_t eq[27];
  for (int p = 0; p < 27; p++) wl[p] = w27[p];
  RB_EQMASKS_27(wl, eq);
  GlcmAcc acc;
  memset(&acc, 0, sizeof acc);
  const int np = T->np[slot];
  if (full) {
    if (np == 18) glcm_fast_angle<18, true>(w27, 1, eq, 1, *T, slot, P, acc);
    else if (np == 12) glcm_fast_angle<12, true>(w27, 1, eq, 1, *T, slot, P, acc);
    else glcm_fast_angle<8, true>(w27, 1, eq, 1, *T, slot, P, acc);
  } else {
    if (np == 18) glcm_fast_angle<18, false>(w27, 1, eq, 1, *T, slot, P, acc);
    else if (np == 12) glcm_fast_angle<12, false>(w27, 1, eq, 1, *T, slot, P, acc);
    else glcm_fast_angle<8, false>(w27, 1, eq, 1, *T, slot, P, acc);
  }
  for (int k = 0; k < GLCM_NF; k++) sums[k] = acc.sum[k];
  *tcls = acc.tcls;
  delete T;
  return acc.tasks;
}

// phase A of one window through glcm_fast_voxel_phaseA<FULL>: out[24], n_ok and the task size classes; returns the
// task bitmask, or < 0 on bad arguments
extern "C" long long emul_glcm_phaseA(const uint8_t* w27, int full, const VoxSettings* s, double* out, int* n_ok,
                                      unsigned long long* tcls) {
  VoxParams P;
  if (params(s, P)) return -1;
  GlcmFastTables* T = new GlcmFastTables;
  glcm_fast_build_tables(*T, s->Ng);
  uint32_t eq[27];
  const uint32_t tasks = full ? glcm_fast_voxel_phaseA<true>(w27, 1, eq, 1, *T, P, out, n_ok, tcls)
                              : glcm_fast_voxel_phaseA<false>(w27, 1, eq, 1, *T, P, out, n_ok, tcls);
  delete T;
  return tasks;
}
