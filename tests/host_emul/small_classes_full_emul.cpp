// TEST-ONLY: the GLSZM and GLDM fast paths' full-window and general bodies and the generic per-voxel math
// compiled with g++, so that tests/test_small_classes_full_window_emul.py can run all three on the same window without
// a GPU.
#include <stdint.h>
#include <string.h>

#include "../../pyradiomics_b200/csrc/host_common.hpp"
#include "../../pyradiomics_b200/csrc/small_fast.cuh"

using namespace rb;

// one 3x3x3 window (z, y, x order) of class cls (C_GLSZM or C_GLDM) through body 0 = general fast body, 1 =
// full-window fast body (the window must be full), 2 = generic per-voxel math; out in feature order.  Returns 0, or
// < 0 on bad arguments.
extern "C" int emul_small_class_window(int cls, const uint8_t* w27, int body, const VoxSettings* s, double* out) {
  if (cls != C_GLSZM && cls != C_GLDM) return -1;
  VoxParams P;
  if (fill_vox_params(cls, 3, 3, 3, *s, P)) return -1;
  if (P.na != 26 || P.rz != 1 || P.ry != 1 || P.rx != 1 || s->Ng > 255) return -5;
  int wl[27];
  bool full = true;
  for (int p = 0; p < 27; p++) { wl[p] = w27[p]; full &= w27[p] != 0; }
  if (body == 2) {
    uint16_t lev[27], w[27];
    for (int p = 0; p < 27; p++) lev[p] = w27[p];
    load_window<uint16_t>(lev, P, 1, 1, 1, w);
    if (cls == C_GLSZM) glszm_voxel<27>(w, P, out);
    else gldm_voxel<27>(w, P, out);
    return 0;
  }
  if (body == 1 && !full) return -2;
  // scratch with a stride and stale contents, as a thread's shared-memory columns have on the device
  unsigned long long mg[13 * 3];
  for (int k = 0; k < 13 * 3; k++) mg[k] = 0x5a5a5a5a5a5a5a5aull - k;
  SmallFastTables* T = new SmallFastTables;
  small_fast_build_tables(*T);
  if (cls == C_GLSZM) {
    if (body == 1) glszm_fast_body<true>(wl, *T, out, mg + 1, 3);
    else glszm_fast_body<false>(wl, *T, out, mg + 1, 3);
  } else {
    if (body == 1) gldm_fast_body<true>(wl, P.alpha, *T, out);
    else gldm_fast_body<false>(wl, P.alpha, *T, out);
  }
  delete T;
  return 0;
}
