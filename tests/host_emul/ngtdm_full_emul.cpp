// TEST-ONLY: the NGTDM fast path's full-window body, its general body and the generic per-voxel math compiled with
// g++, so that tests/test_ngtdm_full_window_emul.py can run all three on the same window without a GPU.
#include <stdint.h>
#include <string.h>

#include "../../pyradiomics_b200/csrc/host_common.hpp"
#include "../../pyradiomics_b200/csrc/small_fast.cuh"

using namespace rb;

// one 3x3x3 window (z, y, x order) through body 0 = general fast body, 1 = full-window fast body (the window must be
// full), 2 = generic ngtdm_voxel; out[5] in feature order.  Returns 0, or < 0 on bad arguments.
extern "C" int emul_ngtdm_window(const uint8_t* w27, int body, const VoxSettings* s, double* out) {
  VoxParams P;
  if (fill_vox_params(C_NGTDM, 3, 3, 3, *s, P)) return -1;
  if (!voxel_fast_path(C_NGTDM, 1, P)) return -5;
  int wl[27];
  bool full = true;
  for (int p = 0; p < 27; p++) { wl[p] = w27[p]; full &= w27[p] != 0; }
  if (body == 2) {
    uint16_t lev[27], w[27];
    for (int p = 0; p < 27; p++) lev[p] = w27[p];
    load_window<uint16_t>(lev, P, 1, 1, 1, w);
    ngtdm_voxel<27>(w, P, out);
    return 0;
  }
  if (body == 1 && !full) return -2;
  SmallFastTables* T = new SmallFastTables;
  small_fast_build_tables(*T);
  // scratch with a stride and stale contents, as a thread's shared-memory columns have on the device
  int pk[27 * 3];
  double ns[27 * 3];
  for (int k = 0; k < 27 * 3; k++) { pk[k] = 0x5a5a5a5a - k; ns[k] = -1e300; }
  if (body == 1) ngtdm_fast_body<true>(wl, *T, out, pk + 1, ns + 1, 3);
  else ngtdm_fast_body<false>(wl, *T, out, pk + 1, ns + 1, 3);
  delete T;
  return 0;
}
