// TEST-ONLY: the first-order full-window body and the generic per-voxel math (firstorder_voxel<27>) compiled with g++
// from the same header, so that tests/test_firstorder_full_window_emul.py can run both on the same window without a GPU.
#include <stdint.h>

#include "../../pyradiomics_b200/csrc/firstorder.cuh"

using namespace rb;

// one full 3x3x3 window (z, y, x order: 27 intensities, none NaN, and 27 non-zero levels) through body 0 = generic
// firstorder_voxel<27>, 1 = firstorder_full_body; out[18] in feature order.  Returns 0, or < 0 if the window is not full.
extern "C" int emul_firstorder_window(const double* x27, const uint16_t* w27, int body, double shift, double vv,
                                      double* out) {
  for (int p = 0; p < 27; p++)
    if (!w27[p] || x27[p] != x27[p]) return -1;
  if (body == 0) {
    double xs[27];
    for (int p = 0; p < 27; p++) xs[p] = x27[p];
    firstorder_voxel<27>(xs, 27, w27, 27, shift, vv, out);
    return 0;
  }
  // scratch with a stride and stale contents, as a thread's shared-memory column has on the device
  double scr[27 * 3];
  for (int k = 0; k < 27 * 3; k++) scr[k] = -1e300 - k;
  firstorder_full_body(x27, w27, shift, vv, scr + 2, 3, out);
  return 0;
}
