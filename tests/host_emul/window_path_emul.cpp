// TEST-ONLY: the rule that sends a voxel window to the generic or the wide kernels (host_common.hpp window_path), and
// the window sizes fill_vox_params gives, compiled with g++ so the rule is checked without a GPU.
#include "../../pyradiomics_b200/csrc/host_common.hpp"

using namespace rb;

extern "C" int emul_window_path(int cap, int force_wide) { return (int)window_path(cap, force_wide != 0); }

// window positions of class cls's launch on a (Z, Y, X) volume, or a negative fill_vox_params error
extern "C" int emul_window_positions(int cls, int Z, int Y, int X, const VoxSettings* s) {
  VoxParams* P = new VoxParams;
  const int rc = fill_vox_params(cls, Z, Y, X, *s, *P);
  const int n = rc ? rc : window_capacity(*P);
  delete P;
  return n;
}
