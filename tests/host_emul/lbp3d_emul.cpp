// Host build of the 3-D LBP per-voxel arithmetic (pyradiomics_b200/csrc/lbp3d.cuh) for tests/test_lbp3d_cpu.py:
// the same lbp3d_voxel the CUDA kernel runs, over a list of voxels, with the B-spline coefficients supplied by the caller.
#include <stdlib.h>

#include "../../pyradiomics_b200/csrc/lbp3d.cuh"

extern "C" int lbp3d_emul(const double* coef, const void* img, int img_dt, int sample_dt, int Z, int Y, int X,
                          const long long* coords, long long np, const double* verts, int nv, const double* harm, int levels,
                          double* out) {
  if (nv > rb::LBP_MAX_NV || levels > rb::LBP_MAX_LEVELS) return -5;
  rb::Lbp3dTables* T = (rb::Lbp3dTables*)calloc(1, sizeof(rb::Lbp3dTables));
  T->nv = nv;
  T->levels = levels;
  T->sample_dt = sample_dt;
  const int kp = levels * (levels + 1) / 2;
  for (int v = 0; v < nv; v++) {
    for (int d = 0; d < 3; d++) T->vert[v][d] = verts[v * 3 + d];
    for (int k = 0; k < kp; k++) {
      T->y_re[v][k] = harm[(v * kp + k) * 2];
      T->y_im[v][k] = harm[(v * kp + k) * 2 + 1];
    }
  }
  for (long long i = 0; i < np; i++)
    rb::lbp3d_voxel(coef, img, img_dt, Z, Y, X, (int)coords[i], (int)coords[np + i], (int)coords[2 * np + i], *T, out + i, np);
  free(T);
  return 0;
}
