// 3-D local binary pattern image type (reference radiomics/imageoperations.py:1169-1314, getLBP3DImage).
//   lbp3d_to_f64_kernel   the image as float64, the input of the B-spline prefilter
//   (resample.cu)         bspline_prefilter_launch(exact_init = true): SciPy's spline_filter coefficients, mirror
//                         boundaries with the closed-form causal initialisation for every line length
//   lbp3d_kernel          one thread per voxel (x fastest, grid-stride): ROI voxels run lbp3d_voxel (lbp3d.cuh) over the
//                         Nv sphere samples, every other voxel gets 0 in all L + 1 maps.  Nothing per vertex is stored
//                         beyond the thread's own Nv samples (the reference materialises (Nv, Np, 3) float64 and
//                         (Np, Nv, K) complex128 arrays).
#include "common.cuh"
#include "lbp3d.cuh"

namespace rb {

int bspline_prefilter_launch(double* coeffs, int Z, int Y, int X, cudaStream_t st, bool exact_init);

__global__ void __launch_bounds__(256) lbp3d_to_f64_kernel(const void* __restrict__ img, int dt, long long n, double* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = load_f64(img, dt, i);
}

__global__ void __launch_bounds__(128)
lbp3d_kernel(const double* __restrict__ coef, const void* __restrict__ img, int img_dt, const uint8_t* __restrict__ roi, int Z,
             int Y, int X, const __grid_constant__ Lbp3dTables T, double* __restrict__ out) {
  const long long n = (long long)Z * Y * X, plane = (long long)Y * X;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    if (!roi[t]) {
      for (int l = 0; l <= T.levels; l++) out[l * n + t] = 0.0;
      continue;
    }
    const int z = (int)(t / plane), rem = (int)(t % plane), y = rem / X, x = rem % X;
    lbp3d_voxel(coef, img, img_dt, Z, Y, X, z, y, x, T, out + t, n);
  }
}

int lbp3d_launch(const void* img, int img_dt, int sample_dt, const uint8_t* roi, int Z, int Y, int X, const double* vertices,
                 int nv, const double* harmonics, int levels, double* coeff_scratch, double* out, cudaStream_t st) {
  if (!img || !roi || !vertices || !harmonics || !coeff_scratch || !out) return fail(RB_ERR_ARG, "lbp3d: null argument");
  if (Z < 1 || Y < 1 || X < 1 || nv < 1 || levels < 1) return fail(RB_ERR_ARG, "lbp3d: empty volume, sphere or level list");
  if (nv > LBP_MAX_NV || levels > LBP_MAX_LEVELS)
    return fail(RB_ERR_UNSUPPORTED, "lbp3d: %d vertices / %d levels (at most %d, icosphere subdivision 2, and %d)", nv, levels,
                LBP_MAX_NV, LBP_MAX_LEVELS);
  static_assert(sizeof(Lbp3dTables) < 32000, "kernel parameter space");
  Lbp3dTables T;
  T.nv = nv;
  T.levels = levels;
  T.sample_dt = sample_dt;
  T.pad_ = 0;
  const int kp = levels * (levels + 1) / 2;
  for (int v = 0; v < nv; v++) {
    for (int d = 0; d < 3; d++) T.vert[v][d] = vertices[v * 3 + d];
    for (int k = 0; k < kp; k++) {
      T.y_re[v][k] = harmonics[(v * kp + k) * 2];
      T.y_im[v][k] = harmonics[(v * kp + k) * 2 + 1];
    }
  }
  const long long n = (long long)Z * Y * X;
  lbp3d_to_f64_kernel<<<grid_for(n, 256, 8), 256, 0, st>>>(img, img_dt, n, coeff_scratch);
  RB_LAUNCH_CHECK();
  const int rc = bspline_prefilter_launch(coeff_scratch, Z, Y, X, st, true);
  if (rc) return rc;
  lbp3d_kernel<<<grid_for(n, 128, 16), 128, 0, st>>>(coeff_scratch, img, img_dt, roi, Z, Y, X, T, out);
  RB_LAUNCH_CHECK();
  return RB_OK;
}

}  // namespace rb
