// 2-D local binary pattern image type (reference radiomics/imageoperations.py:1094-1166, getLBP2DImage).
//   lbp2d_kernel<METHOD, T>  one thread per voxel of the whole volume, all slices in one launch, threads numbered in memory
//                            order (x fastest, grid-stride) whatever the slicing axis, so the centre loads and the stores
//                            coalesce.  The slice a voxel belongs to is an index mapping (lbp2d_slice_of), not a transposed
//                            copy; the P samples' 4 corners are read in the image's own dtype and come from L1 / L2
//                            (neighbouring threads share them).  The per-pixel math is lbp2d_pixel (lbp2d.cuh).  T = double
//                            is rb_lbp2d_dev's float64 volume; any other T is rb_lbp2d_cast_dev's store in the image's own
//                            dtype through numpy_cast, the reference's per-slice assignment without a float64 volume between.
#include "common.cuh"
#include "lbp2d.cuh"

namespace rb {

template <int METHOD, typename T>
__global__ void __launch_bounds__(256)
lbp2d_kernel(const void* __restrict__ img, int dt, int Z, int Y, int X, int axis, const __grid_constant__ Lbp2dOffsets O,
             T* __restrict__ out) {
  const long long n = (long long)Z * Y * X, plane = (long long)Y * X;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(t / plane), rem = (int)(t % plane), y = rem / X, x = rem % X;
    Lbp2dSlice s;
    int r, c;
    lbp2d_slice_of(img, dt, Z, Y, X, axis, z, y, x, s, r, c);
    out[t] = numpy_cast<T>(lbp2d_pixel<METHOD>(s, r, c, O));
  }
}

template <typename T>
static void lbp2d_launch_as(dim3 grid, const void* img, int dt, int Z, int Y, int X, int axis, const Lbp2dOffsets& O, int method,
                            void* out, cudaStream_t st) {
  T* o = (T*)out;
  switch (method) {
    case LBP2D_DEFAULT: lbp2d_kernel<LBP2D_DEFAULT, T><<<grid, 256, 0, st>>>(img, dt, Z, Y, X, axis, O, o); break;
    case LBP2D_ROR: lbp2d_kernel<LBP2D_ROR, T><<<grid, 256, 0, st>>>(img, dt, Z, Y, X, axis, O, o); break;
    case LBP2D_UNIFORM: lbp2d_kernel<LBP2D_UNIFORM, T><<<grid, 256, 0, st>>>(img, dt, Z, Y, X, axis, O, o); break;
    case LBP2D_NRI_UNIFORM: lbp2d_kernel<LBP2D_NRI_UNIFORM, T><<<grid, 256, 0, st>>>(img, dt, Z, Y, X, axis, O, o); break;
    default: lbp2d_kernel<LBP2D_VAR, T><<<grid, 256, 0, st>>>(img, dt, Z, Y, X, axis, O, o); break;
  }
}

// out_dt: the rb_dtype code of `out` (RB_DT_FLOAT64 for rb_lbp2d_dev, the image's own for rb_lbp2d_cast_dev)
int lbp2d_launch(const void* img, int dt, int Z, int Y, int X, int axis, int P, const double* rp, const double* cp, int method,
                 int out_dt, void* out, cudaStream_t st) {
  if (!img || !rp || !cp || !out) return fail(RB_ERR_ARG, "lbp2d: null argument");
  if (Z < 1 || Y < 1 || X < 1) return fail(RB_ERR_ARG, "lbp2d: empty volume %d x %d x %d", Z, Y, X);
  if (axis < 0 || axis > 2) return fail(RB_ERR_ARG, "lbp2d: axis %d (0..2)", axis);
  if (method < LBP2D_DEFAULT || method > LBP2D_VAR) return fail(RB_ERR_ARG, "lbp2d: unknown method code %d", method);
  if (P < 1 || P > LBP2D_MAX_P) return fail(RB_ERR_UNSUPPORTED, "lbp2d: %d samples (1..%d)", P, LBP2D_MAX_P);
  Lbp2dOffsets O;
  O.P = P;
  O.pad_ = 0;
  for (int k = 0; k < LBP2D_MAX_P; k++) {
    O.rp[k] = k < P ? rp[k] : 0.0;
    O.cp[k] = k < P ? cp[k] : 0.0;
  }
  const long long n = (long long)Z * Y * X;
  const dim3 grid = grid_for(n, 256, 16);
  switch (out_dt) {
    case RB_DT_INT16: lbp2d_launch_as<int16_t>(grid, img, dt, Z, Y, X, axis, O, method, out, st); break;
    case RB_DT_INT32: lbp2d_launch_as<int32_t>(grid, img, dt, Z, Y, X, axis, O, method, out, st); break;
    case RB_DT_FLOAT32: lbp2d_launch_as<float>(grid, img, dt, Z, Y, X, axis, O, method, out, st); break;
    case RB_DT_UINT8: lbp2d_launch_as<uint8_t>(grid, img, dt, Z, Y, X, axis, O, method, out, st); break;
    case RB_DT_UINT16: lbp2d_launch_as<uint16_t>(grid, img, dt, Z, Y, X, axis, O, method, out, st); break;
    case RB_DT_INT64: lbp2d_launch_as<int64_t>(grid, img, dt, Z, Y, X, axis, O, method, out, st); break;
    default: lbp2d_launch_as<double>(grid, img, dt, Z, Y, X, axis, O, method, out, st); break;
  }
  RB_LAUNCH_CHECK();
  return RB_OK;
}

}  // namespace rb
