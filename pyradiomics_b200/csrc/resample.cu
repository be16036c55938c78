// Image resampling onto the feature-extraction grid (SURVEY.md section 8f rank 4; reference radiomics/imageoperations.py:
// 448-612 -> sitk.ResampleImageFilter with sitkBSpline for the image, sitkNearestNeighbor for the mask).
//   bspline_prefilter_kernel   cubic B-spline coefficients of the image, one axis per pass, in place: the recursive filter
//                              of ITK's BSplineDecompositionImageFilter (pole sqrt(3)-2, gain 6, mirror boundaries, causal
//                              initialisation truncated at 1e-10 like ITK's) -- one line per thread, threads side by side
//                              along x for the y / z passes (coalesced), 32 lines per warp through a shared tile for x.
//   resample_kernel            one thread per OUTPUT voxel: continuous input index = start + index * step (axis-aligned
//                              grids), cubic B-spline evaluation over the 4x4x4 mirrored neighbourhood / linear / nearest,
//                              0 outside the input buffer, cast to the output pixel type by clamping + truncation like
//                              ITK's ResampleImageFilter (pinned: the reference's `_resampling` baselines are reproduced
//                              exactly with truncation, not with rounding).
#include "common.cuh"

namespace rb {

constexpr double BSPLINE_POLE = -0.26794919243112270647;      // sqrt(3) - 2

__device__ __forceinline__ void bspline_line(double* c, long long stride, int N) {
  if (N == 1) return;
  const double z = BSPLINE_POLE;
  for (int n = 0; n < N; n++) c[n * stride] *= 6.0;            // (1 - z)(1 - 1/z)
  const int horizon = 18;                                        // ceil(log(1e-10) / log|z|)
  if (horizon < N) {
    double zn = z, sum = c[0];
    for (int n = 1; n < horizon; n++) { sum += zn * c[n * stride]; zn *= z; }
    c[0] = sum;
  } else {
    const double iz = 1.0 / z;
    double zn = z, z2n = pow(z, (double)(N - 1));
    double sum = c[0] + z2n * c[(long long)(N - 1) * stride];
    z2n *= z2n * iz;
    for (int n = 1; n <= N - 2; n++) { sum += (zn + z2n) * c[n * stride]; zn *= z; z2n *= iz; }
    c[0] = sum / (1.0 - zn * zn);
  }
  for (int n = 1; n < N; n++) c[n * stride] += z * c[(n - 1) * stride];
  c[(long long)(N - 1) * stride] = (z / (z * z - 1.0)) * (z * c[(long long)(N - 2) * stride] + c[(long long)(N - 1) * stride]);
  for (int n = N - 2; n >= 0; n--) c[n * stride] = z * (c[(n + 1) * stride] - c[n * stride]);
}

__global__ void __launch_bounds__(128)
bspline_prefilter_kernel(double* __restrict__ c, int Z, int Y, int X, int axis) {
  const int N = axis == 0 ? Z : axis == 1 ? Y : X;
  const long long plane = (long long)Y * X;
  const long long stride = axis == 0 ? plane : axis == 1 ? X : 1;
  const long long nlines = (long long)Z * Y * X / N;
  for (long long l = (long long)blockIdx.x * blockDim.x + threadIdx.x; l < nlines; l += (long long)gridDim.x * blockDim.x) {
    long long base;
    if (axis == 2) base = l * X;
    else if (axis == 1) { const long long z = l / X, x = l % X; base = z * plane + x; }
    else base = l;
    bspline_line(c + base, stride, N);
  }
}

// x axis: a warp owns 32 consecutive lines and stages them through shared memory (the whole line: X <= 2048), so global
// accesses are coalesced rows instead of 32 lanes X elements apart
__global__ void __launch_bounds__(128)
bspline_prefilter_x_kernel(double* __restrict__ c, long long nlines, int X) {
  extern __shared__ double sm_lines[];             // [4 warps][32 lines][X + 1]
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  double* mine = sm_lines + (size_t)w * 32 * (X + 1);
  for (long long l0 = ((long long)blockIdx.x * 4 + w) * 32; l0 < nlines; l0 += (long long)gridDim.x * 4 * 32) {
    for (int r = 0; r < 32; r++)
      if (l0 + r < nlines)
        for (int x = lane; x < X; x += 32) mine[r * (X + 1) + x] = c[(l0 + r) * X + x];
    __syncwarp();
    if (l0 + lane < nlines) bspline_line(mine + lane * (X + 1), 1, X);
    __syncwarp();
    for (int r = 0; r < 32; r++)
      if (l0 + r < nlines)
        for (int x = lane; x < X; x += 32) c[(l0 + r) * X + x] = mine[r * (X + 1) + x];
    __syncwarp();
  }
}

__device__ __forceinline__ int mirror(int i, int n) {
  if (n == 1) return 0;
  const int period = 2 * n - 2;
  i = i < 0 ? -i : i;
  i %= period;
  return i >= n ? period - i : i;
}

enum { RS_NEAREST = 0, RS_LINEAR = 1, RS_BSPLINE3 = 3 };
enum { PT_I16 = 0, PT_I32 = 1, PT_F32 = 2, PT_F64 = 3, PT_U8 = 4, PT_U16 = 5, PT_I64 = 6 };

__device__ __forceinline__ double src_value(const void* p, int dt, long long i) {
  switch (dt) {
    case PT_I16: return (double)((const int16_t*)p)[i];
    case PT_I32: return (double)((const int32_t*)p)[i];
    case PT_F32: return (double)((const float*)p)[i];
    case PT_F64: return ((const double*)p)[i];
    case PT_U8: return (double)((const uint8_t*)p)[i];
    case PT_U16: return (double)((const uint16_t*)p)[i];
    default: return (double)((const long long*)p)[i];
  }
}
// ITK ResampleImageFilter::CastPixelWithBoundsChecking: clamp to the pixel range, then static_cast (truncation)
__device__ __forceinline__ void store_value(void* p, int dt, long long i, double v) {
  switch (dt) {
    case PT_I16: ((int16_t*)p)[i] = (int16_t)(v < -32768.0 ? -32768.0 : v > 32767.0 ? 32767.0 : v); break;
    case PT_I32: ((int32_t*)p)[i] = (int32_t)(v < -2147483648.0 ? -2147483648.0 : v > 2147483647.0 ? 2147483647.0 : v); break;
    case PT_F32: ((float*)p)[i] = (float)v; break;
    case PT_F64: ((double*)p)[i] = v; break;
    case PT_U8: ((uint8_t*)p)[i] = (uint8_t)(v < 0.0 ? 0.0 : v > 255.0 ? 255.0 : v); break;
    case PT_U16: ((uint16_t*)p)[i] = (uint16_t)(v < 0.0 ? 0.0 : v > 65535.0 ? 65535.0 : v); break;
    default: ((long long*)p)[i] = (long long)v; break;
  }
}

struct ResampleGeom {
  int iz, iy, ix;          // input size
  int oz, oy, ox;          // output size
  double start[3], step[3];    // continuous input index of output voxel 0 and per-voxel increment, (z, y, x)
};

__global__ void __launch_bounds__(256)
resample_kernel(const void* __restrict__ src, int src_dt, const __grid_constant__ ResampleGeom G, int interp, double default_value,
                void* __restrict__ dst, int dst_dt) {
  const long long n = (long long)G.oz * G.oy * G.ox, oplane = (long long)G.oy * G.ox, iplane = (long long)G.iy * G.ix;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int oz = (int)(t / oplane), rem = (int)(t % oplane), oy = rem / G.ox, ox = rem % G.ox;
    const double cz = G.start[0] + G.step[0] * oz, cy = G.start[1] + G.step[1] * oy, cx = G.start[2] + G.step[2] * ox;
    // ITK IsInsideBuffer: continuous index in [-0.5, size - 0.5)
    const bool inside = cz >= -0.5 && cz < G.iz - 0.5 && cy >= -0.5 && cy < G.iy - 0.5 && cx >= -0.5 && cx < G.ix - 0.5;
    double v = default_value;
    if (inside) {
      if (interp == RS_NEAREST) {
        const int z = (int)floor(cz + 0.5), y = (int)floor(cy + 0.5), x = (int)floor(cx + 0.5);       // RoundHalfIntegerUp
        v = src_value(src, src_dt, (long long)min(max(z, 0), G.iz - 1) * iplane + (long long)min(max(y, 0), G.iy - 1) * G.ix + min(max(x, 0), G.ix - 1));
      } else if (interp == RS_LINEAR) {
        const double fz = floor(cz), fy = floor(cy), fx = floor(cx);
        const double wz = cz - fz, wy = cy - fy, wx = cx - fx;
        v = 0;
        for (int dz = 0; dz < 2; dz++) for (int dy = 0; dy < 2; dy++) for (int dx = 0; dx < 2; dx++) {
          const int z = min(max((int)fz + dz, 0), G.iz - 1), y = min(max((int)fy + dy, 0), G.iy - 1), x = min(max((int)fx + dx, 0), G.ix - 1);
          v += (dz ? wz : 1 - wz) * (dy ? wy : 1 - wy) * (dx ? wx : 1 - wx) * src_value(src, src_dt, (long long)z * iplane + (long long)y * G.ix + x);
        }
      } else {
        // cubic B-spline over the 4x4x4 neighbourhood starting at floor(c) - 1, mirrored at the borders;
        // src = the coefficients (float64) from bspline_prefilter
        const double* c = (const double*)src;
        double W[3][4];
        int I[3][4];
        const double cc[3] = {cz, cy, cx};
        const int nn[3] = {G.iz, G.iy, G.ix};
#pragma unroll
        for (int d = 0; d < 3; d++) {
          const double f = floor(cc[d]);
          const double w = cc[d] - f;
          W[d][3] = (1.0 / 6.0) * w * w * w;
          W[d][0] = (1.0 / 6.0) + 0.5 * w * (w - 1.0) - W[d][3];
          W[d][2] = w + W[d][0] - 2.0 * W[d][3];
          W[d][1] = 1.0 - W[d][0] - W[d][2] - W[d][3];
#pragma unroll
          for (int k = 0; k < 4; k++) I[d][k] = mirror((int)f - 1 + k, nn[d]);
        }
        v = 0;
#pragma unroll
        for (int a = 0; a < 4; a++)
#pragma unroll
          for (int b = 0; b < 4; b++) {
            const double wab = W[0][a] * W[1][b];
            const long long row = (long long)I[0][a] * iplane + (long long)I[1][b] * G.ix;
#pragma unroll
            for (int k = 0; k < 4; k++) v += wab * W[2][k] * c[row + I[2][k]];
          }
      }
    }
    store_value(dst, dst_dt, t, v);
  }
}

static int grid_rs(long long n, int block, int per_sm) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  long long need = (n + block - 1) / block, cap = (long long)sms * per_sm;
  return (int)(need < cap ? (need < 1 ? 1 : need) : cap);
}

int bspline_prefilter_launch(double* coeffs, int Z, int Y, int X, cudaStream_t st) {
  if (Z < 1 || Y < 1 || X < 1) return fail(RB_ERR_ARG, "empty volume");
  const long long n = (long long)Z * Y * X;
  // ITK's BSplineDecompositionImageFilter filters dimension 0 (x) first, then y, then z
  if (X > 1) {
    const size_t sh = (size_t)4 * 32 * (X + 1) * sizeof(double);
    if (sh <= 200 * 1024) {
      cudaFuncSetAttribute(bspline_prefilter_x_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh);
      bspline_prefilter_x_kernel<<<grid_rs((n / X + 31) / 32, 4, 4), 128, sh, st>>>(coeffs, n / X, X);
    } else {
      bspline_prefilter_kernel<<<grid_rs(n / X, 128, 8), 128, 0, st>>>(coeffs, Z, Y, X, 2);
    }
  }
  if (Y > 1) bspline_prefilter_kernel<<<grid_rs(n / Y, 128, 8), 128, 0, st>>>(coeffs, Z, Y, X, 1);
  if (Z > 1) bspline_prefilter_kernel<<<grid_rs(n / Z, 128, 8), 128, 0, st>>>(coeffs, Z, Y, X, 0);
  RB_LAUNCH_CHECK();
  return RB_OK;
}

int resample_launch(const void* src, int src_dt, const int* in_size, void* dst, int dst_dt, const int* out_size, const double* start,
                    const double* step, int interp, double default_value, cudaStream_t st) {
  if (interp != RS_NEAREST && interp != RS_LINEAR && interp != RS_BSPLINE3) return fail(RB_ERR_UNSUPPORTED, "interpolator %d (0 nearest, 1 linear, 3 cubic B-spline)", interp);
  if (interp == RS_BSPLINE3 && src_dt != PT_F64) return fail(RB_ERR_ARG, "the B-spline evaluation reads float64 coefficients");
  ResampleGeom G;
  G.iz = in_size[0]; G.iy = in_size[1]; G.ix = in_size[2];
  G.oz = out_size[0]; G.oy = out_size[1]; G.ox = out_size[2];
  for (int d = 0; d < 3; d++) { G.start[d] = start[d]; G.step[d] = step[d]; }
  const long long n = (long long)G.oz * G.oy * G.ox;
  if (n <= 0) return RB_OK;
  resample_kernel<<<grid_rs(n, 256, 8), 256, 0, st>>>(src, src_dt, G, interp, default_value, dst, dst_dt);
  RB_LAUNCH_CHECK();
  return RB_OK;
}

}  // namespace rb
