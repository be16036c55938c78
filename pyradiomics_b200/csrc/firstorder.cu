// Voxel-based first-order feature maps: one thread per centre voxel gathers its kernel window of raw
// intensities + discretised levels and evaluates firstorder_voxel<> (firstorder.cuh).
#include "common.cuh"
#include "firstorder.cuh"

namespace rb {

__device__ __forceinline__ double fo_load(const void* p, int dt, long long i) {
  switch (dt) {
    case 0: return (double)((const int16_t*)p)[i];
    case 1: return (double)((const int32_t*)p)[i];
    case 2: return (double)((const float*)p)[i];
    case 3: return ((const double*)p)[i];
    case 4: return (double)((const uint8_t*)p)[i];
    case 5: return (double)((const uint16_t*)p)[i];
    default: return (double)((const long long*)p)[i];
  }
}

struct FoParams {
  int Z, Y, X, rz, ry, rx, z0, z1, out_z0, dtype, level_bytes;
  double shift, voxel_volume, init_value;
};

template <int WCAP>
__global__ void __launch_bounds__(128)
firstorder_kernel(const void* __restrict__ img, const uint8_t* __restrict__ mask, const uint8_t* __restrict__ centers,
                  const void* __restrict__ lev, FoParams P, double* __restrict__ out, long long fstride) {
  const long long plane = (long long)P.Y * P.X;
  const long long total = (long long)(P.z1 - P.z0) * plane;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int z = P.z0 + (int)(t / plane), rem = (int)(t % plane), y = rem / P.X, x = rem % P.X;
    const long long vi = (long long)z * plane + rem, oi = (long long)(z - P.out_z0) * plane + rem;
    const bool is_center = centers ? centers[vi] != 0 : (mask ? mask[vi] != 0 : true);
    if (!is_center) {
#pragma unroll
      for (int k = 0; k < FIRSTORDER_NF; k++) out[k * fstride + oi] = P.init_value;
      continue;
    }
    double xs[WCAP];
    uint16_t w[WCAP];
    int n = 0, wn = 0;
    for (int dz = -P.rz; dz <= P.rz; dz++)
      for (int dy = -P.ry; dy <= P.ry; dy++)
        for (int dx = -P.rx; dx <= P.rx; dx++, wn++) {
          const int zz = z + dz, yy = y + dy, xx = x + dx;
          w[wn] = 0;
          if (zz < 0 || zz >= P.Z || yy < 0 || yy >= P.Y || xx < 0 || xx >= P.X) continue;
          const long long j = (long long)zz * plane + (long long)yy * P.X + xx;
          if (mask && !mask[j]) continue;
          xs[n++] = fo_load(img, P.dtype, j);
          w[wn] = P.level_bytes == 1 ? (uint16_t)((const uint8_t*)lev)[j] : ((const uint16_t*)lev)[j];
        }
    double f[FIRSTORDER_NF];
    firstorder_voxel<WCAP>(xs, n, w, wn, P.shift, P.voxel_volume, f);
#pragma unroll
    for (int k = 0; k < FIRSTORDER_NF; k++) out[k * fstride + oi] = f[k];
  }
}

int firstorder_launch(const void* img, int dtype, const uint8_t* mask, const uint8_t* centers, const void* lev,
                      int level_bytes, int Z, int Y, int X, int rz, int ry, int rx, double shift, double voxel_volume,
                      double init_value, double* out, long long fstride, int z0, int z1, int out_z0, cudaStream_t st) {
  FoParams P{Z, Y, X, rz, ry, rx, z0, z1, out_z0, dtype, level_bytes, shift, voxel_volume, init_value};
  const long long total = (long long)(z1 - z0) * Y * X;
  if (total <= 0) return RB_OK;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  long long need = (total + 127) / 128, cap = (long long)sms * 32;
  const int grid = (int)(need < cap ? need : cap);
  const int wcap = (2 * rz + 1) * (2 * ry + 1) * (2 * rx + 1);
  if (wcap <= 27) firstorder_kernel<27><<<grid, 128, 0, st>>>(img, mask, centers, lev, P, out, fstride);
  else if (wcap <= 125) firstorder_kernel<125><<<grid, 128, 0, st>>>(img, mask, centers, lev, P, out, fstride);
  else if (wcap <= 343) firstorder_kernel<343><<<grid, 128, 0, st>>>(img, mask, centers, lev, P, out, fstride);
  else return fail(RB_ERR_UNSUPPORTED, "kernelRadius > 3 is outside the implemented envelope");
  RB_LAUNCH_CHECK();
  return RB_OK;
}

}  // namespace rb
